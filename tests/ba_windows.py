"""Edits of synthetic localBA windows (ov2slam_b200.synth.make_ba_problem) whose Ceres program differs from the declared one:
keyframes no residual touches, a keyframe whose residuals the first outlier scan removes, a stereo keyframe touched only by
right-camera residuals in its own anchor frame, landmarks without residuals.  Shared by the GPU path tests and the oracle
pins; every edit returns a new window and leaves its argument alone."""
import numpy as np

OBS_KEYS = ("obs_cam", "obs_lm", "obs_px", "obs_type")


def clone(pb):
    return {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in pb.items()}


def used_keyframes(pb, active=None):
    """bool[ncam]: the non-constant keyframes that some (active) pose-dependent residual touches as observer or anchor, i.e.
    the pose blocks Program::RemoveFixedBlocks keeps (a right-camera residual in the anchor frame, obs_type 2, depends on
    the inverse depth alone)."""
    m = np.ones(len(pb["obs_cam"]), bool) if active is None else np.asarray(active, bool).copy()
    if pb.get("obs_type") is not None:
        m &= pb["obs_type"] != 2
    u = np.zeros(len(pb["pose"]), bool)
    u[pb["obs_cam"][m]] = True
    u[pb["lm_anchor_cam"][pb["obs_lm"][m]]] = True
    return u & (pb["pose_const"] == 0)


def _append_keyframes(pb, k, const):
    out = clone(pb)
    step = np.zeros((k, 7))
    step[:, 0] = 0.2 * np.arange(1, k + 1)
    for key in ("pose", "truth_pose"):
        if key in out:
            out[key] = np.ascontiguousarray(np.vstack([out[key], out[key][-1] + step]))
    out["pose_const"] = np.concatenate([out["pose_const"], np.full(k, 1 if const else 0, np.uint8)])
    return out


def add_unused_keyframes(pb, k):
    """Append k non-constant keyframes that no residual touches (Ceres drops their blocks)."""
    return _append_keyframes(pb, k, const=False)


def add_constant_keyframes(pb, k):
    """Append k constant keyframes that no residual touches: a larger keyframe table, the same program."""
    return _append_keyframes(pb, k, const=True)


def push_keyframe(pb, kf, px=40.0, seed=0):
    """Move every residual whose observer or anchor is keyframe `kf` by `px` pixels in a random direction: the first outlier
    scan flags them all, so the refinement's program has neither the keyframe nor the landmarks anchored in it."""
    out = clone(pb)
    hit = (out["obs_cam"] == kf) | (out["lm_anchor_cam"][out["obs_lm"]] == kf)
    ang = np.random.default_rng(seed).uniform(0, 2 * np.pi, int(hit.sum()))
    out["obs_px"][hit] += px * np.stack([np.cos(ang), np.sin(ang)], 1)
    out["obs_px"] = out["obs_px"].astype(np.float32).astype(np.float64)
    return out


def keep_residuals(pb, keep):
    out = clone(pb)
    for key in OBS_KEYS:
        if out.get(key) is not None:
            out[key] = np.ascontiguousarray(out[key][keep])
    return out


def type2_only_keyframe(pb, kf):
    """Stereo window: every landmark anchored in `kf` keeps only its right-camera residual in the anchor frame (obs_type 2)
    and `kf` observes nothing else, so no pose-dependent residual touches the keyframe."""
    anch = pb["lm_anchor_cam"][pb["obs_lm"]] == kf
    drop = (pb["obs_cam"] == kf) & (pb["obs_type"] != 2) | anch & (pb["obs_type"] != 2)
    return keep_residuals(pb, ~drop)


def drop_landmark_residuals(pb, lms):
    """Remove every residual of the landmarks `lms`: they stay in the window without a residual block."""
    return keep_residuals(pb, ~np.isin(pb["obs_lm"], lms))


def small_shrinking_windows():
    """Oracle-size windows of the four program changes, by name: two unused non-constant keyframes; keyframe 5 dropping out
    of the refinement (with the landmarks anchored in it); stereo keyframe 2 touched only by anchor-frame right-camera
    residuals; two landmarks in three without a residual (fewer residuals than landmarks)."""
    from ov2slam_b200 import synth
    lone = synth.make_ba_problem(64, 6, 300, 450)
    return {
        "unused_keyframes": add_unused_keyframes(synth.make_ba_problem(61, 6, 200, 800), 2),
        "keyframe_leaves_refinement": push_keyframe(synth.make_ba_problem(62, 7, 250, 1000), 5),
        "type2_only_keyframe": type2_only_keyframe(synth.make_ba_problem(63, 6, 200, 600, stereo=True), 2),
        "landmarks_without_residuals": drop_landmark_residuals(lone, np.arange(300)[np.arange(300) % 3 != 0]),
    }
