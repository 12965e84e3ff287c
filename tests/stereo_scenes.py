"""Synthetic stereo keyframes for MapManager::stereoMatching: one keyframe of keypoints on an EuRoC-sized rig, as the self-test of the
drop-in (host/stereo_selftest.cpp) reads it, as the reference's own stereoMatching is driven with it, and as ov2_stereo_matching's
flat arrays."""
import numpy as np

from ov2slam_b200 import synth


def quat_of(R):
    """Unit quaternion (x, y, z, w) of a rotation matrix with positive trace (small rotations only)."""
    w = 0.5 * np.sqrt(1.0 + np.trace(R))
    return np.array([(R[2, 1] - R[1, 2]) / (4 * w), (R[0, 2] - R[2, 0]) / (4 * w), (R[1, 0] - R[0, 1]) / (4 * w), w])


def stereo_scene(seed, rect, nkps=320, w=752, h=480, cs=35, depth=None, Dr=None):
    """Dr: the right camera's k1, k2, p1, p2 (None: no distortion model)."""
    rng = np.random.default_rng(seed)
    K = np.array([458.654, 457.296, 367.215, 248.375])
    Rrig = np.eye(3) if rect else synth._so3_exp(np.array([0.004, -0.006, 0.003]))
    trig = np.array([0.11, 0.0, 0.0]) if rect else np.array([0.11, 0.002, -0.001])        # right camera in the left camera's frame
    Rwc, twc = synth._so3_exp(rng.normal(0, 0.2, 3)), rng.normal(0, 1.0, 3)
    px = np.stack([rng.uniform(4, w - 4, nkps), rng.uniform(4, h - 4, nkps)], 1).astype(np.float32)
    bv = np.stack([(px[:, 0].astype(np.float64) - K[2]) / K[0], (px[:, 1].astype(np.float64) - K[3]) / K[1], np.ones(nkps)], 1)
    bv /= np.linalg.norm(bv, axis=1, keepdims=True)
    is3d = rng.random(nkps) < 0.6
    has_mp = is3d & (rng.random(nkps) > 0.08)
    z = rng.uniform(0.8, 8.0, nkps)
    cam = bv / bv[:, 2:3] * z[:, None] + rng.normal(0, 0.002, (nkps, 3))
    if depth is not None:
        cam = bv / bv[:, 2:3] * depth
    wpt = cam @ Rwc.T + twc
    # p_right = R_rl p_left + t_rl ;  F with  r^T F l = 0
    Rrl, trl = Rrig.T, -Rrig.T @ trig
    tx = np.array([[0, -trl[2], trl[1]], [trl[2], 0, -trl[0]], [-trl[1], trl[0], 0]])
    Kmat = np.array([[K[0], 0, K[2]], [0, K[1], K[3]], [0, 0, 1]])
    Frl = np.linalg.inv(Kmat).T @ tx @ Rrl @ np.linalg.inv(Kmat)
    return dict(rect=rect, w=w, h=h, cs=cs, nbw=int(np.ceil(w / cs)), nbh=int(np.ceil(h / cs)), K=K, Rrig=Rrig, trig=trig, Rwc=Rwc, twc=twc,
                Frl=Frl, lmid=(100 + np.arange(nkps)).astype(np.int32), is3d=is3d, has_mp=has_mp, px=px, unpx=px.copy(), bv=bv, wpt=wpt,
                Dr=None if Dr is None else np.asarray(Dr, np.float64))


def write_stereo_scene(path, sc):
    """The scene file of host/stereo_selftest.cpp."""
    n = len(sc["lmid"])
    with open(path, "wb") as f:
        f.write(np.array([n, sc["rect"], sc["w"], sc["h"], sc["cs"], sc["nbw"], sc["nbw"] * sc["nbh"]], np.int32).tobytes())
        for a in (sc["K"], sc["K"], np.concatenate([sc["trig"], quat_of(sc["Rrig"])]), np.concatenate([sc["twc"], quat_of(sc["Rwc"])]), sc["Frl"]):
            f.write(np.ascontiguousarray(a, np.float64).tobytes())
        for i in range(n):
            f.write(np.array([sc["lmid"][i], sc["is3d"][i], sc["has_mp"][i]], np.int32).tobytes())
            f.write(np.concatenate([sc["px"][i], sc["unpx"][i]]).astype(np.float32).tobytes())
            f.write(np.concatenate([sc["bv"][i], sc["wpt"][i]]).astype(np.float64).tobytes())
        if sc["Dr"] is not None:
            f.write(np.ascontiguousarray(sc["Dr"], np.float64).tobytes())


def read_stereo_result(path):
    """host/stereo_selftest.cpp's result: the keypoint order (lmids as Frame::getKeypoints() returned them), per keypoint in that
    order the stereo flag and the right pixel, the number of observations removed from the map, and Tcw and Trl (12 doubles each)
    as the drop-in flattens them."""
    raw = np.fromfile(path, np.uint8)
    n = int(raw[:4].view(np.int32)[0])
    order = raw[4:4 + 4 * n].view(np.int32)
    rec = raw[4 + 4 * n:4 + 16 * n].reshape(n, 12)
    is_stereo = rec[:, :4].copy().view(np.int32).reshape(n) != 0
    rpx = rec[:, 4:].copy().view(np.float32).reshape(n, 2)
    removed = int(raw[4 + 16 * n:8 + 16 * n].view(np.int32)[0])
    T = raw[8 + 16 * n:].copy().view(np.float64)
    assert len(T) == 24
    return dict(order=order, is_stereo=is_stereo, rpx=rpx, removed=removed, Tcw=T[:12], Trl=T[12:])


def flat_scene(sc, order):
    """The scene as ov2_stereo_matching's arrays for one keyframe, keypoints in the reference's Frame::getKeypoints() order, the grid
    lists in insertion (scene) order."""
    idx = {int(l): i for i, l in enumerate(sc["lmid"])}
    perm = np.array([idx[int(l)] for l in order], np.int64)
    pos = np.empty(len(perm), np.int64)
    pos[perm] = np.arange(len(perm))
    Rcw = sc["Rwc"].T
    Rrl = sc["Rrig"].T
    cs, nbw, nbh = sc["cs"], sc["nbw"], sc["nbh"]
    cells = [[] for _ in range(nbw * nbh)]
    for i in range(len(sc["lmid"])):
        p = sc["px"][i]
        cells[int(np.floor(p[1] / np.float32(cs))) * nbw + int(np.floor(p[0] / np.float32(cs)))].append(int(pos[i]))
    return dict(offsets=np.array([0, len(perm)], np.int32), Tcw=np.concatenate([Rcw.reshape(-1), -Rcw @ sc["twc"]])[None],
                K=np.asarray(sc["K"], np.float64)[None], Trl=np.concatenate([Rrl.reshape(-1), -Rrl @ sc["trig"]])[None],
                dist=None if sc["Dr"] is None else np.concatenate([sc["Dr"], [0.0]])[None],
                Frl=np.asarray(sc["Frl"]).reshape(1, 9), img_wh=np.array([[sc["w"], sc["h"]]], np.int32),
                px=sc["px"][perm], unpx=sc["unpx"][perm], bv=sc["bv"][perm], is3d=sc["is3d"][perm].astype(np.uint8),
                has_mp=sc["has_mp"][perm].astype(np.uint8), wpt=sc["wpt"][perm], rectified=int(sc["rect"]),
                cell_offsets=np.array([0, nbw * nbh], np.int32), grid=np.array([[cs, nbw]], np.int32),
                cell_ptr=np.concatenate([[0], np.cumsum([len(c) for c in cells])]).astype(np.int32),
                cell_kps=np.array([j for c in cells for j in c], np.int32))
