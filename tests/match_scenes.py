"""Hand-placed Mapper::matchToMap problems (the flat arrays ov2_match_to_map takes) for the edge tests: keypoints, map points,
descriptors, keyframe sets and candidates put where a test wants them, on any image and grid geometry, with world points that
project exactly onto a chosen pixel.  The frame and every keyframe sit at the world origin (identity Tcw), so a camera-frame
point is its world point and Z is the world z exactly."""
import numpy as np

from oracle import match_ref as M

f32 = np.float32
IDENTITY = np.array([1.0, 0, 0, 0, 1.0, 0, 0, 0, 1.0, 0, 0, 0])
EUROC_DIST = np.array([-0.28340811, 0.07395907, 0.00019359, 1.76187114e-05, 0.0])
# image size and pinhole intrinsics of the shipped parameter files' cameras; the grid cell (nmaxdist) is 35, 45 or 50 px
GEOMETRIES = {"euroc": (752, 480, (458.654, 457.296, 367.215, 248.375)),
              "kitti": (1241, 376, (718.856, 718.856, 607.1928, 185.2157)),
              "tartanair": (640, 480, (320.0, 320.0, 320.0, 240.0))}


def flip(d, nbits, start=0):
    """`d` with bits start .. start + nbits - 1 flipped: Hamming distance `nbits` from `d`."""
    out = np.array(d, np.uint8).copy()
    for b in range(start, start + nbits):
        out[b >> 3] ^= np.uint8(1 << (b & 7))
    return out


class Scene:
    def __init__(self, w=752, h=480, cs=35, K=GEOMETRIES["euroc"][2], dist=None, nkfs=1, dmax=4.0, ratio=0.2, view_th=0.5, seed=0):
        self.w, self.h, self.cs, self.K, self.dist, self.nkfs = w, h, cs, np.asarray(K, np.float64), dist, nkfs
        self.dmax, self.ratio, self.view_th = f32(dmax), f32(ratio), f32(view_th)
        self.rng = np.random.default_rng(seed)
        self.kp_px, self.kp_lm = [], []
        self.mp_xyz, self.mp_desc, self.mp_obs = [], [], []
        self.cand = []

    def random_desc(self):
        return self.rng.integers(0, 256, 32, dtype=np.uint8)

    def project(self, xyz):
        return M.project_dist(M.camera_point(IDENTITY, xyz), self.K, self.dist)

    def map_point(self, xyz, descs=(), kfs=(), obs_px=None):
        """A map point with the given descriptors, observed by keyframes `kfs` at `obs_px` (default: where `xyz` projects, so
        that a candidate at the same place has no co-projection error).  Returns its index."""
        if obs_px is None:
            obs_px = [self.project(xyz)] * len(kfs) if len(kfs) else []
        self.mp_xyz.append(np.asarray(xyz, np.float64))
        self.mp_desc.append([np.asarray(d, np.uint8) for d in descs])
        self.mp_obs.append([(int(k), tuple(f32(v) for v in p)) for k, p in zip(kfs, obs_px)])
        return len(self.mp_xyz) - 1

    def keypoint(self, px, lm=-1):
        self.kp_px.append((f32(px[0]), f32(px[1])))
        self.kp_lm.append(int(lm))
        return len(self.kp_px) - 1

    def candidate(self, mp):
        self.cand.append(int(mp))
        return len(self.cand) - 1

    @staticmethod
    def _walk(f, t, target, up):
        """Step t one representable value at a time (its own type: float or double) until the non-decreasing f(t) equals
        `target`; where f jumps over it, stop on the side `up` asks for."""
        for _ in range(100000):
            val = f(t)
            if val == target:
                return t
            nt = np.nextafter(t, t.dtype.type(np.inf if val < target else -np.inf))
            nval = f(nt)
            if (val < target) != (nval < target) and nval != target:
                return (nt if val < target else t) if up else (t if val < target else nt)
            t = nt
        raise AssertionError("projection walk did not converge")

    def point_at(self, u, v, z=1.0, up=(True, True)):
        """A world point at depth `z` that projects onto pixel (u, v) exactly where that pixel is reachable; otherwise, per axis,
        onto the nearest reachable value above (up) or below it."""
        fx, fy, cx, cy = (float(k) for k in self.K)
        u, v = f32(u), f32(v)
        if self.dist is None:
            # pinhole: px depends on X alone, py on Y alone; walk them one double at a time
            X = self._walk(lambda X: self.project((X, 0.0, z))[0], np.float64((float(u) - cx) / fx * z), u, up[0])
            Y = self._walk(lambda Y: self.project((0.0, Y, z))[1], np.float64((float(v) - cy) / fy * z), v, up[1])
            return np.array([float(X), float(Y), z])
        # radial-tangential: the normalised point is rounded to float first, so walk over floats; x and y interact through r2
        k1, k2, p1, p2, k3 = (float(c) for c in self.dist)
        xd, yd = (float(u) - cx) / fx, (float(v) - cy) / fy
        x, y = xd, yd
        for _ in range(50):                           # fixed-point undistortion in double as the starting point
            r2 = x * x + y * y
            cd = 1 + k1 * r2 + k2 * r2 * r2 + k3 * r2 ** 3
            x, y = (xd - (2 * p1 * x * y + p2 * (r2 + 2 * x * x))) / cd, (yd - (p1 * (r2 + 2 * y * y) + 2 * p2 * x * y)) / cd
        x, y = f32(x), f32(y)
        proj = lambda a, b: M.project_dist((float(a), float(b), 1.0), self.K, self.dist)
        for _ in range(4):
            x = self._walk(lambda a: proj(a, y)[0], x, u, up[0])
            y = self._walk(lambda b: proj(x, b)[1], y, v, up[1])
        xyz = np.array([float(x) * z, float(y) * z, z])
        assert self.project(xyz) == proj(x, y), "the depth changed the normalised point"
        return xyz

    def scene(self):
        nbw, nbh = int(np.ceil(f32(self.w) / self.cs)), int(np.ceil(f32(self.h) / self.cs))
        kp_px = np.array(self.kp_px, np.float32).reshape(-1, 2)
        cell = (np.floor(kp_px[:, 1] / f32(self.cs)).astype(int) * nbw + np.floor(kp_px[:, 0] / f32(self.cs)).astype(int))
        assert np.all((cell >= 0) & (cell < nbw * nbh)), "keypoint outside the grid"
        kfmask = np.zeros((len(self.mp_xyz), 4), np.uint64)
        obs_ptr, obs_kf, obs_px = [0], [], []
        for m, obs in enumerate(self.mp_obs):
            for k, p in obs:
                assert 0 <= k < min(self.nkfs, 256)
                kfmask[m, k >> 6] |= np.uint64(1) << np.uint64(k & 63)
                obs_kf.append(k)
                obs_px.append(p)
            obs_ptr.append(len(obs_kf))
        descs = [d for ds in self.mp_desc for d in ds]
        return dict(K=self.K, dist=self.dist, img_w=self.w, img_h=self.h, ncellsize=self.cs, nbwcells=nbw, Tcw=IDENTITY.copy(),
                    cell_ptr=np.concatenate([[0], np.cumsum(np.bincount(cell, minlength=nbw * nbh))]).astype(np.int32),
                    cell_kp=np.argsort(cell, kind="stable").astype(np.int32), kp_px=kp_px,
                    kp_lm=np.array(self.kp_lm, np.int32), mp_xyz=np.array(self.mp_xyz, np.float64).reshape(-1, 3),
                    mp_desc_ptr=np.concatenate([[0], np.cumsum([len(ds) for ds in self.mp_desc])]).astype(np.int32),
                    desc=np.array(descs, np.uint8).reshape(-1, 32), mp_kfmask=kfmask, mp_obs_ptr=np.array(obs_ptr, np.int32),
                    obs_kf=np.array(obs_kf, np.int32), obs_px=np.array(obs_px, np.float32).reshape(-1, 2),
                    kf_Tcw=np.tile(IDENTITY, (self.nkfs, 1)), cand_mp=np.array(self.cand, np.int32),
                    dmaxpxdist=self.dmax, fdistratio=self.ratio, view_th=self.view_th)


# ------------------------------------------------------------------------------------------------------------ lane rounds
CORNER = [(-1, -1), (-1, 0), (0, -1), (0, 0)]       # the four cells a projection visits, in the order the kernel visits them


def lane_scene(counts, dists, seed=0):
    """One candidate projecting 1.5 px right of and below the corner of cell (3, 4) of the 35-px EuRoC grid, and counts[i]
    keypoints in the i-th of the four cells it visits, all within 2.9 px of the projection.  dists[(i, q)] is the Hamming
    distance of the q-th keypoint of cell i; the other keypoints cycle through: no map point, a map point without descriptor,
    a map point ~128 bits away."""
    s = Scene(seed=seed)
    r0, c0 = 3, 4
    D = s.random_desc()
    xyz = s.point_at(c0 * 35 + 1.5, r0 * 35 + 1.5, z=2.0)
    s.candidate(s.map_point(xyz, [D]))
    ids = {}
    for i, (dr, dc) in enumerate(CORNER):
        px = (c0 * 35 + (1.5 if dc == 0 else -0.5), r0 * 35 + (1.5 if dr == 0 else -0.5))
        for q in range(counts[i]):
            if (i, q) in dists:
                lm = s.map_point(xyz, [flip(D, dists[(i, q)])])
            elif q % 3 == 0:
                lm = -1
            elif q % 3 == 1:
                lm = s.map_point(xyz)
            else:
                lm = s.map_point(xyz, [s.random_desc()])
            ids[(i, q)] = s.keypoint(px, lm)
    return s.scene(), ids


LANE_CASES = {
    # the best and the second in different rounds of the same cell, then a third round, and across cells
    "best_second_rounds": ((32, 33, 64, 65), {(2, 10): 20, (2, 50): 3, (3, 64): 30, (0, 31): 25}, (2, 50)),
    # equal distances at lane 31 of one round and lane 0 of the next: the later keypoint takes the best place
    "tie_lane31_lane0": ((5, 5, 64, 5), {(2, 31): 0, (2, 32): 0}, (2, 32)),
    "tie_across_cells": ((33, 5, 5, 40), {(0, 32): 0, (3, 0): 0}, (3, 0)),
    # the only valid keypoint in a final partial round
    "only_in_last_round_65": ((5, 5, 65, 5), {(2, 64): 7}, (2, 64)),
    "only_in_last_round_100": ((100, 5, 5, 5), {(0, 99): 7}, (0, 99)),
    "only_in_last_round_33": ((5, 33, 5, 5), {(1, 32): 7}, (1, 32)),
    # many valid keypoints over four rounds: the best in round 3, the second in round 1
    "dense_100": ((100, 64, 65, 32), {**{(0, q): 40 + q % 9 for q in range(1, 100, 2)}, (0, 70): 5, (0, 3): 30, (3, 31): 33}, (0, 70)),
    # best and second within the ratio: rejected, with the second in a later round
    "ratio_across_rounds": ((5, 5, 64, 5), {(2, 5): 30, (2, 40): 32}, None),
}


# -------------------------------------------------------------------------------------------------------- keyframe masks
def mask_scene(nkfs, seed=0):
    """Candidates along a row, each with one keypoint at its projection (Hamming distance 5).  Returns the scene and, per
    candidate, whether its keyframe set is disjoint from the keypoint's map point's (the pair must then stay a candidate)."""
    s = Scene(nkfs=nkfs, seed=seed)
    words = (nkfs + 63) // 64
    cases = []
    for w in range(words):                                          # overlap only in word w (the other words disjoint)
        top = min(64 * w + 63, nkfs - 1)
        for bit in sorted({64 * w, top}):
            other_c = [64 * v + 1 for v in range(words) if v != w and 64 * v + 1 < nkfs]
            other_k = [64 * v + 2 for v in range(words) if v != w and 64 * v + 2 < nkfs]
            cases.append((other_c + [bit], other_k + [bit], False))
    cases.append(([64 * v + 1 for v in range(words) if 64 * v + 1 < nkfs], [64 * v + 2 for v in range(words) if 64 * v + 2 < nkfs], True))
    cases.append(([nkfs - 1], [nkfs - 2], True))
    want = []
    for i, (kc, kk, disjoint) in enumerate(cases):
        u, v = 20.5 + 30 * (i % 24), 40.5 + 60 * (i // 24)
        xyz = s.point_at(u, v, z=3.0)
        D = s.random_desc()
        s.candidate(s.map_point(xyz, [D], kfs=kc))
        s.keypoint(s.project(xyz), s.map_point(xyz, [flip(D, 5)], kfs=kk))
        want.append(disjoint)
    return s.scene(), want


# ------------------------------------------------------------------------------------------------------------ thresholds
def threshold_scene(kind, on_edge):
    """One candidate at pixel (200.5, 150.5) with its threshold parameter set to exactly the value the oracle computes for
    it (on_edge) or one float / double past it.  Returns (scene, the oracle's value equals the parameter on the edge,
    whether the candidate must match)."""
    s = Scene()
    D = s.random_desc()
    z = 2.0
    if kind == "depth":
        z = 0.1 if on_edge else float(np.nextafter(0.1, 0.0))
    xyz = s.point_at(200.5, 150.5, z=2.0 if kind != "depth" else 0.1)
    xyz[2] = z                                                       # the depth case steps z alone
    p = s.project(xyz)
    cand_desc = [] if kind == "no_descriptor" else [D]
    s.candidate(s.map_point(xyz, cand_desc))
    kp_off = (2.5, 1.5) if kind == "pixel" else (0.0, 0.0)
    kfs, obs = (), None
    if kind == "no_observations" and not on_edge:                  # one observation half a pixel off: a mean of 0.5
        kfs, obs = (0,), [(p[0] + f32(0.5), p[1])]
    if kind == "coprojection":
        kfs = (0, 1, 2)
        obs = [(p[0] + f32(1.3), p[1] + f32(0.4)), (p[0] + f32(0.2), p[1] + f32(2.1)), (p[0] + f32(1.7), p[1] + f32(1.1))]
        s.nkfs = 3
    nbits = {"hamming": 64 if on_edge else 65}.get(kind, 10)
    lm = s.map_point(xyz, [flip(D, nbits)], kfs=kfs, obs_px=obs)
    s.keypoint((p[0] + f32(kp_off[0]), p[1] + f32(kp_off[1])), lm)
    if kind == "ratio":                                              # a second keypoint 50 bits away
        s.keypoint(p, s.map_point(xyz, [flip(D, 50, start=100)]))
    sc = s.scene()
    X, Y, Z = M.camera_point(sc["Tcw"], xyz)
    if kind == "pixel":
        edge = M.pixel_distance(p[0], p[1], *sc["kp_px"][0])
        sc["dmaxpxdist"] = edge if on_edge else np.nextafter(edge, f32(0))
        return sc, M.pixel_distance(p[0], p[1], *sc["kp_px"][0]) == edge, on_edge
    if kind == "coprojection":
        edge, nb = M.coprojection(sc, xyz, lm)
        sc["dmaxpxdist"] = edge if on_edge else np.nextafter(edge, f32(0))
        return sc, nb == 3 and M.pixel_distance(p[0], p[1], *sc["kp_px"][0]) == 0 and edge > 0, on_edge
    if kind == "no_observations":           # zero radius: nb == 0 is never dropped by the mean, one observation 0.5 px off is
        sc["dmaxpxdist"] = f32(0.0)
        nb_want = (None, 0) if on_edge else (f32(0.5), 1)
        return sc, M.coprojection(sc, xyz, lm) == nb_want and M.pixel_distance(p[0], p[1], *sc["kp_px"][0]) == 0, on_edge
    if kind == "depth":
        return sc, Z == 0.1 if on_edge else Z == np.nextafter(0.1, 0.0), on_edge
    if kind == "view_angle":
        edge = M.view_angle(X, Y, Z)
        sc["view_th"] = edge if on_edge else np.nextafter(edge, f32(np.inf))
        return sc, abs(M.view_angle(X, Y, Z)) == edge, on_edge
    if kind == "hamming":
        sc["fdistratio"] = f32(0.25)
        return sc, M.min_dist(0.25) == 64, on_edge
    if kind == "ratio":                                              # best 45 (46 one bit worse) against a second of 50
        sc["desc"] = sc["desc"].copy()
        sc["desc"][sc["mp_desc_ptr"][lm]] = flip(D, 45 if on_edge else 46)
        return sc, 0.9 * 50.0 == 45.0, on_edge
    if kind == "no_descriptor":                                      # computeMinDescDist returns 1000 for an empty side
        sc["fdistratio"] = f32(1000 / 256) if on_edge else np.nextafter(f32(1000 / 256), f32(0))
        return sc, M.min_dist(f32(1000 / 256)) == 1000 and (on_edge or M.min_dist(sc["fdistratio"]) < 1000), on_edge
    raise KeyError(kind)


THRESHOLDS = ("pixel", "coprojection", "no_observations", "depth", "view_angle", "hamming", "ratio", "no_descriptor")


# --------------------------------------------------------------------------------------------------- grid and image edges
def grid_edge_scene(geom, cs, distorted):
    """Candidates projecting onto cell boundaries, row and column 0, the last partial cell row and column, px == 0, the last
    float below the width / height, and the width / height itself, each with a keypoint at its projection (5 bits away) and
    one 1 px to the left and above (20 and 30 bits).  fmax_proj_pxdist 2 as shipped; no view-angle cull.  Returns the scene,
    and per candidate its target pixel and whether the projection is inside the image."""
    w, h, K = GEOMETRIES[geom]
    s = Scene(w, h, cs, K, EUROC_DIST if distorted else None, dmax=2.0, view_th=0.0)
    nbw, nbh = -(-w // cs), -(-h // cs)
    below = lambda n: np.nextafter(f32(n), f32(0))
    targets = [((cs, cs), (1, 1)), ((2 * cs, 3 * cs), (1, 1)), ((cs, 100.5), (1, 1)), ((100.5, cs), (1, 1)),
               ((10.5, 10.5), (1, 1)), ((0, 50.5), (1, 1)), ((50.5, 0), (1, 1)), ((0, 0), (1, 1)),
               (((nbw - 1) * cs, (nbh - 1) * cs), (1, 1)), (((nbw - 1) * cs + 1.5, (nbh - 1) * cs + 1.5), (1, 1)),
               ((below(w), 100.5), (0, 1)), ((100.5, below(h)), (1, 0)), ((below(w), below(h)), (0, 0)),
               ((w, 100.5), (1, 1)), ((100.5, h), (1, 1)), ((w, h), (1, 1))]
    out = []
    for (u, v), up in targets:
        xyz = s.point_at(u, v, z=2.0, up=tuple(bool(x) for x in up))
        p = s.project(xyz)
        D = s.random_desc()
        s.candidate(s.map_point(xyz, [D]))
        inside = bool(p[0] >= 0 and p[1] >= 0 and p[0] < w and p[1] < h)
        kp = (min(p[0], below(w)), min(p[1], below(h)))
        s.keypoint(kp, s.map_point(xyz, [flip(D, 5)]))
        if kp[0] >= 1:
            s.keypoint((kp[0] - f32(1), kp[1]), s.map_point(xyz, [flip(D, 20)]))
        if kp[1] >= 1:
            s.keypoint((kp[0], kp[1] - f32(1)), s.map_point(xyz, [flip(D, 30)]))
        out.append(((f32(u), f32(v)), p, inside))
    return s.scene(), out


# -------------------------------------------------------------------------------------------------------- descriptor sets
def descriptor_set_scene(sizes=(1, 7, 16)):
    """A candidate / keypoint pair for every combination of descriptor counts; the minimum (6 bits) on the last pair, and 8
    bits on the first pair where the keypoint's map point has more than one descriptor."""
    s = Scene()
    want = []
    for i, (na, nb) in enumerate((a, b) for a in sizes for b in sizes):
        xyz = s.point_at(30.5 + 70 * (i % 10), 60.5 + 90 * (i // 10), z=4.0)
        A = [s.random_desc() for _ in range(na)]
        B = [s.random_desc() for _ in range(nb)]
        B[-1] = flip(A[-1], 6)
        if nb > 1:
            B[0] = flip(A[0], 8, start=50)
        s.candidate(s.map_point(xyz, A))
        s.keypoint(s.project(xyz), s.map_point(xyz, B))
        want.append(6.0)
    return s.scene(), want


# ---------------------------------------------------------------------------------------------------- per-keypoint pass
def keypoint_pass_scene(seed=0):
    """Three keypoints, each the best of 40 or more candidates, candidate order shuffled: equal distances (the highest index
    wins), a strictly smaller distance (it stays), and candidates without descriptor at 1000 (fdistratio 1000 / 256)."""
    s = Scene(ratio=1000 / 256, seed=seed)
    groups = []
    for g, (u, v) in enumerate(((100.5, 100.5), (300.5, 200.5), (500.5, 300.5))):
        xyz = s.point_at(u, v, z=3.0)
        D = s.random_desc()
        kp = s.keypoint(s.project(xyz), s.map_point(xyz, [D]))
        n = 40 if g != 1 else 41
        for i in range(n):
            if g == 0:
                descs = [flip(D, 9, start=i)]
            elif g == 1:
                descs = [flip(D, 4 if i == 7 else 9, start=i)]
            else:
                descs = []
            groups.append((kp, s.map_point(xyz, descs)))
    order = s.rng.permutation(len(groups))
    for k in order:
        s.candidate(groups[k][1])
    return s.scene(), [groups[k][0] for k in order]
