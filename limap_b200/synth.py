"""Seeded synthetic scenes of the shapes in BASELINE.json `configs` (SURVEY.md §8d).

Scene box [-5,5]^3 * scale with G ground-truth 3D segments, cameras on a radius-12*scale band looking
at the origin (SIMPLE_PINHOLE f=692.82, cx=400, cy=300, 800x600 -- Hypersim after max_image_dim 800),
per view L segments = projections of visible GT lines with N(0, noise_px) endpoint noise, random
truncation and random start/end flips, padded with clutter; neighbours = N nearest cameras; matches
per (line, neighbour) = the true correspondent (when visible) + nearest-midpoint decoys, K per line
(mimics the top-k NN matcher, src/limap/line2d/endpoints/matcher.py:71-112).
No dataset or network access is needed; everything derives from the seed.
"""
from dataclasses import dataclass, field

import numpy as np


@dataclass
class Scene:
    img_ids: np.ndarray        # [V] int32, ascending
    model_ids: np.ndarray      # [V] int32 (0 SIMPLE_PINHOLE)
    kvec: np.ndarray           # [V,4] fx,fy,cx,cy
    qvec: np.ndarray           # [V,4] wxyz
    tvec: np.ndarray           # [V,3]
    line_off: np.ndarray       # [V+1] int64
    segs: np.ndarray           # [sum L,4] float64
    gt_id: np.ndarray          # [sum L] int32 GT line of each segment (-1 clutter)
    neighbors: dict            # img_id -> list of img ids
    matches: dict              # img_id -> {ng_img_id: (M,2) int32}
    ranges: tuple              # (lo[3], hi[3])
    gt_lines: np.ndarray = field(default=None)  # [G,6]
    meta: dict = field(default_factory=dict)

    @property
    def n_views(self):
        return len(self.img_ids)

    def n_rows(self, img_ids=None):
        """Match rows (the M1 unit) of the given source images (default: all that have matches)."""
        ids = self.matches.keys() if img_ids is None else img_ids
        return int(sum(len(m) for i in ids for m in self.matches[i].values()))

    def lines_of(self, view):
        return self.segs[self.line_off[view]:self.line_off[view + 1]]

    def bulk_matches(self, img_ids=None):
        """(src_ids[b], ng_ids[b], row_off[b+1], pairs[rows,2]) over all (image, neighbour) blocks."""
        ids = sorted(self.matches.keys()) if img_ids is None else list(img_ids)
        src, ng, off, parts = [], [], [0], []
        for i in ids:
            for g in sorted(self.matches[i].keys()):
                m = self.matches[i][g]
                src.append(i)
                ng.append(g)
                off.append(off[-1] + len(m))
                parts.append(m)
        pairs = np.concatenate(parts, 0) if parts else np.zeros((0, 2), np.int32)
        return (np.asarray(src, np.int32), np.asarray(ng, np.int32), np.asarray(off, np.int64),
                np.ascontiguousarray(pairs, dtype=np.int32))

    def flat_matches(self, img_id):
        """(ng_ids[n], row_off[n+1], pairs[rows,2]) of one image, neighbours ascending (std::map order)."""
        m = self.matches[img_id]
        ngs = sorted(m.keys())
        row_off = np.zeros(len(ngs) + 1, np.int64)
        for i, g in enumerate(ngs):
            row_off[i + 1] = row_off[i] + len(m[g])
        pairs = (np.concatenate([m[g] for g in ngs], axis=0) if ngs else np.zeros((0, 2), np.int32))
        return np.asarray(ngs, np.int32), row_off, np.ascontiguousarray(pairs, dtype=np.int32)


def _rot_to_quat(R):
    """Eigen-style (Shepperd) rotation matrix -> quaternion wxyz."""
    t = np.trace(R)
    if t > 0:
        s = np.sqrt(t + 1.0)
        w = 0.5 * s
        s = 0.5 / s
        return np.array([w, (R[2, 1] - R[1, 2]) * s, (R[0, 2] - R[2, 0]) * s, (R[1, 0] - R[0, 1]) * s])
    i = int(np.argmax(np.diag(R)))
    j, k = (i + 1) % 3, (i + 2) % 3
    s = np.sqrt(R[i, i] - R[j, j] - R[k, k] + 1.0)
    q = np.zeros(4)
    q[1 + i] = 0.5 * s
    s = 0.5 / s
    q[0] = (R[k, j] - R[j, k]) * s
    q[1 + j] = (R[j, i] + R[i, j]) * s
    q[1 + k] = (R[k, i] + R[i, k]) * s
    return q


def make_scene(V=10, L=100, N=5, K=4, seed=1234, scale=1.0, noise_px=0.5, G=None, id_stride=1,
               width=800, height=600, focal=692.82, shuffle_rows=False, match_views=None, camera_mix=False):
    rng = np.random.default_rng(seed)
    G = int(L * 1.3) if G is None else G
    # ground-truth 3D segments
    mid = rng.uniform(-5, 5, (G, 3))
    d = rng.normal(size=(G, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    half = rng.uniform(0.25, 1.5, (G, 1))
    P0 = np.clip(mid - d * half, -5, 5) * scale
    P1 = np.clip(mid + d * half, -5, 5) * scale
    gt_lines = np.concatenate([P0, P1], axis=1)
    # cameras on a band of a sphere looking at the origin
    az = rng.uniform(0, 2 * np.pi, V)
    el = rng.uniform(-0.5, 0.5, V)
    rad = 12.0 * scale * rng.uniform(0.95, 1.05, V)
    Cs = np.stack([rad * np.cos(el) * np.cos(az), rad * np.cos(el) * np.sin(az), rad * np.sin(el)], 1)
    kvec = np.tile(np.array([focal, focal, width / 2.0, height / 2.0]), (V, 1))
    model_ids = np.zeros(V, np.int32)
    if camera_mix:
        # one camera per view: odd views PINHOLE with fx != fy, even views SIMPLE_PINHOLE, principal points off-centre
        crng = np.random.default_rng(seed + 7919)
        fx = focal * crng.uniform(0.85, 1.15, V)
        fy = np.where(np.arange(V) % 2 == 1, fx * crng.uniform(0.9, 1.1, V), fx)
        kvec = np.stack([fx, fy, width / 2.0 + crng.uniform(-20, 20, V), height / 2.0 + crng.uniform(-20, 20, V)], 1)
        model_ids = (np.arange(V) % 2).astype(np.int32)
    qvec = np.zeros((V, 4))
    tvec = np.zeros((V, 3))
    Rs = np.zeros((V, 3, 3))
    for v in range(V):
        z = -Cs[v] / np.linalg.norm(Cs[v])
        up = np.array([0.0, 0.0, 1.0]) + rng.normal(scale=0.05, size=3)
        x = np.cross(z, up)
        x /= np.linalg.norm(x)
        y = np.cross(z, x)
        R = np.stack([x, y, z], 0)
        Rs[v] = R
        qvec[v] = _rot_to_quat(R)
        tvec[v] = -R @ Cs[v]
    img_ids = (np.arange(V) * id_stride + (3 if id_stride > 1 else 0)).astype(np.int32)

    segs_all, gt_all, line_off = [], [], [0]
    line_of_gt = -np.ones((V, G), np.int64)
    for v in range(V):
        R, t = Rs[v], tvec[v]
        Xc0 = P0 @ R.T + t
        Xc1 = P1 @ R.T + t
        ok = (Xc0[:, 2] > 0.5 * scale) & (Xc1[:, 2] > 0.5 * scale)
        p0 = Xc0[:, :2] / Xc0[:, 2:3] * kvec[v, 0:2] + kvec[v, 2:4]
        p1 = Xc1[:, :2] / Xc1[:, 2:3] * kvec[v, 0:2] + kvec[v, 2:4]
        inside = lambda p: (p[:, 0] >= 0) & (p[:, 0] <= width) & (p[:, 1] >= 0) & (p[:, 1] <= height)
        ok &= inside(p0) & inside(p1) & (np.linalg.norm(p1 - p0, axis=1) > 8.0)
        vis = np.flatnonzero(ok)
        rng.shuffle(vis)
        vis = vis[:L]
        a, b = p0[vis].copy(), p1[vis].copy()
        # random truncation along the line, noise, random flips
        ta = rng.uniform(0.0, 0.2, (len(vis), 1))
        tb = rng.uniform(0.0, 0.2, (len(vis), 1))
        a2 = a + (b - a) * ta
        b2 = b - (b - a) * tb
        a2 += rng.normal(scale=noise_px, size=a2.shape)
        b2 += rng.normal(scale=noise_px, size=b2.shape)
        flip = rng.random(len(vis)) < 0.5
        s = np.where(flip[:, None], b2, a2)
        e = np.where(flip[:, None], a2, b2)
        seg = np.concatenate([s, e], 1)
        gt = vis.astype(np.int32)
        n_clutter = L - len(vis)
        if n_clutter > 0:
            c0 = rng.uniform([0, 0], [width, height], (n_clutter, 2))
            ang = rng.uniform(0, np.pi, n_clutter)
            ln = rng.uniform(10, 120, n_clutter)
            c1 = c0 + np.stack([np.cos(ang), np.sin(ang)], 1) * ln[:, None]
            seg = np.concatenate([seg, np.concatenate([c0, c1], 1)], 0)
            gt = np.concatenate([gt, -np.ones(n_clutter, np.int32)])
        perm = rng.permutation(len(seg))
        seg, gt = seg[perm], gt[perm]
        line_of_gt[v, gt[gt >= 0]] = np.flatnonzero(gt >= 0)
        segs_all.append(seg)
        gt_all.append(gt)
        line_off.append(line_off[-1] + len(seg))
    segs = np.ascontiguousarray(np.concatenate(segs_all, 0), dtype=np.float64)
    gt_id = np.concatenate(gt_all)
    line_off = np.asarray(line_off, np.int64)

    # neighbours: N nearest camera centres
    Nn = min(N, V - 1)
    if V <= 4096:
        D = np.linalg.norm(Cs[:, None, :] - Cs[None, :, :], axis=2)
        np.fill_diagonal(D, np.inf)
        nb_idx = np.argsort(D, axis=1)[:, :Nn]
    else:  # Rome16K-sized scenes: no V x V distance matrix
        from scipy.spatial import cKDTree as _Tree
        _, nn_c = _Tree(Cs).query(Cs, k=Nn + 1)
        nb_idx = np.stack([row[row != v][:Nn] for v, row in enumerate(nn_c)])
    neighbors = {int(img_ids[v]): [int(img_ids[u]) for u in nb_idx[v]] for v in range(V)}

    # matches with decoys
    from scipy.spatial import cKDTree
    mids = [(s[:, :2] + s[:, 2:]) * 0.5 for s in segs_all]
    need_tree = set(range(V)) if match_views is None else {int(u) for v in match_views for u in nb_idx[v]}
    trees = [cKDTree(m) if v in need_tree else None for v, m in enumerate(mids)]
    matches = {}
    for v in (range(V) if match_views is None else match_views):
        mv = {}
        Lv = len(segs_all[v])
        for u in nb_idx[v]:
            Lu = len(segs_all[u])
            kk = min(K, Lu)
            g = gt_all[v]
            tgt = np.where(g >= 0, line_of_gt[u, np.maximum(g, 0)], -1)
            qpts = np.where((tgt >= 0)[:, None], mids[u][np.maximum(tgt, 0)], mids[v])
            _, nn = trees[u].query(qpts, k=kk)
            nn = nn.reshape(Lv, kk)
            # make sure the true correspondent is the first candidate when it exists
            has = tgt >= 0
            nn[has, 0] = tgt[has]
            rows = np.stack([np.repeat(np.arange(Lv), kk), nn.reshape(-1)], 1).astype(np.int32)
            if shuffle_rows:
                rows = rows[rng.permutation(len(rows))]
            mv[int(img_ids[u])] = np.ascontiguousarray(rows)
        matches[int(img_ids[v])] = mv
    lo = np.array([-5.0, -5.0, -5.0]) * scale * 1.25
    hi = np.array([5.0, 5.0, 5.0]) * scale * 1.25
    return Scene(img_ids=img_ids, model_ids=model_ids, kvec=np.ascontiguousarray(kvec),
                 qvec=np.ascontiguousarray(qvec), tvec=np.ascontiguousarray(tvec), line_off=line_off,
                 segs=segs, gt_id=gt_id, neighbors=neighbors, matches=matches, ranges=(lo, hi),
                 gt_lines=gt_lines, meta=dict(V=V, L=L, N=N, K=K, seed=seed, scale=scale,
                                              noise_px=noise_px))


def concat_scenes(scenes):
    """One scene out of several independent blocks: views, lines and matches of block b keep their content and get
    image ids offset by the views of the blocks before it (neighbours stay inside a block). Used for equal-work weak
    scaling: N blocks of the same shape = N times the work of one block, one block per GPU."""
    img_ids, model_ids, kvec, qvec, tvec, segs, gt_id, line_off = [], [], [], [], [], [], [], [0]
    neighbors, matches = {}, {}
    lo, hi = np.full(3, np.inf), np.full(3, -np.inf)
    id0 = 0
    for sc in scenes:
        ids = sc.img_ids.astype(np.int64) + id0
        img_ids.append(ids.astype(np.int32))
        model_ids.append(sc.model_ids); kvec.append(sc.kvec); qvec.append(sc.qvec); tvec.append(sc.tvec)
        segs.append(sc.segs); gt_id.append(sc.gt_id)
        line_off.extend((sc.line_off[1:] + line_off[-1]).tolist())
        for i, nb in sc.neighbors.items():
            neighbors[int(i) + id0] = [int(j) + id0 for j in nb]
        for i, m in sc.matches.items():
            matches[int(i) + id0] = {int(g) + id0: v for g, v in m.items()}
        lo, hi = np.minimum(lo, sc.ranges[0]), np.maximum(hi, sc.ranges[1])
        id0 = int(ids[-1]) + 1
    return Scene(img_ids=np.concatenate(img_ids), model_ids=np.concatenate(model_ids),
                 kvec=np.ascontiguousarray(np.concatenate(kvec)), qvec=np.ascontiguousarray(np.concatenate(qvec)),
                 tvec=np.ascontiguousarray(np.concatenate(tvec)), line_off=np.asarray(line_off, np.int64),
                 segs=np.ascontiguousarray(np.concatenate(segs)), gt_id=np.concatenate(gt_id), neighbors=neighbors,
                 matches=matches, ranges=(lo, hi), gt_lines=None,
                 meta=dict(blocks=[sc.meta for sc in scenes]))


# BASELINE.json `configs` -> generator arguments (SURVEY.md §8d)
CONFIGS = {
    "hypersim10": dict(V=10, L=800, N=9, K=10, seed=1234),              # configs[0] stand-in
    "hypersim100": dict(V=100, L=1000, N=20, K=10, seed=1235),          # configs[1] (the metric's config)
    "sweep500": dict(V=500, L=400, N=40, K=10, seed=1236),              # configs[2]
    "rome16k": dict(V=15000, L=300, N=20, K=10, seed=1238),             # configs[4] (generate with match_views=<shard>)
}


@dataclass
class FitScene:
    """Per-image 3D fits of every 2D segment of a Scene (the input of merging.merging, merging.py:6-21): lines3d[n,2,3]
    in the scene's flat segment order, zeros where the fit failed; neighbours as ng_ids[ng_off[v] .. ng_off[v+1])."""
    img_ids: np.ndarray
    model_ids: np.ndarray
    kvec: np.ndarray
    qvec: np.ndarray
    tvec: np.ndarray
    line_off: np.ndarray
    segs: np.ndarray
    lines3d: np.ndarray
    neighbors: dict
    ng_off: np.ndarray = None
    ng_ids: np.ndarray = None

    def __post_init__(self):
        self.set_neighbors(self.neighbors)

    def set_neighbors(self, neighbors):
        self.neighbors = {int(k): [int(x) for x in v] for k, v in neighbors.items()}
        lists = [self.neighbors.get(int(i), []) for i in self.img_ids]
        self.ng_off = np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(np.int64)
        self.ng_ids = np.asarray([x for lst in lists for x in lst], np.int32)

    def segs_of(self, view):
        return self.segs[self.line_off[view]:self.line_off[view + 1]]

    def fits_of(self, view):
        return self.lines3d[self.line_off[view]:self.line_off[view + 1]]


def make_fits(scene, depth_noise=1e-3, fail_frac=0.1, seed=0, degenerate_frac=0.01):
    """What line fitting from depth (runners/line_fitnmerge.py:30-56) would give on `scene`: each endpoint of a segment
    of a GT line is back-projected onto that line (the point of the line closest to the endpoint's ray), then moved along
    the ray by a relative depth error N(0, depth_noise). Clutter and a `fail_frac` share of the segments get zero fits
    (failed fits, line_fitnmerge.py:52-55); a `degenerate_frac` share gets start == end != 0."""
    from .base import _quat_to_R
    rng = np.random.default_rng(seed)
    n = len(scene.segs)
    lines3d = np.zeros((n, 2, 3))
    for v in range(len(scene.img_ids)):
        R = _quat_to_R(scene.qvec[v])
        t = scene.tvec[v]
        C = -R.T @ t
        fx, fy, cx, cy = scene.kvec[v]
        if scene.model_ids[v] == 0:
            fy = fx
        for g in range(int(scene.line_off[v]), int(scene.line_off[v + 1])):
            gid = int(scene.gt_id[g])
            if gid < 0:
                continue
            P0, P1 = scene.gt_lines[gid, :3], scene.gt_lines[gid, 3:]
            u = (P1 - P0) / np.linalg.norm(P1 - P0)
            for k in range(2):
                x, y = scene.segs[g, 2 * k:2 * k + 2]
                r = R.T @ np.array([(x - cx) / fx, (y - cy) / fy, 1.0])
                r /= np.linalg.norm(r)
                # closest points of the ray C + s r and the line P0 + w u
                w0 = C - P0
                b, d, e = r @ u, r @ w0, u @ w0
                den = 1.0 - b * b
                s = (b * e - d) / den if den > 1e-12 else -d
                lines3d[g, k] = C + r * s * (1.0 + depth_noise * rng.normal())
    fail = rng.random(n) < fail_frac
    lines3d[fail] = 0.0
    nz = np.flatnonzero(np.abs(lines3d).sum(axis=(1, 2)) > 0)
    degen = nz[rng.random(len(nz)) < degenerate_frac]
    lines3d[degen, 1] = lines3d[degen, 0]
    return FitScene(img_ids=scene.img_ids.copy(), model_ids=scene.model_ids.copy(), kvec=scene.kvec.copy(),
                    qvec=scene.qvec.copy(), tvec=scene.tvec.copy(), line_off=scene.line_off.copy(),
                    segs=scene.segs.copy(), lines3d=lines3d, neighbors=dict(scene.neighbors))


@dataclass
class TrackSet:
    """Flat line tracks for the refinement path (BASELINE.json configs[3]): sup_off[T+1]; per support:
    2D segment, camera (kvec,qvec,tvec), image id and the per-node 3D line (track.line3d_list)."""
    sup_off: np.ndarray
    segs: np.ndarray      # [n,4]
    kvec: np.ndarray      # [n,4]
    qvec: np.ndarray      # [n,4]
    tvec: np.ndarray      # [n,3]
    img_ids: np.ndarray   # [n] int32
    line3d: np.ndarray    # [n,6]
    line_init: np.ndarray  # [T,6]
    gt: np.ndarray        # [T,6]

    @property
    def n_tracks(self):
        return len(self.sup_off) - 1


def make_tracks(T=100, S=30, V=300, seed=1237, noise_px=0.5, perturb=0.05, scale=1.0, width=800,
                height=600, focal=692.82):
    """T ground-truth 3D segments, each observed in S of V ring cameras (one 2D segment per view, noisy
    endpoints, random truncation); the start line is the GT perturbed by N(0, perturb) on its endpoints
    (cf. src/limap/optimize/functions.py:6-13); line3d_list = noisy copies of the GT segment."""
    rng = np.random.default_rng(seed)
    az = rng.uniform(0, 2 * np.pi, V)
    el = rng.uniform(-0.5, 0.5, V)
    rad = 12.0 * scale * rng.uniform(0.95, 1.05, V)
    Cs = np.stack([rad * np.cos(el) * np.cos(az), rad * np.cos(el) * np.sin(az), rad * np.sin(el)], 1)
    Rs, qs, ts = np.zeros((V, 3, 3)), np.zeros((V, 4)), np.zeros((V, 3))
    for v in range(V):
        z = -Cs[v] / np.linalg.norm(Cs[v])
        x = np.cross(z, np.array([0.0, 0.0, 1.0]) + rng.normal(scale=0.05, size=3))
        x /= np.linalg.norm(x)
        R = np.stack([x, np.cross(z, x), z], 0)
        Rs[v], qs[v], ts[v] = R, _rot_to_quat(R), -R @ Cs[v]
    mid = rng.uniform(-4, 4, (T, 3))
    d = rng.normal(size=(T, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    half = rng.uniform(0.25, 1.5, (T, 1))
    gt = np.concatenate([(mid - d * half), (mid + d * half)], 1) * scale
    K = np.array([focal, focal, width / 2.0, height / 2.0])
    sup_off = np.arange(T + 1, dtype=np.int64) * S
    n = T * S
    views = np.stack([rng.choice(V, S, replace=False) for _ in range(T)]).reshape(-1)
    R = Rs[views]
    t = ts[views]
    P0 = np.repeat(gt[:, :3], S, 0)
    P1 = np.repeat(gt[:, 3:], S, 0)
    ta = rng.uniform(0.0, 0.2, (n, 1))
    tb = rng.uniform(0.0, 0.2, (n, 1))
    A = P0 + (P1 - P0) * ta
    B = P1 - (P1 - P0) * tb
    def proj(X):
        Xc = np.einsum("nij,nj->ni", R, X) + t
        return Xc[:, :2] / Xc[:, 2:3] * focal + K[2:4]
    a = proj(A) + rng.normal(scale=noise_px, size=(n, 2))
    b = proj(B) + rng.normal(scale=noise_px, size=(n, 2))
    flip = rng.random(n) < 0.5
    segs = np.where(flip[:, None], np.concatenate([b, a], 1), np.concatenate([a, b], 1))
    line3d = np.concatenate([A, B], 1) + rng.normal(scale=0.02 * scale, size=(n, 6))
    line_init = gt + rng.normal(scale=perturb * scale, size=gt.shape)
    return TrackSet(sup_off=sup_off, segs=np.ascontiguousarray(segs), kvec=np.tile(K, (n, 1)),
                    qvec=np.ascontiguousarray(qs[views]), tvec=np.ascontiguousarray(ts[views]),
                    img_ids=views.astype(np.int32), line3d=np.ascontiguousarray(line3d),
                    line_init=np.ascontiguousarray(line_init), gt=gt)


def make_track_lines(T, dup_frac=0.3, seed=0, extent=20.0, unc=0.05, noise=0.002):
    """Track lines for the remerge pair test: T unit-scale 3D segments (start3, end3, uncertainty) in a cube,
    a `dup_frac` share of them noisy, partly shifted copies of other tracks (the fragments remerging joins)."""
    rng = np.random.default_rng(seed)
    n_base = max(1, int(round(T * (1.0 - dup_frac))))
    c = rng.uniform(-extent, extent, (n_base, 3))
    d = rng.normal(size=(n_base, 3))
    d /= np.linalg.norm(d, axis=1)[:, None]
    half = rng.uniform(0.5, 1.5, (n_base, 1))
    L = np.concatenate([c - d * half, c + d * half, np.full((n_base, 1), unc)], 1)
    n_dup = T - n_base
    if n_dup > 0:
        src = rng.integers(0, n_base, n_dup)
        shift = rng.uniform(-0.8, 0.8, (n_dup, 1)) * half[src]
        D = L[src].copy()
        D[:, :3] += d[src] * shift + rng.normal(scale=noise, size=(n_dup, 3))
        D[:, 3:6] += d[src] * shift + rng.normal(scale=noise, size=(n_dup, 3))
        D[:, 6] = unc * rng.uniform(0.5, 2.0, n_dup)
        L = np.concatenate([L, D])
    return np.ascontiguousarray(L[rng.permutation(T)])


def make_vp_images(n_images, n_segments=300, seed=0, width=800, height=600, noise=0.3, clutter_frac=0.15):
    """Images of 2D segments with three dominant vanishing points (two far ones, one near the image centre) plus
    clutter -- the Manhattan-like structure J-Linkage is run on (vplib/JLinkage/JLinkage.cc:14-127). Every segment
    is at least 45 px long, so all pass the detector's min_length of 40. Returns a list of [n_segments, 4] arrays."""
    rng = np.random.default_rng(seed)
    out = []
    n_cl = int(round(n_segments * clutter_frac))
    base = n_segments - n_cl
    counts = [base - 2 * (base // 3), base // 3, base // 3]
    for _ in range(n_images):
        vps = [np.array([rng.uniform(1500, 4000) * rng.choice([-1, 1]), rng.uniform(200, 400), 1.0]),
               np.array([rng.uniform(300, 500), rng.uniform(2500, 5000) * rng.choice([-1, 1]), 1.0]),
               np.array([rng.uniform(350, 450), rng.uniform(250, 350), 1.0])]
        segs = []
        for vp, n in zip(vps, counts):
            p = rng.uniform([0, 0], [width, height], (n, 2))
            d = vp[:2] / vp[2] - p
            d /= np.linalg.norm(d, axis=1, keepdims=True)
            L = rng.uniform(45, 160, (n, 1))
            segs.append(np.concatenate([p + rng.normal(scale=noise, size=(n, 2)),
                                        p + d * L + rng.normal(scale=noise, size=(n, 2))], 1))
        a = rng.uniform([0, 0], [width, height], (n_cl, 2))
        ang = rng.uniform(0, np.pi, n_cl)
        ln = rng.uniform(45, 150, (n_cl, 1))
        segs.append(np.concatenate([a, a + ln * np.stack([np.cos(ang), np.sin(ang)], 1)], 1))
        segs = np.concatenate(segs, 0)
        out.append(np.ascontiguousarray(segs[rng.permutation(len(segs))]))
    return out


def make_sfm_points(scene, n_points=2000, seed=0, p_detect=0.7, max_track=None):
    """A sparse point model for a Scene: random 3D points in the scene box, each tracked by the views that see it
    (inside the image, in front of the camera) and 'detect' it with probability p_detect. Returns (centres[V,3],
    xyz[P,3], track_off[P+1], track_img[...]) with image INDICES (view order), points with fewer than 2 views dropped."""
    rng = np.random.default_rng(seed)
    V = scene.n_views
    s = float(scene.meta.get("scale", 1.0)) if isinstance(scene.meta, dict) else 1.0
    X = rng.uniform(-5, 5, (n_points, 3)) * s
    from .base import CameraPose
    Rs = np.stack([CameraPose(scene.qvec[v], scene.tvec[v]).R() for v in range(V)])
    centres = np.stack([-Rs[v].T @ scene.tvec[v] for v in range(V)])
    off, img, keep = [0], [], []
    for p in range(n_points):
        Xc = np.einsum("vij,j->vi", Rs, X[p]) + scene.tvec
        z = Xc[:, 2]
        u = Xc[:, 0] / z * scene.kvec[:, 0] + scene.kvec[:, 2]
        w = Xc[:, 1] / z * scene.kvec[:, 1] + scene.kvec[:, 3]
        vis = (z > 0.5 * s) & (u >= 0) & (u <= 800) & (w >= 0) & (w <= 600) & (rng.random(V) < p_detect)
        t = np.flatnonzero(vis)
        if max_track is not None and len(t) > max_track:
            t = np.sort(rng.choice(t, max_track, replace=False))
        if len(t) < 2:
            continue
        keep.append(p)
        img.append(t.astype(np.int32))
        off.append(off[-1] + len(t))
    return (np.ascontiguousarray(centres), np.ascontiguousarray(X[keep]), np.asarray(off, np.int64),
            np.ascontiguousarray(np.concatenate(img) if img else np.zeros(0, np.int32)))
