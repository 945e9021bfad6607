"""J-Linkage VP detection (jlinkage_kernel + lm_vp_detect_indexed) at its batch, size, model-count, threshold and tie
edges, against the CPU oracle (oracle.oracle.detect_vps): labels bit-identical, VPs equal up to sign within 1e-9.

The consensus decision `d < th` is planted at d == th and one ulp either side of it by a float32 numpy restatement of
the kernel's arithmetic (every operation rounded, none fused), which is itself checked against the oracle without a
GPU. The host post-processing (length filter, cluster-size and perpendicular-support filters, renumbering, VP fit,
vp_cap retry) is driven at its equalities with exactly representable geometry."""
import ctypes as C

import numpy as np
import pytest

F = np.float32
MASK64 = (1 << 64) - 1
# jlinkage_kernel's static shared memory (s_best[8] and s_pick: 9 x 16 bytes; ptxas -v for sm_90a: 144 bytes smem).
# If the shared-memory edge tests below fail, first check that the compiler still gives the kernel 144 static bytes.
STATIC_SMEM = 144
BENCH_CFG = dict(min_num_supports=10, min_length=40.0, inlier_threshold=1.0)


# ---- float32 restatement of the kernel's hypothesis and consensus arithmetic (vp_kernels.cu) --------------------

def splitmix64(seed, counter):
    z = (seed + 0x9E3779B97F4A7C15 * (counter + 1)) & MASK64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & MASK64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & MASK64
    return z ^ (z >> 31)


def hypothesis_pair(seed, image_index, m, n, n_models):
    """The two valid segments that model m of an image with n valid segments is drawn from."""
    z = splitmix64(seed, image_index * n_models + m)
    i = (z & 0xFFFFFFFF) % n
    j = (z >> 32) % (n - 1)
    return i, j + (j >= i)


def line_coords(p):
    x1, y1, x2, y2 = (F(v) for v in p)
    return (y1 - y2, x2 - x1, x1 * y2 - x2 * y1)


def cross(a, b):
    return (a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0])


def model_vp(pi, pj):
    v = cross(line_coords(pi), line_coords(pj))
    nr = np.sqrt((v[0] * v[0] + v[1] * v[1]) + v[2] * v[2])
    return tuple(c / nr for c in v) if nr > F(0) else v


def consensus_d(x1, y1, x2, y2, vp):
    """Tardif's distance of endpoint 1 to the line through the midpoint and the VP; scalars or float32 arrays."""
    x1, y1, x2, y2 = (np.asarray(v, F) for v in (x1, y1, x2, y2))
    m = ((x1 + x2) * F(0.5), (y1 + y2) * F(0.5), np.ones_like(x1))
    lx, ly, lz = cross(m, tuple(F(c) for c in vp))
    den = np.sqrt(lx * lx + ly * ly)
    num = np.abs((lx * x1 + ly * y1) + lz)
    with np.errstate(invalid="ignore", divide="ignore"):
        return num / den


# ---- helpers ---------------------------------------------------------------------------------------------------

def _off(imgs):
    return np.concatenate([[0], np.cumsum([len(s) for s in imgs])]).astype(np.int64)


def _flat(imgs):
    return np.ascontiguousarray(np.concatenate(imgs, 0) if len(imgs) else np.zeros((0, 4)), np.float64)


def oracle_results(imgs, image_index=None, **cfg):
    """[(labels, vps)] per image from the CPU oracle."""
    from oracle import oracle as orc
    off = _off(imgs)
    lab, vp_off, vps = orc.detect_vps(off, _flat(imgs), image_index=image_index, **cfg)
    return [(lab[off[i]:off[i + 1]], vps[vp_off[i]:vp_off[i + 1]]) for i in range(len(imgs))]


def _detector(n_models=5000, seed=7, min_num_supports=5, min_length=40.0, inlier_threshold=1.0):
    from limap_b200.vplib import JLinkageDetector
    return JLinkageDetector(dict(min_num_supports=min_num_supports, min_length=min_length,
                                 inlier_threshold=inlier_threshold), seed=seed, n_models=n_models)


def gpu_results(imgs, image_index=None, n_models=5000, seed=7, **cfg):
    res = _detector(n_models, seed, **cfg).detect_batch(imgs, image_index=image_index)
    return [(np.asarray(r.labels, np.int32), np.asarray(r.vps, np.float64).reshape(-1, 3)) for r in res]


def assert_same(got, want, what=""):
    assert len(got) == len(want)
    for k, ((gl, gv), (ol, ov)) in enumerate(zip(got, want)):
        assert np.array_equal(gl, ol), f"{what}: labels differ in image {k}"
        assert gv.shape == ov.shape, f"{what}: VP count differs in image {k}"
        for a, b in zip(gv, ov):
            assert min(np.abs(a - b).max(), np.abs(a + b).max()) < 1e-9, f"{what}: VP differs in image {k}"


def check_against_oracle(imgs, image_index=None, n_models=5000, seed=7, **cfg):
    want = oracle_results(imgs, image_index=image_index, n_models=n_models, seed=seed, **cfg)
    got = gpu_results(imgs, image_index=image_index, n_models=n_models, seed=seed, **cfg)
    assert_same(got, want, f"n_models={n_models} cfg={cfg}")
    return want


def _image(n, seed, clutter_frac=0.15):
    from limap_b200.synth import make_vp_images
    return make_vp_images(1, n, seed=seed, clutter_frac=clutter_frac)[0] if n > 0 else np.zeros((0, 4))


def _shrink(segs, length):
    """Same segments cut to `length` px from their first endpoint."""
    d = segs[:, 2:] - segs[:, :2]
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    return np.concatenate([segs[:, :2], segs[:, :2] + length * d], 1)


# ---- 1. batch shape: persistent CTAs over ~700 images, slab reuse, reversed order, single-image calls -------------

def _vp_grid():
    """CTAs of one jlinkage_kernel launch with many images: 2 per SM (264 on an H100 SXM). CTA c runs images c,
    c + grid, c + 2 grid, ..."""
    import torch
    return 2 * torch.cuda.get_device_properties(0).multi_processor_count


def _batch_scene(grid):
    """~700 images (more than `grid` CTAs, so every CTA runs two or three images) of sizes 0, 5, min_lines - 1,
    min_lines, min_lines + 1, 31, 32, 33, 40-150 and 255-257 (one CTA of 256 threads and one thread past it) valid
    segments (min_lines = 20 for min_num_supports = 10), plus images whose segments are all shorter than min_length
    and images whose short segments leave 19 or 20 valid."""
    assert 44 + grid < 700
    rng = np.random.default_rng(2024)
    edge = [0, 5, 19, 20, 21, 31, 32, 33]
    imgs = []
    for k in range(700):
        kind = k % 7
        if kind < 3:
            imgs.append(_image(edge[rng.integers(len(edge))], 1000 + k))
        elif kind == 3:
            imgs.append(_shrink(_image(int(rng.integers(20, 80)), 1000 + k), 39.5))  # nothing valid
        elif kind == 4:  # 19 or 20 valid segments among short ones
            img = np.concatenate([_image(19 + k % 2, 1000 + k), _shrink(_image(15, 5000 + k), 30.0)])
            imgs.append(img[rng.permutation(len(img))])
        else:
            imgs.append(_image(int(rng.integers(40, 151)), 1000 + k))
    # a large image followed, on the same CTA, by a small one and the other way round
    for k in range(0, 40, 4):
        imgs[k], imgs[k + grid] = _image(150, 9000 + k), _image(20, 9100 + k)
        imgs[k + 1], imgs[k + 1 + grid] = _image(21, 9200 + k), _image(150, 9300 + k)
    for k, n in zip((40, 41, 42), (255, 256, 257)):
        imgs[k], imgs[k + grid] = _image(n, 9400 + k), _image(33, 9500 + k)
    return imgs


@pytest.mark.gpu
def test_batch_of_700_images_reversed_and_single_calls():
    grid = _vp_grid()
    imgs = _batch_scene(grid)
    want = oracle_results(imgs, seed=7, n_models=5000, **BENCH_CFG)
    got = gpu_results(imgs, seed=7, **BENCH_CFG)
    assert_same(got, want, "700-image batch")
    assert sum(len(v) for _, v in want) > 100 and sum(len(v) == 0 for _, v in want) > 100
    # reversed order, same image indices: other CTAs, other slab contents before each image
    n = len(imgs)
    rev = gpu_results(imgs[::-1], image_index=np.arange(n)[::-1], seed=7, **BENCH_CFG)
    assert_same(rev[::-1], got, "reversed batch")
    for k in (0, 1, grid - 1, grid, grid + 1, 41, 500, n - 1):
        assert_same(gpu_results([imgs[k]], image_index=[k], seed=7, **BENCH_CFG), [got[k]], f"image {k} alone")


@pytest.mark.gpu
def test_empty_and_kernel_free_batches():
    from limap_b200.vplib import JLinkageDetector
    det = JLinkageDetector(dict(BENCH_CFG), seed=7)
    assert det.detect_batch([]) == []
    assert det.stats()["n_images"] == 0 and det.stats()["n_vps"] == 0
    # no image reaches min_lines: the kernel is not launched and every label is -1
    imgs = [np.zeros((0, 4)), _image(19, 3), _shrink(_image(40, 4), 20.0)]
    res = det.detect_batch(imgs)
    assert [r.labels for r in res] == [[-1] * len(s) for s in imgs] and all(r.count_vps() == 0 for r in res)
    assert det.stats()["kernel_ms"] == 0


# ---- 2. the benched shape: 1000 images x 300 segments, first, second and later images of a CTA -------------------

@pytest.mark.gpu
def test_bench_shape_first_and_later_images_of_each_cta():
    from limap_b200.synth import make_vp_images
    imgs = make_vp_images(1000, 300, seed=77)
    got = gpu_results(imgs, seed=7, **BENCH_CFG)
    g = _vp_grid()
    assert 3 * g + 1 < 998
    # first images of their CTAs (< g), second (g to 2g - 1), third (2g to 3g - 1) and later ones
    pick = sorted({0, 1, g // 2, g - 1, g, g + 1, 2 * g - 1, 2 * g, 2 * g + 1, 3 * g - 1, 3 * g, 3 * g + 1, 900, 998, 999})
    want = oracle_results([imgs[k] for k in pick], image_index=pick, seed=7, n_models=5000, **BENCH_CFG)
    assert_same([got[k] for k in pick], want, "bench shape")
    assert all(len(v) >= 3 for _, v in want)


# ---- 3. model counts and the shared-memory limit ------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("n_models", [1, 31, 32, 33, 4000, 4007, 4008, 4096, 5000])
def test_model_counts(n_models):
    # with 300 segments, dynamic shared memory is 12 n_models + 916 bytes and the kernel's static bytes come on top:
    # 4007 models is the largest count within the 48 KB default limit, 4008 the smallest that needs the opt-in
    # attribute (its dynamic bytes alone, 49 012, would still fit)
    assert (12 * 4007 + 916 + STATIC_SMEM <= 48 * 1024) and (12 * 4008 + 916 + STATIC_SMEM > 48 * 1024 >= 12 * 4008 + 916)
    imgs = [_image(300, 31), _image(33, 32), _image(120, 33), _image(20, 34)]
    check_against_oracle(imgs, n_models=n_models, seed=11, min_num_supports=5)


def _largest_model_count(max_n):
    import torch
    optin = torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    return (optin - STATIC_SMEM - 3 * max_n - 16) // 12  # vp_smem_bytes = 12 n_models + 3 max_n + 16


@pytest.mark.gpu
def test_largest_accepted_model_count_runs_and_one_more_is_refused():
    """m models fill the opt-in shared memory of a block with the kernel's static bytes counted; m + 1 fit the limit
    on their dynamic bytes alone, but not with the static bytes, so the host must refuse them instead of launching."""
    from limap_b200._cabi import LimapB200Error
    imgs = [_image(40, 41), _image(25, 42)]
    m = _largest_model_count(40)
    assert 4096 < m < 65536
    check_against_oracle(imgs, n_models=m, seed=5, min_num_supports=5)
    with pytest.raises(LimapB200Error, match="too large for shared memory"):
        gpu_results(imgs, n_models=m + 1, seed=5, min_num_supports=5)
    # the same count fits with fewer segments per image
    check_against_oracle([_image(37, 43)], n_models=m + 1, seed=5, min_num_supports=5)


@pytest.mark.gpu
def test_host_rejections():
    from limap_b200._cabi import LimapB200Error
    img = [_image(30, 1)]
    for m in (0, 65536):
        with pytest.raises(LimapB200Error, match="n_models must be"):
            gpu_results(img, n_models=m)
    # 8193 valid segments in one image: refused before anything is allocated for them
    rng = np.random.default_rng(0)
    p = rng.uniform(0, 800, (8193, 2))
    big = np.concatenate([p, p + [45.0, 0.0]], 1)
    with pytest.raises(LimapB200Error, match="8192"):
        gpu_results([img[0], big])


# ---- 4. the consensus decision d < th planted at d == th and one ulp either side --------------------------------

PLANT_SEED = 3
PLANT_N = 24  # valid segments; min_num_supports = 2 gives min_lines = 20
HYP_I, HYP_J = (100.0, 500.0, 120.0, 100.0), (700.0, 500.0, 680.0, 100.0)  # lines meeting near (400, -5500)


def _bits(a):
    return np.asarray(a, F).view(np.int32)


def _flt(b):
    return np.asarray(b, np.int32).view(F)


def _plant_at(vp, th, target, length):
    """A segment from near the origin towards the VP whose float32 consensus distance is exactly `target`. Endpoint 2
    lies 2 th - 0.1 px off the line from the origin to the VP, endpoint 1 is (x1, 0): x1 is bisected on its bits to
    where d crosses target, then searched ulp by ulp. Near the origin x1 moves num by far less than an ulp of num,
    so every float value of d near th is reached."""
    v = np.array([float(c) for c in vp])
    u = v[:2] / v[2]
    u /= np.linalg.norm(u)
    n = np.array([-u[1], u[0]])
    for s in (1.0, -1.0):
        x2, y2 = (F(c) for c in length * u + s * (2 * float(th) - 0.1) * n)

        def d(b):
            return consensus_d(_flt(b), F(0), x2, y2, vp)

        lo, hi = int(_bits(F(0))), int(_bits(F(0.25)))
        if not d(lo) < target < d(hi):
            continue
        while hi - lo > 1:
            mid = (lo + hi) // 2
            lo, hi = (mid, hi) if d(mid) < target else (lo, mid)
        cand = lo + np.arange(-4096, 4096, dtype=np.int32)
        hit = np.flatnonzero(d(cand) == target)
        if len(hit):
            return (float(_flt(cand[hit[0]])), 0.0, float(x2), float(y2))
    raise AssertionError(f"no float32 endpoint gives d == {target!r}")


def planted_consensus_scene(th):
    """One image, one model. The model's pair (drawn by splitmix64 like the kernel) gets two segments whose lines meet
    near (400, -5500); three segments are planted at d == nextafter(th, 0), d == th and d == nextafter(th, inf); the
    rest are horizontal segments far outside the threshold. Returns (segments, planted slots, predicted labels): the
    inliers of the one model form the one cluster (label 0, kept because its two hypothesis segments lie far apart),
    every other segment stays a singleton that min_num_supports = 2 drops (label -1)."""
    th = F(th)
    i, j = hypothesis_pair(PLANT_SEED, 0, 0, PLANT_N, 1)
    vp = model_vp(HYP_I, HYP_J)
    segs = np.array([[200.0 + 25 * k, 550.0 + 10 * k, 245.0 + 25 * k, 550.0 + 10 * k] for k in range(PLANT_N)])
    segs[i], segs[j] = HYP_I, HYP_J
    free = [k for k in range(PLANT_N) if k not in (i, j)]
    targets = (np.nextafter(th, F(0)), th, np.nextafter(th, F(np.inf)))
    slots = free[3:6]
    for slot, t, length in zip(slots, targets, (50.0, 60.0, 70.0)):
        segs[slot] = _plant_at(vp, th, t, length)
    d = consensus_d(segs[:, 0], segs[:, 1], segs[:, 2], segs[:, 3], vp)
    assert [d[s] for s in slots] == list(targets)
    pred = np.where(d < th, 0, -1).astype(np.int32)
    assert list(pred[slots]) == [0, -1, -1] and pred[i] == 0 and pred[j] == 0 and (pred == 0).sum() == 3
    return segs, slots, pred


PLANT_CFG = dict(n_models=1, seed=PLANT_SEED, min_num_supports=2, min_length=0.0)


@pytest.mark.parametrize("th", [1.0, 0.5, 2.0])
def test_consensus_restatement_matches_oracle_at_threshold(th):
    segs, slots, pred = planted_consensus_scene(th)
    (lab, vps), = oracle_results([segs], inlier_threshold=th, **PLANT_CFG)
    assert np.array_equal(lab, pred)
    assert len(vps) == 1


@pytest.mark.gpu
@pytest.mark.parametrize("th", [1.0, 0.5, 2.0])
def test_consensus_planted_at_threshold(th):
    segs, slots, pred = planted_consensus_scene(th)
    want = check_against_oracle([segs], inlier_threshold=th, **PLANT_CFG)
    assert np.array_equal(want[0][0], pred)


# ---- 5. ties and degenerate input --------------------------------------------------------------------------------

def _degenerate_scenes():
    rng = np.random.default_rng(5)
    base = _image(40, 51)
    dup = np.concatenate([base, base[:20], base[5:15]])  # duplicated segments: identical preference sets, exact ties
    dup = dup[rng.permutation(len(dup))]
    same = np.repeat(base[:1], 30, 0)  # every hypothesis is (0, 0, 0): no inlier anywhere
    pts = _image(30, 52)
    zero = np.concatenate([pts, np.repeat(pts[:10, :2], 2, 1)])  # 10 zero-length segments (points)
    zero = zero[rng.permutation(len(zero))]
    only_zero = np.repeat(pts[:25, :2], 2, 1)  # every hypothesis has norm 0
    far = _image(80, 53) + 1e5  # float coordinates near 1e5 keep about 2 decimals
    collinear = np.concatenate([base[:25], base[:25, [0, 1, 0, 1]] + 2.0 * (base[:25] - base[:25, [0, 1, 0, 1]])])
    return dict(duplicated=(dup, {}), identical=(same, {}), zero_length=(zero, dict(min_length=0.0)),
                only_zero_length=(only_zero, dict(min_length=0.0)), far_coordinates=(far, {}),
                collinear=(collinear, {}))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["duplicated", "identical", "zero_length", "only_zero_length", "far_coordinates",
                                  "collinear"])
def test_ties_and_degenerate_input(name):
    segs, cfg = _degenerate_scenes()[name]
    want = check_against_oracle([segs], seed=13, **{"min_num_supports": 5, **cfg})
    if name in ("identical", "only_zero_length"):
        assert (want[0][0] == -1).all()


# ---- 6. host post-processing edges (engine_vp.cu) --------------------------------------------------------------

def _clutter(rng, n, lo=20.0, hi=70.0):
    """Segments of 45-150 px at angles between lo and hi degrees (away from the planted axis-parallel families)."""
    a = rng.uniform([0, 0], [800, 600], (n, 2))
    ang = np.radians(rng.uniform(lo, hi, n)) * rng.choice([-1, 1], n)
    return np.concatenate([a, a + rng.uniform(45, 150, (n, 1)) * np.stack([np.cos(ang), np.sin(ang)], 1)], 1)


def _toward(starts, vp, length):
    d = np.asarray(vp, float) - starts
    return np.concatenate([starts, starts + length * d / np.linalg.norm(d, axis=1, keepdims=True)], 1)


def _host_len(s):
    """The host's fp64 segment length, in its operation order."""
    return np.sqrt((s[:, 0] - s[:, 2]) * (s[:, 0] - s[:, 2]) + (s[:, 1] - s[:, 3]) * (s[:, 1] - s[:, 3]))


def _min_length_scene(short):
    """19 segments of 45-160 px and one 24-32-40 triangle hypotenuse of exactly 40 px, or of one ulp under 40 px when
    `short`: 20 (= min_lines) or 19 valid segments."""
    end_y = np.nextafter(132.0, 0.0) if short else 132.0
    segs = np.concatenate([_image(19, 61), [[200.0, 100.0, 224.0, end_y]]])
    assert (_host_len(segs) >= 40.0).sum() == (19 if short else 20)
    return [segs], dict(min_num_supports=3)


def _expect_min_length(short, res):
    (lab, vps), = res
    assert (len(vps) == 0 and (lab == -1).all()) if short else len(vps) >= 2


def _family_scene(k):
    """A family of k segments towards a VP far right (first in the list), one of 8 towards a VP far above and
    clutter, 22 segments; min_num_supports = 5. k = 5: the family is one cluster of exactly min_num_supports members
    and is kept; k = 4: it is dropped, and the cluster after it is renumbered to 0."""
    rng = np.random.default_rng(62)
    fam_a = _toward(np.stack([np.full(k, 60.0) + 37 * np.arange(k), 40.0 + 110 * np.arange(k)], 1), (2600.0, 330.0), 90.0)
    fam_b = _toward(np.stack([300.0 + 55 * np.arange(8), np.full(8, 560.0) - 9 * np.arange(8)], 1), (520.0, -3400.0), 85.0)
    return [np.concatenate([fam_a, fam_b, _clutter(rng, 14 - k)])], dict(min_num_supports=5)


def _expect_family(k, res):
    (lab, vps), = res
    a, b = lab[:k], lab[k:k + 8]
    assert (b == b[0]).all() and b[0] >= 0
    if k == 5:
        assert (a == 0).all() and (lab == 0).sum() == 5 and b[0] == 1
    else:
        assert (a == -1).all() and b[0] == 0


def _perp_scene(offset):
    """Exactly horizontal segments (first in the list) at y = 0 (200 px), y = offset (100 px), 150, 300 and 450, exactly
    vertical ones at x = 400, 500, ..., 900, and clutter; min_num_supports = 5. The 100 px segment's endpoints lie
    exactly `offset` from the line y = 0, so count_valid_supports_2d(th = 3.0) joins the two at offset 3.0 (4 supports:
    the family is dropped) and not at nextafter(3.0, 4.0) (5 supports: kept). Both families have VPs at infinity."""
    rng = np.random.default_rng(63)
    hor = np.array([[0.0, 0.0, 200.0, 0.0], [40.0, offset, 140.0, offset], [10.0, 150.0, 190.0, 150.0],
                    [5.0, 300.0, 175.0, 300.0], [30.0, 450.0, 160.0, 450.0]])
    ver = np.array([[400.0 + 100 * k, 50.0, 400.0 + 100 * k, 110.0 + 10 * k] for k in range(6)])
    return [np.concatenate([hor, ver, _clutter(rng, 9)])], dict(min_num_supports=5)


def _expect_perp(joined, res):
    (lab, vps), = res
    ver = lab[5:11]
    assert (ver == ver[0]).all()
    if joined:
        assert (lab[:5] == -1).all() and ver[0] == 0
    else:
        assert (lab[:5] == 0).all() and ver[0] == 1
        assert vps[0][2] == 0 and abs(abs(vps[0][0]) - 1) < 1e-15
    assert vps[ver[0]][2] == 0 and abs(abs(vps[ver[0]][1]) - 1) < 1e-15


def _singletons_scene():
    """120 clutter segments and 3 collinear extensions of them, 40 models, min_num_supports = 1: every cluster,
    singletons included, becomes a VP, more than the 64 the detector sizes its first call for. The segments of no
    model's consensus set stay singletons; singleton and collinear clusters fit a rank-deficient matrix."""
    rng = np.random.default_rng(64)
    c = _clutter(rng, 120, 0.0, 180.0)
    segs = np.concatenate([c, c[:3, [0, 1, 0, 1]] + 1.5 * (c[:3] - c[:3, [0, 1, 0, 1]])])
    return [segs], dict(min_num_supports=1, n_models=40)


def _expect_singletons(res):
    (lab, vps), = res
    assert len(vps) > 64 and lab.max() == len(vps) - 1 and (lab >= 0).all()
    assert any((lab == v).sum() == 1 for v in range(len(vps)))


HOST_SCENES = {
    "min_length_at_40": (lambda: _min_length_scene(False), lambda r: _expect_min_length(False, r)),
    "min_length_below_40": (lambda: _min_length_scene(True), lambda r: _expect_min_length(True, r)),
    "cluster_of_min_num_supports": (lambda: _family_scene(5), lambda r: _expect_family(5, r)),
    "cluster_one_short_renumbered": (lambda: _family_scene(4), lambda r: _expect_family(4, r)),
    "perp_offset_at_3": (lambda: _perp_scene(3.0), lambda r: _expect_perp(True, r)),
    "perp_offset_above_3": (lambda: _perp_scene(np.nextafter(3.0, 4.0)), lambda r: _expect_perp(False, r)),
    "singleton_vps": (_singletons_scene, _expect_singletons),
}


@pytest.mark.parametrize("name", list(HOST_SCENES))
def test_host_scene_decisions_on_oracle(name):
    """The planted scenes take the decision they are built for on the oracle (so the GPU parity below covers it)."""
    make, expect = HOST_SCENES[name]
    imgs, cfg = make()
    expect(oracle_results(imgs, seed=17, **cfg))


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(HOST_SCENES))
def test_host_post_processing_edges(name):
    make, expect = HOST_SCENES[name]
    imgs, cfg = make()
    expect(check_against_oracle(imgs, seed=17, **cfg))


@pytest.mark.gpu
def test_vp_cap_retry_equals_a_call_sized_for_all_vps():
    from limap_b200._cabi import VPConfig, check, lib, ptr
    (segs,), cfg = _singletons_scene()
    det = _detector(seed=17, **cfg)
    r, = det.detect_batch([segs])  # room for 64 VPs: the detector calls again with room for all
    assert r.count_vps() > 64
    c = det.config_
    vcfg = VPConfig(c["min_length"], c["inlier_threshold"], det.th_perp_supports_effective,
                    int(c["min_num_supports"]), det.n_models, det.seed)
    off = np.array([0, len(segs)], np.int64)
    flat = np.ascontiguousarray(segs, np.float64)
    labels, vp_off, vps = np.full(len(segs), -7, np.int32), np.zeros(2, np.int64), np.zeros((256, 3))
    n = check(lib().lm_vp_detect_indexed(det._ctx.handle, 1, ptr(off), ptr(flat), C.byref(vcfg), None, ptr(labels),
                                         ptr(vp_off), ptr(vps), 256))
    assert n == r.count_vps() and list(vp_off) == [0, n]
    assert np.array_equal(labels, np.asarray(r.labels, np.int32))
    assert np.array_equal(vps[:n], np.asarray(r.vps))
