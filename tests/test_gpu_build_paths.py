"""The from-scratch map build (build_factor in vxs_voxelize.cu) and the batched bottom level of the hierarchical BA (vxs_hba_bottom_batch) at the
shapes where their host drivers switch: CUDA vs the CPU oracle.

Map build.  Scenes are grids of small planar patches in which every (root cell, frame) pair holds exactly k points, so the layer-0 record
average is exactly k and the k_rec_clusters group width, the radix pass count, the frame-bit width and the root-box guard are reached by
construction.  Each scene builder checks its invariant on the oracle side, and mirrors the recut decision tree in numpy (fp64 covariance,
eigvalsh) to check that no plane / tras_opt decision lies within rounding of its threshold, so that a different summation order cannot flip
one.  Device factors are compared with the oracle's: ids and per-(voxel, frame) counts bit-exact, sums 1e-12, eigenvalues 1e-7 of lambda_max.

Bottom batch.  Every window is an independent seeded 3-plane room; a batch concatenates the clouds of a few distinct windows and lists them in
win_first in any order, repeats included.  Each window's expected result is the oracle's hba_window(max_iter = 1) on that window alone; its
LM bookkeeping (iterations, convergence) is the trace of the oracle's lidar_ba(max_iter = 4) on the window's GBA factor."""
import functools

import numpy as np
import pytest

import oracle_api as oa
import scenes
import voxel_slam_b200 as vx
from parity_checks import compare_bottom_window, compare_factors
from voxel_slam_b200.api import VXS_ERR_TOO_FEW_VOXELS, VXS_WARN_SINGULAR

VXS_ERR_ARG, VXS_ERR_RANGE = -2, -6
MARGIN = 1e-8      # relative distance every map decision and every LM decision keeps from its threshold

# worst observed error / tolerance per comparator family (printed at the end of the module, run with -s to see it)
WORST = {}


def note(family, ratio):
    WORST[family] = max(WORST.get(family, 0.0), float(ratio))


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    if WORST:
        print("\nworst error/tolerance: " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(WORST.items())))


@pytest.fixture(scope="module")
def ctx():
    c = vx.Context(0)
    c.timing(True)
    yield c
    c.close()


@functools.lru_cache(maxsize=None)
def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


# ------------------------------------------------------------------------------------------------ host selection rules (vxs_voxelize.cu)
def bits_for(v):
    """vxs_sortscan.cuh bits_for: the smallest b with 2^b > v, at least 1"""
    return max(int(v).bit_length(), 1)


def pick_rec_group(avg):
    """build_factor: lanes per (node, frame) record of k_rec_clusters from the average points per record"""
    return 32 if avg > 48.0 else (8 if avg > 12.0 else (4 if avg > 3.0 else 1))


def radix_passes(key_bits):
    return -(-key_bits // 8)


def layer0_key_bits(cells_box, nframes):
    """layer-0 sort key: (linear root cell << FB) | frame, FB = bits_for(frames incl. the fix pseudo-frame)"""
    return bits_for(cells_box) + bits_for(nframes)


def window_sort_passes(nwin):
    """vxs_hba_bottom_batch sorts a chunk's voxels by window on bits_for(nwin) bits"""
    return radix_passes(bits_for(nwin))


# ------------------------------------------------------------------------------------------------ scenes of planar patches
def rot_exp(w):
    th = np.linalg.norm(w)
    K = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])
    if th == 0:
        return np.eye(3)
    return np.eye(3) + np.sin(th) / th * K + (1 - np.cos(th)) / th ** 2 * K @ K


def make_poses(W, seed, identity=False):
    rng = np.random.default_rng(seed)
    P = np.zeros((W, 12))
    for i in range(W):
        R = np.eye(3) if identity else rot_exp(rng.normal(0, 0.05, 3))
        P[i, :9] = R.reshape(9)
        P[i, 9:] = 0 if identity else rng.uniform(-0.3, 0.3, 3)
    return P


def world_of(body, poses, off):
    w = np.empty((body.shape[0], 3))
    for i in range(poses.shape[0]):
        R, t = poses[i, :9].reshape(3, 3), poses[i, 9:]
        w[off[i]:off[i + 1]] = body[off[i]:off[i + 1]].astype(np.float64) @ R.T + t
    return w


def patch_scene(cells, W, k, seed, vs=1.0, identity=False, dtype=np.float64, counts=None, thick=2e-3, grid=0):
    """every (cell, frame) pair gets exactly k points (or counts[frame]) of the cell's planar patch: a square of side 0.9 vs inside the cell,
    normal along a per-cell axis, thickness `thick` vs.  grid > 0 rounds the world points to multiples of 1 / grid.  Returns body points frame
    by frame, offsets, poses and the world points."""
    rng = np.random.default_rng(seed)
    cells = np.asarray(cells, dtype=np.int64).reshape(-1, 3)
    C = cells.shape[0]
    axis = rng.integers(0, 3, C)
    poses = make_poses(W, seed + 1, identity)
    kk = [k] * W if counts is None else list(counts)
    world, off = [], [0]
    for i in range(W):
        u = rng.uniform(0.05, 0.95, (C, kk[i], 3))
        u[np.arange(C), :, axis] = 0.5 + thick * rng.standard_normal((C, kk[i]))
        world.append(((cells[:, None, :] + u) * vs).reshape(-1, 3))
        off.append(off[-1] + C * kk[i])
    off = np.array(off, dtype=np.int64)
    world = np.concatenate(world) if W else np.zeros((0, 3))
    if grid:
        world = np.round(world * grid) / grid
    body = np.empty_like(world)
    for i in range(W):
        R, t = poses[i, :9].reshape(3, 3), poses[i, 9:]
        body[off[i]:off[i + 1]] = (world[off[i]:off[i + 1]] - t) @ R
    body = body.astype(dtype)
    return dict(pts=body, off=off, poses=poses, world=world_of(body, poses, off), cells=cells)


def record_stats(world, frame, vs):
    """(number of (root cell, frame) records, their point counts) from the oracle's voxel keys"""
    key = oa.voxel_keys(world, vs)[0]
    _, cnt = np.unique(np.concatenate([key, frame[:, None]], axis=1), axis=0, return_counts=True)
    return len(cnt), cnt


def mirror_recut(world, frame, W, mp, gba):
    """numpy restatement of the recut decisions (k_node_decide / the oracle's recut + tras_opt) on the world points.  Asserts that every alive
    node's plane test and every plane's tras_opt test keep a relative MARGIN from their thresholds; returns (voxels taken, their entries)."""
    vs = mp.voxel_size
    key = oa.voxel_keys(world, vs)[0]
    cen = (0.5 + key.astype(np.float64)) * vs
    path = np.zeros(len(world), dtype=np.int64)
    q = np.float32(vs / 4)
    idx = np.arange(len(world))
    V = E = 0
    for layer in range(mp.max_layer + 1):
        if len(idx) == 0:
            break
        _, inv = np.unique(np.concatenate([key[idx], path[idx, None]], axis=1), axis=0, return_inverse=True)
        inv = inv.reshape(-1)
        nn = inv.max() + 1
        n = np.bincount(inv, minlength=nn).astype(np.float64)
        infr = frame[idx] < W
        nwin = np.zeros(nn, dtype=np.int64)
        pairs = np.unique(np.stack([inv[infr], frame[idx][infr]], axis=1), axis=0)
        if len(pairs):
            nwin = np.bincount(pairs[:, 0], minlength=nn)
        p = world[idx]
        mean = np.stack([np.bincount(inv, p[:, a], nn) for a in range(3)], 1) / n[:, None]
        cov = np.zeros((nn, 3, 3))
        for a in range(3):
            for b in range(3):
                cov[:, a, b] = np.bincount(inv, p[:, a] * p[:, b], nn) / n - mean[:, a] * mean[:, b]
        alive = (n > 10) if gba else ((n > mp.min_point[min(layer, 3)]) & (nwin > 0))
        lam = np.zeros((nn, 3))
        if alive.any():
            lam[alive] = np.linalg.eigvalsh(cov[alive])
        l0, l1, l2 = lam[:, 0], lam[:, 1], np.where(alive, lam[:, 2], 1.0)
        mev, thre = mp.min_eigen_value, mp.plane_thre[min(layer, 3)]
        a_ok, b_ok = l0 < mev, l0 / l2 < thre
        plane = alive & a_ok & b_ok
        a_far, b_far = np.abs(l0 - mev) > MARGIN * mev, np.abs(l0 / l2 - thre) > MARGIN * thre
        assert np.all((a_far & b_far)[plane]), "a plane decision within rounding of its threshold"
        assert np.all(((~a_ok & a_far) | (~b_ok & b_far))[alive & ~plane]), "a non-plane decision within rounding of its threshold"
        r01 = l0 / np.where(plane, l1, 1.0)
        assert np.all((np.abs(r01 - 0.12) > MARGIN * 0.12)[plane]), "a tras_opt decision within rounding of its threshold"
        take = plane & (r01 <= 0.12)
        if gba:
            take &= nwin > 1
        V += int(take.sum()); E += int(nwin[take].sum())
        sub = alive & ~plane
        if layer == mp.max_layer:
            break
        idx = idx[sub[inv]]
        bit = world[idx] > cen[idx]
        path[idx] = path[idx] * 8 + 4 * bit[:, 0] + 2 * bit[:, 1] + bit[:, 2]
        cen[idx] += (2 * bit - 1) * np.float64(q)
        q = np.float32(q / np.float32(2))
    return V, E


def frames_of(off):
    return np.repeat(np.arange(len(off) - 1), np.diff(off))


def oracle_window_factor(sc, mp, fix=None, threads=1):
    W = len(sc["off"]) - 1
    of = oa.build_window_factor(mp, sc["pts"], sc["off"], sc["poses"], fix_pts=fix, threads=threads)
    world, fr = sc["world"], frames_of(sc["off"])
    if fix is not None:
        world, fr = np.concatenate([world, fix]), np.concatenate([fr, np.full(len(fix), W)])
    V, E = mirror_recut(world, fr, W, mp, gba=False)
    ex = of.export()
    assert V == of.size() and E == int(np.count_nonzero(ex["clusters10"][:, :, 9])), (V, E, of.size())
    return of


def oracle_gba_factor(sc, mp, threads=2):
    W = len(sc["off"]) - 1
    of = oa.build_gba_factor(mp, sc["pts"], sc["off"], sc["poses"], threads=threads, stride_floats=sc["pts"].shape[1])
    V, E = mirror_recut(world_of(sc["pts"][:, :3], sc["poses"], sc["off"]), frames_of(sc["off"]), W, mp, gba=True)
    assert V == of.size(), (V, of.size())
    return of


def grid_cells(nx, ny, nz=1, origin=(0, 0, 0)):
    g = np.stack(np.meshgrid(np.arange(nx), np.arange(ny), np.arange(nz), indexing="ij"), -1).reshape(-1, 3)
    return g + np.asarray(origin)


def widen(pts, stride):
    wide = np.zeros((pts.shape[0], stride), dtype=np.float32)
    wide[:, :3] = pts
    wide[:, 3:] = 7.0
    return wide


MP0 = vx.MapParams.make(voxel_size=1.0, max_layer=0)
GBA0 = vx.MapParams.make(voxel_size=1.0, min_eigen_value=0.0025, max_layer=0)


# record width: k points per (cell, frame) -> G; window mode needs k W > min_point (5), GBA mode k W > 10 and two frames per plane
BAND = [(3, 1), (4, 4), (12, 4), (13, 8), (48, 8), (49, 32)]


@functools.lru_cache(maxsize=None)
def band_scene(mode, k):
    W = 4 if mode == "window" else max(4, -(-11 // k))
    sc = patch_scene(grid_cells(6, 5, 2, (-3, 1, -1)), W, k, 100 + k, dtype=np.float64 if mode == "window" else np.float32)
    R, cnt = record_stats(sc["world"], frames_of(sc["off"]), 1.0)
    assert R == 60 * W and np.all(cnt == k)                 # layer-0 average exactly k
    if mode == "gba":
        sc["pts"] = widen(sc["pts"], 12)
        return sc, oracle_gba_factor(sc, GBA0)
    return sc, oracle_window_factor(sc, MP0)


def build_gpu(ctx, mode, sc, mp, of, fix=None, f=None):
    W = len(sc["off"]) - 1
    f = f or vx.Factor(ctx, W)
    if mode == "window":
        n, ids = ctx.build_window_factor(mp, sc["pts"], sc["off"], sc["poses"], f, fix_pts=fix, want_ids=True, ids_cap=of.size() + 16)
    else:
        n, ids = ctx.build_gba_factor(mp, sc["pts"], sc["off"], sc["poses"], f, stride_floats=sc["pts"].shape[1], want_ids=True, ids_cap=of.size() + 16)
    assert n == f.counts()[0] == of.size()
    return f, ids


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["window", "gba_stride12"])
@pytest.mark.parametrize("k,G", BAND, ids=[f"k{k}-G{g}" for k, g in BAND])
def test_record_width_band_edges(ctx, mode, k, G):
    sc, of = band_scene(mode.split("_")[0], k)
    assert pick_rec_group(float(k)) == G and of.size() == 60
    ctx.timing_reset()
    f, ids = build_gpu(ctx, mode.split("_")[0], sc, GBA0 if mode != "window" else MP0, of)
    assert ctx.timing_read()["k_rec_clusters"][1] == 1
    compare_factors(f, ids, of, len(sc["off"]) - 1, note)


# grid-stride loop of k_rec_clusters: more records than the capped grid (sm_count * 16 blocks of 256 threads) has groups
@functools.lru_cache(maxsize=None)
def stride_scene(G):
    if G == 32:
        k, W, cells = 49, 2, grid_cells(100, 86)                  # 17 200 records
    else:
        k, W, cells = 2, 3, grid_cells(427, 427)                  # 546 987 records, 1.09 M points
    sc = patch_scene(cells, W, k, 200 + G)
    R, cnt = record_stats(sc["world"], frames_of(sc["off"]), 1.0)
    assert np.all(cnt == k) and R == len(cells) * W
    return sc, oracle_window_factor(sc, MP0, threads=8), R, k


@pytest.mark.gpu
@pytest.mark.parametrize("G", [32, 1], ids=["G32-many-records", "G1-1M-points"])
def test_record_grid_stride_loop(ctx, G):
    sc, of, R, k = stride_scene(G)
    assert pick_rec_group(float(k)) == G
    assert R > sm_count() * 16 * 256 // G               # every group loops over at least two records
    f, ids = build_gpu(ctx, "window", sc, MP0, of)
    compare_factors(f, ids, of, len(sc["off"]) - 1, note)


# radix passes at layer 0: key_bits = bits_for(root box) + bits_for(W)
RADIX = [(8, 2, (4, 4, 2)), (9, 4, (4, 4, 2)), (16, 4, (64, 64, 1)), (17, 8, (64, 64, 1))]


@functools.lru_cache(maxsize=None)
def radix_scene(W, box):
    corners = np.array([[0, 0, 0], [box[0] - 1, box[1] - 1, box[2] - 1], [1, 2, 0], [box[0] - 1, 0, 0]])
    sc = patch_scene(corners, W, 6, 300 + W)
    return sc, oracle_window_factor(sc, MP0)


@pytest.mark.gpu
@pytest.mark.parametrize("key_bits,W,box", RADIX, ids=[f"bits{b}-W{w}-box{x[0]}x{x[1]}x{x[2]}" for b, w, x in RADIX])
def test_radix_pass_count(ctx, key_bits, W, box):
    sc, of = radix_scene(W, box)
    assert layer0_key_bits(box[0] * box[1] * box[2], W) == key_bits
    ctx.timing_reset()
    f, ids = build_gpu(ctx, "window", sc, MP0, of)
    assert ctx.timing_read()["k_radix_scatter"][1] == radix_passes(key_bits)
    compare_factors(f, ids, of, W, note)


# the 2^40-cell guard on the root box: patches at opposite corners of a cube of side 10321 (2^40 - 87 321 615 cells) and 10322
@functools.lru_cache(maxsize=None)
def cube_scene(side):
    lo = -(side // 2)
    hi = lo + side - 1
    # at 5e3 m the fp64 covariance of a patch cancels ~8 digits, and two summation orders differ by more than the eigenvalue tolerance;
    # on a 1/512 m grid every point sum is exact (x^2 needs 44 bits), so the comparison sees the build and not the cancellation
    sc = patch_scene([[lo, lo, lo], [hi, hi, hi], [lo, hi, lo]], 2, 8, 400, identity=True, grid=512)
    assert np.abs(sc["world"]).max() < 5200
    return sc


@pytest.mark.gpu
def test_root_box_guard_at_2_pow_40_cells(ctx):
    sc = cube_scene(10321)
    assert 10321 ** 3 == 2 ** 40 - 87321615
    of = oracle_window_factor(sc, MP0)
    assert of.size() == 3
    ctx.timing_reset()
    f, ids = build_gpu(ctx, "window", sc, MP0, of)
    assert ctx.timing_read()["k_radix_scatter"][1] == radix_passes(40 + bits_for(2)) == 6
    compare_factors(f, ids, of, 2, note)
    big = cube_scene(10322)
    assert 10322 ** 3 >= 2 ** 40
    with pytest.raises(vx.VxsError) as e:
        ctx.build_window_factor(MP0, big["pts"], big["off"], big["poses"], f)
    assert e.value.code == VXS_ERR_RANGE


# frame-bit width FB = bits_for(W [+ 1 with fixed map points])
FRAMES = [(w, False) for w in (1, 2, 3, 4, 7, 8, 15, 16, 31, 32, 33)] + [(w, True) for w in (7, 15, 31)]


@functools.lru_cache(maxsize=None)
def frames_scene(W, fix):
    cells = grid_cells(3, 2, 2, (-1, 0, -2))
    sc = patch_scene(cells, W, 6, 500 + W)
    fx = None
    if fix:   # fixed map points on the same patches, in world coordinates
        f = patch_scene(cells, 1, 5, 500 + W, identity=True)
        fx = f["world"]
    return sc, fx, oracle_window_factor(sc, MP0, fix=fx)


@pytest.mark.gpu
@pytest.mark.parametrize("W,fix", FRAMES, ids=[f"W{w}{'-fix' if x else ''}-FB{bits_for(w + x)}" for w, x in FRAMES])
def test_frame_bit_width(ctx, W, fix):
    sc, fx, of = frames_scene(W, fix)
    assert of.size() == 12
    if fix:
        assert bits_for(W + 1) == bits_for(W) + 1 and np.abs(of.export()["fix10"]).max() > 0
    f, ids = build_gpu(ctx, "window", sc, MP0, of, fix=fx)
    compare_factors(f, ids, of, W, note)


# octant descent: points exactly on the child-centre planes of layers 1-3 belong to the "not greater" side
@functools.lru_cache(maxsize=None)
def octant_scene():
    """root cells with negative indices; each cell holds one planar patch per layer-3 child (normal axis cycling with the child index), and the
    patch of child (a, b, c) lies exactly on its upper face along its normal axis when that face is a split plane (index < 7)"""
    rng = np.random.default_rng(600)
    W, per = 2, 4
    pts = [[] for _ in range(W)]
    for cell in ([-1, -2, 0], [-3, 0, -1]):
        for a in range(8):
            for b in range(8):
                for c in range(8):
                    ch = np.array([a, b, c])
                    ax = (a + b + c) % 3
                    for fr in range(W):
                        u = (ch + rng.uniform(0.1, 0.9, (per, 3))) / 8
                        u[:, ax] = (ch[ax] + 1) / 8 if ch[ax] < 7 else (ch[ax] + 0.5) / 8
                        pts[fr].append(np.asarray(cell) + u)
    world = [np.concatenate(p) for p in pts]
    off = np.concatenate([[0], np.cumsum([len(p) for p in world])]).astype(np.int64)
    sc = dict(pts=np.concatenate(world), off=off, poses=make_poses(W, 0, identity=True))
    sc["world"] = sc["pts"].copy()
    frac = (sc["world"] - np.floor(sc["world"])) * 8
    on = np.isclose(frac, np.round(frac), rtol=0, atol=0) & (np.round(frac) % 8 != 0)
    assert on.any(axis=1).mean() > 0.8                      # most points sit exactly on a split plane of layer 1, 2 or 3
    mp = vx.MapParams.make(voxel_size=1.0, max_layer=3)
    of = oracle_window_factor(sc, mp)
    ids = of.export()["ids"]
    assert (ids["layer"] == 3).sum() > 100 and (ids["x"] < 0).all()
    return sc, mp, of


@pytest.mark.gpu
def test_octant_boundaries_layers_1_to_3(ctx):
    sc, mp, of = octant_scene()
    f, ids = build_gpu(ctx, "window", sc, mp, of)
    compare_factors(f, ids, of, 2, note)


# degenerate inputs
def degenerate_scene(case):
    cells = grid_cells(4, 3, 1, (2, -5, 0))
    if case in ("empty-first-frame", "empty-middle-frame", "empty-last-frame"):
        j = {"empty-first-frame": 0, "empty-middle-frame": 2, "empty-last-frame": 4}[case]
        return patch_scene(cells, 5, 6, 700, counts=[0 if i == j else 6 for i in range(5)])
    if case == "N0":
        return patch_scene(cells, 3, 0, 701)
    if case == "N1":
        sc = patch_scene(cells[:1], 1, 1, 702)
        return sc
    if case == "one-root-cell":
        return patch_scene([[3, -2, 1]], 4, 20, 703)
    if case == "frame-without-planes":
        sc = patch_scene(cells, 4, 6, 704)
        rng = np.random.default_rng(705)
        blob = np.array([10, 10, 10]) + rng.uniform(0.05, 0.95, (40, 3))    # a 3-D blob in a cell of its own, seen by frame 2 only
        R, t = sc["poses"][2, :9].reshape(3, 3), sc["poses"][2, 9:]
        ins = sc["off"][3]
        sc["pts"] = np.concatenate([sc["pts"][:ins], (blob - t) @ R, sc["pts"][ins:]])
        sc["off"] = sc["off"] + np.array([0, 0, 0, 40, 40])
        sc["world"] = world_of(sc["pts"], sc["poses"], sc["off"])
        return sc
    raise KeyError(case)


DEGENERATE = ["empty-first-frame", "empty-middle-frame", "empty-last-frame", "N0", "N1", "one-root-cell", "frame-without-planes"]


@pytest.mark.gpu
@pytest.mark.parametrize("case", DEGENERATE)
def test_degenerate_inputs(ctx, case):
    sc = degenerate_scene(case)
    W = len(sc["off"]) - 1
    of = oracle_window_factor(sc, MP0)
    expect = {"N0": 0, "N1": 0, "one-root-cell": 1}.get(case)
    assert expect is None and of.size() > 0 or of.size() == expect
    f, ids = build_gpu(ctx, "window", sc, MP0, of)
    compare_factors(f, ids, of, W, note)
    if case == "frame-without-planes":
        _, fr, _, _, _ = f.read_structure()
        assert 2 in fr and of.size() == 12                  # the blob is not a voxel; frame 2's patch entries are


@pytest.mark.gpu
def test_ids_cap_below_voxel_count(ctx):
    sc, of = band_scene("window", 13)
    V = of.size()
    f = vx.Factor(ctx, 4)
    n, full = ctx.build_window_factor(MP0, sc["pts"], sc["off"], sc["poses"], f, want_ids=True, ids_cap=V)
    cap = V - 7
    n2, part = ctx.build_window_factor(MP0, sc["pts"], sc["off"], sc["poses"], f, want_ids=True, ids_cap=cap)
    assert n == n2 == V and len(part) == cap and np.array_equal(part, full[:cap])
    compare_factors(f, full, of, 4, note)


# reuse: grow-only scratch and factor, SoA strides Rcap / Ncap that change between builds
@pytest.mark.gpu
@pytest.mark.parametrize("order", ["large-small", "small-large", "plain-fix-plain"])
def test_reuse_between_builds(ctx, order):
    large = (stride_scene(32)[0], stride_scene(32)[1])
    small = band_scene("window", 4)
    fixs = frames_scene(7, True)
    seq = {"large-small": [large, small], "small-large": [small, large], "plain-fix-plain": [small, (fixs[0], fixs[2], fixs[1]), large]}[order]
    f = vx.Factor(ctx, 8)
    for item in seq:
        sc, of = item[0], item[1]
        fx = item[2] if len(item) > 2 else None
        f, ids = build_gpu(ctx, "window", sc, MP0, of, fix=fx, f=f)
        compare_factors(f, ids, of, len(sc["off"]) - 1, note)


@pytest.mark.gpu
def test_hba_window_with_changing_window_size():
    """vxs_hba_window keeps its factor on the context, created at the first call's W"""
    c = vx.Context(0)
    try:
        coarse = vx.MapParams.make(voxel_size=2.0, min_eigen_value=0.1, max_layer=2)
        fine = vx.MapParams.make(voxel_size=1.0, min_eigen_value=0.0025, max_layer=2)
        for W in (10, 16, 4):
            tr, est = scenes.poses_true_est(W, 8.0, 70 + W, rot_sigma=3e-3, pos_sigma=2e-2)
            xyz, off = scenes.make_points(W, 2000, 8.0, 70 + W, tr, dtype=np.float32)
            g = c.hba_window(coarse, fine, xyz, off, est, max_iter=3, thread_num=2)
            r = oa.hba_window(coarse, fine, xyz, off, est, max_iter=3, thread_num=2)
            assert g["outer_iters"] == r["outer_iters"]
            assert np.max(np.abs(g["resis_log"] - r["resis_log"]) / r["resis_log"]) < 1e-6
            inc = np.max(np.abs(r["poses"] - est))
            note("hba_window poses", np.max(np.abs(g["poses"] - r["poses"])) / (1e-5 * inc))
            assert np.max(np.abs(g["poses"] - r["poses"])) < 1e-5 * inc
            assert np.max(np.abs(g["hess"] - r["hess"])) < 1e-6 * np.max(np.abs(r["hess"]))
    finally:
        c.close()


# ------------------------------------------------------------------------------------------------ bottom batch
FINE = vx.MapParams.make(voxel_size=1.0, min_eigen_value=0.0025, max_layer=2)
PATHS = dict(reject=(60, 2e-2, 1e-1), early=(60, 1e-4, 1e-3), full=(62, 2e-2, 1e-1))


@functools.lru_cache(maxsize=None)
def window_data(seed, ws, rs=3e-3, ps=2e-2, pts=1500, empty=-1, scatter=False):
    tr, est = scenes.poses_true_est(ws, 8.0, seed, rot_sigma=rs, pos_sigma=ps)
    xyz, off = scenes.make_points(ws, pts, 8.0, seed, tr, dtype=np.float32)
    if scatter:      # no plane anywhere
        xyz = np.random.default_rng(seed).uniform(-50, 50, xyz.shape).astype(np.float32)
    if empty >= 0:
        keep = np.ones(len(xyz), bool)
        keep[off[empty]:off[empty + 1]] = False
        cnt = np.diff(off)
        cnt[empty] = 0
        xyz, off = xyz[keep], np.concatenate([[0], np.cumsum(cnt)]).astype(np.int64)
    return xyz, off, est


def lm_margins_ok(trace):
    """every accept / reject (sign of r1 - r2) and every 1e-6 stop test is far from its threshold"""
    rel = np.abs((trace["r1"] - trace["r2"]) / trace["r1"])
    return bool(np.all(rel > 1e-10) and np.all(np.abs(rel - 1e-6) > 0.5e-6))


@functools.lru_cache(maxsize=None)
def window_oracle(spec):
    xyz, off, est = window_data(*spec)
    ws = len(off) - 1
    r = oa.hba_window(FINE, FINE, xyz, off, est, max_iter=1, thread_num=2)
    of = oa.build_gba_factor(FINE, xyz, off, est, threads=2)
    nvox = of.size()
    if nvox < 2:
        return dict(nvox=nvox, est=est)
    assert r["status"] == 0 and r["outer_iters"] == 1
    V, _ = mirror_recut(world_of(xyz, est, off), frames_of(off), ws, FINE, gba=True)
    assert V == nvox
    lb = of.lidar_ba(est, max_iter=4, thd_num=2)
    # the two oracle routes (HBA_add_edge with max_iter = 1, and damping_iter(up = 4) on the window's GBA factor) agree
    assert np.max(np.abs(lb["poses"] - r["poses"])) < 1e-12 and np.max(np.abs(lb["resis"] - r["resis_log"][:2]) / r["resis_log"][:2]) < 1e-12
    assert lm_margins_ok(lb["trace"])
    return dict(r=r, e=oa.hba_edges(r["hess"], ws, r["poses"]), trace=lb["trace"], conv=lb["is_converge"], nvox=nvox, est=est)


def make_batch(specs):
    """clouds of the distinct windows back to back; win_first lists the windows of `specs` in order (repeats allowed)"""
    uniq = list(dict.fromkeys(specs))
    xs, offs, ests, first, base, pbase = [], [0], [], {}, 0, 0
    for s in uniq:
        xyz, off, est = window_data(*s)
        first[s] = base
        xs.append(xyz); ests.append(est)
        offs.extend((off[1:] + pbase).tolist())
        base += len(off) - 1; pbase += int(off[-1])
    return np.concatenate(xs), np.array(offs, dtype=np.int64), np.concatenate(ests), np.array([first[s] for s in specs], dtype=np.int32)


def check_batch(g, specs, win_first, statuses=None, note=note):
    """every window against its own oracle run; repeated windows agree with each other to 1e-10"""
    seen = {}
    for w, s in enumerate(specs):
        o = window_oracle(s)
        want = 0 if statuses is None else statuses[w]
        assert g["status"][w] == want, (w, g["status"][w], want)
        if want == 0:
            compare_bottom_window(g, w, o["r"], o["e"], o["est"], note)
            assert g["lm_iters"][w] == len(o["trace"]), (w, g["lm_iters"][w], len(o["trace"]))
            assert g["is_converge"][w] == int(np.all(o["trace"]["accepted"] == 1)) == int(o["conv"])
        if s in seen:
            v = seen[s]
            d = max(np.max(np.abs(g["poses"][w] - g["poses"][v])), np.max(np.abs(g["resis"][w] - g["resis"][v]) / np.maximum(np.abs(g["resis"][v]), 1e-300)))
            note("repeated windows", d / 1e-10)
            assert d < 1e-10 and np.array_equal(g["edge_valid"][w], g["edge_valid"][v]) and g["lm_iters"][w] == g["lm_iters"][v]
        else:
            seen[s] = w


def run_batch(ctx, specs, ws, thread_num=2, chunk=0, want_hess=True):
    xyz, off, est, wf = make_batch(specs)
    return ctx.hba_bottom_batch(FINE, xyz, off, est, wf, win_size=ws, thread_num=thread_num, max_points_per_chunk=chunk, want_hess=want_hess), wf


WIN_SIZES = [2, 3, 15, 16]


@pytest.mark.gpu
@pytest.mark.parametrize("ws", WIN_SIZES, ids=[f"ws{w}-n{6 * w}" for w in WIN_SIZES])
def test_bottom_win_size(ctx, ws):
    pts = 1000 if ws > 10 else 1500
    pool = [(80 + ws + i, ws, 3e-3, 2e-2, pts) for i in range(3)]
    specs = [pool[1], pool[0], pool[2], pool[1]]
    g, wf = run_batch(ctx, specs, ws)
    check_batch(g, specs, wf)


@pytest.mark.gpu
def test_bottom_win_size_17_is_an_argument_error(ctx):
    xyz, off, est = window_data(81, 17, pts=300)
    with pytest.raises(vx.VxsError) as e:
        ctx.hba_bottom_batch(FINE, xyz, off, est, np.array([0], dtype=np.int32), win_size=17)
    assert e.value.code == VXS_ERR_ARG


NWIN = [127, 128, 129, 255, 256, 257]
POOL3 = [(90 + i, 3, 3e-3, 2e-2, 1500) for i in range(4)]


@pytest.mark.gpu
@pytest.mark.parametrize("nwin", NWIN, ids=[f"nwin{n}-sortpasses{window_sort_passes(n)}" for n in NWIN])
def test_bottom_window_count(ctx, nwin):
    specs = [POOL3[i] for i in np.random.default_rng(nwin).integers(0, 4, nwin)]     # unordered, repeated win_first
    assert nwin * 3 > 256                                    # the residual kernel reads the poses from global memory
    g, wf = run_batch(ctx, specs, 3, want_hess=False)
    assert len(g["status"]) == nwin and len(set(wf.tolist())) == 4
    check_batch(g, specs, wf)


CHUNK_POOL = [(s, 4, 3e-3, 2e-2, 1500) for s in (100, 102, 103, 104, 113)]


@pytest.mark.gpu
@pytest.mark.parametrize("split", ["exact-2-windows", "2-windows-minus-1", "below-one-window"])
def test_bottom_chunking_equals_one_chunk(ctx, split):
    specs = CHUNK_POOL + [CHUNK_POOL[0]]
    one = 4 * 1500
    chunk = {"exact-2-windows": 2 * one, "2-windows-minus-1": 2 * one - 1, "below-one-window": one // 3}[split]
    g0, wf = run_batch(ctx, specs, 4)
    g, _ = run_batch(ctx, specs, 4, chunk=chunk)
    check_batch(g, specs, wf)
    d = max(np.max(np.abs(g["poses"] - g0["poses"])), np.max(np.abs(g["resis"] - g0["resis"]) / g0["resis"]))
    note("chunked vs one chunk", d / 1e-10)
    assert d < 1e-10
    for k in ("status", "lm_iters", "edge_valid", "is_converge"):
        assert np.array_equal(g[k], g0[k]), k


def lm_path_specs():
    return {k: (s, 4, rs, ps, 1500) for k, (s, rs, ps) in PATHS.items()}


def check_lm_paths():
    sp = lm_path_specs()
    acc = {k: window_oracle(s)["trace"]["accepted"].tolist() for k, s in sp.items()}
    assert acc["reject"][:3] == [1, 0, 1]                    # rejects a step, then accepts
    assert len(acc["early"]) < 4 and all(acc["early"])       # stops on the 1e-6 test
    assert acc["full"] == [1, 1, 1, 1]                       # runs all 4 iterations
    return sp


@pytest.mark.gpu
def test_bottom_lm_paths_mixed_in_one_batch(ctx):
    sp = check_lm_paths()
    specs = [sp["reject"], sp["early"], sp["full"], sp["early"], sp["reject"]]
    g, wf = run_batch(ctx, specs, 4)
    check_batch(g, specs, wf)
    assert g["lm_iters"].tolist() == [4, 3, 4, 3, 4] and g["is_converge"].tolist() == [0, 1, 1, 1, 0]


TOO_FEW_POOL = [(s, 4, 3e-3, 2e-2, p) for s, p in ((111, 600), (113, 1500), (114, 1500))]


def too_few_setup():
    counts = [window_oracle(s)["nvox"] for s in TOO_FEW_POOL]
    x = int(np.argmin(counts))
    c = counts[x]
    assert all(n > c + 1 for i, n in enumerate(counts) if i != x)
    return TOO_FEW_POOL[x], [s for i, s in enumerate(TOO_FEW_POOL) if i != x], c


@pytest.mark.gpu
@pytest.mark.parametrize("where", ["first", "middle", "last"])
def test_bottom_too_few_voxels(ctx, where):
    bad, good, c = too_few_setup()
    pos = {"first": 0, "middle": 1, "last": 2}[where]
    specs = list(good)
    specs.insert(pos, bad)
    # thread_num = the window's voxel count: it passes
    g, wf = run_batch(ctx, specs, 4, thread_num=c)
    check_batch(g, specs, wf)
    # one more: it gets VXS_ERR_TOO_FEW_VOXELS, keeps its poses, reports r1 and no convergence; its neighbours are unaffected
    g, wf = run_batch(ctx, specs, 4, thread_num=c + 1)
    st = [0] * 3
    st[pos] = VXS_ERR_TOO_FEW_VOXELS
    assert g["status"].tolist() == st
    o = window_oracle(bad)
    assert np.array_equal(g["poses"][pos], o["est"]) and g["is_converge"][pos] == 0 and g["lm_iters"][pos] == 0
    assert abs(g["resis"][pos][0] - o["trace"]["r1"][0]) < 1e-7 * o["trace"]["r1"][0] and g["resis"][pos][1] == 0
    h, _ = run_batch(ctx, good, 4, thread_num=c + 1)
    rest = [w for w in range(3) if w != pos]
    assert np.max(np.abs(g["poses"][rest] - h["poses"])) < 1e-10 and np.max(np.abs(g["resis"][rest] - h["resis"]) / h["resis"]) < 1e-10
    assert np.array_equal(g["lm_iters"][rest], h["lm_iters"]) and np.array_equal(g["edge_valid"][rest], h["edge_valid"])


@pytest.mark.gpu
def test_bottom_chunk_without_voxels(ctx):
    empty = (120, 4, 3e-3, 2e-2, 1500, -1, True)
    assert window_oracle(empty)["nvox"] == 0
    good = TOO_FEW_POOL[1]
    specs = [good, empty, good]
    g, wf = run_batch(ctx, specs, 4, chunk=4 * 1500)          # one window per chunk: the middle chunk has V = 0
    assert g["status"].tolist() == [0, VXS_ERR_TOO_FEW_VOXELS, 0]
    assert np.array_equal(g["poses"][1], window_data(*empty)[2]) and g["is_converge"][1] == 0 and g["lm_iters"][1] == 0
    assert np.all(g["resis"][1] == 0) and not g["edge_valid"][1].any()
    check_batch(g, specs, wf, statuses=[0, VXS_ERR_TOO_FEW_VOXELS, 0])


@pytest.mark.gpu
@pytest.mark.parametrize("slot", [0, 2], ids=["slot0-gauge", "slot2-singular"])
def test_bottom_empty_keyframe(ctx, slot):
    ws = 5
    spec = (132, ws, 3e-3, 2e-2, 1500, slot)
    other = (133, ws, 3e-3, 2e-2, 1500)
    o = window_oracle(spec)
    g, wf = run_batch(ctx, [other, spec], ws)
    check_batch(g, [other], wf[:1])
    est = o["est"]
    if slot == 0:
        assert g["status"][1] == 0
        check_batch({k: (v[1:] if isinstance(v, np.ndarray) else v) for k, v in g.items()}, [spec], wf[1:])
        return
    assert g["status"][1] == VXS_WARN_SINGULAR
    assert np.array_equal(g["poses"][1][slot], est[slot])
    keep = [j for j in range(ws) if j != slot]
    inc = np.max(np.abs(o["r"]["poses"] - est))
    assert np.max(np.abs(g["poses"][1][keep] - o["r"]["poses"][keep])) < 1e-5 * inc
    pairs = [(i, j) for i in range(ws) for j in range(i + 1, ws)]
    assert not any(g["edge_valid"][1][p] for p, (i, j) in enumerate(pairs) if slot in (i, j))
    assert g["lm_iters"][1] == len(o["trace"])


# ------------------------------------------------------------------------------------------------ negative controls
@pytest.mark.gpu
def test_negative_control_point_across_a_cell_face(ctx):
    sc, of = band_scene("window", 13)
    moved = dict(sc)
    moved["pts"] = sc["pts"].copy()
    R, t = sc["poses"][0, :9].reshape(3, 3), sc["poses"][0, 9:]
    w = sc["world"][0].copy()
    w[0] = np.floor(w[0]) - 0.02                             # one point of frame 0 into the neighbouring cell along x
    moved["pts"][0] = (w - t) @ R
    f = vx.Factor(ctx, 4)
    n, ids = ctx.build_window_factor(MP0, moved["pts"], moved["off"], moved["poses"], f, want_ids=True, ids_cap=of.size() + 16)
    with pytest.raises(AssertionError):
        compare_factors(f, ids, of, 4)


@pytest.mark.gpu
def test_negative_control_win_first_off_by_one(ctx):
    sp = lm_path_specs()
    specs = [sp["full"], sp["reject"]]
    xyz, off, est, wf = make_batch(specs)
    wf = wf.copy()
    wf[0] += 1                                                # window 0 starts one keyframe late against its oracle
    g = ctx.hba_bottom_batch(FINE, xyz, off, est, wf, win_size=4, want_hess=True)
    with pytest.raises(AssertionError):
        check_batch(g, specs, wf, note=lambda family, ratio: None)


# ------------------------------------------------------------------------------------------------ the scene builders' invariants (CPU)
def test_scene_builders_hold_their_invariants():
    """the oracle-side checks the GPU cases rely on: exact record averages and bands, key bits, decision margins, voxel counts for thread_num,
    the intended LM trace patterns"""
    for mode in ("window", "gba"):
        for k, G in BAND:
            _, of = band_scene(mode, k)
            assert pick_rec_group(float(k)) == G and of.size() == 60
    for key_bits, W, box in RADIX:
        assert layer0_key_bits(box[0] * box[1] * box[2], W) == key_bits and radix_scene(W, box)[1].size() == 4
    assert layer0_key_bits(10321 ** 3, 2) == 42 and oracle_window_factor(cube_scene(10321), MP0).size() == 3
    for W, fix in FRAMES:
        assert frames_scene(W, fix)[2].size() == 12
    octant_scene()
    for case in DEGENERATE:
        oracle_window_factor(degenerate_scene(case), MP0)
    assert [window_sort_passes(n) for n in NWIN] == [1, 1, 1, 1, 2, 2]
    for s in POOL3 + CHUNK_POOL + [(132, 5, 3e-3, 2e-2, 1500, 0), (132, 5, 3e-3, 2e-2, 1500, 2), (133, 5, 3e-3, 2e-2, 1500)]:
        assert window_oracle(s)["nvox"] > 2
    assert window_oracle((120, 4, 3e-3, 2e-2, 1500, -1, True))["nvox"] == 0
    check_lm_paths()
    too_few_setup()
