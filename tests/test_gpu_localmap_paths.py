"""The resident local map (vxs_map.cu) where its pools grow, its root hash is rebuilt and its point_fix pool is compacted: CUDA vs the oracle's
sliding-window simulator (oracle_api.SlidingSim, which tests/test_ref_pin.py pins against the reference's OctoTree code), mgsize = 1.

Scenes are planar patches on a grid of 1 m root cells.  Each scan puts exactly k points into each of its cells, on a plane whose normal axis
is fixed per cell.  Every coordinate is a multiple of 1/512 m and every pose is a signed permutation with a dyadic translation, so world
points, slot sums, pcr_add and pcr_fix are exact in fp64 and agree bit for bit whatever the summation order.  Each case asserts that it
crossed its boundary, through the kernel launch counts of the timers, counts() or the oracle's state, and compares every leaf after every
scan (bit-exact cell / layer / flags / point counts, sums to 1e-10; 1e-8 once a BA moved the poses).  test_scenes_cross_their_boundaries
runs every scene through the oracle alone and checks the recut margins and the boundary facts without a GPU."""
import functools

import numpy as np
import pytest

import oracle_api as oa
import voxel_slam_b200 as vx
from parity_checks import compare_factor, compare_leaves, leaf_key

VXS_ERR_ARG = -2
GRID = 512                     # every coordinate is a multiple of 1 / GRID m
LOW, HIGH = 5 / 16, 13 / 16    # patch height inside its cell along the cell's normal axis, and the height of the points that break the plane
MARGIN = 1e-6                  # relative distance every plane / tras_opt decision keeps from its threshold
VAR = (np.eye(3) * 2.0 ** -14).reshape(9)
NODE_CAP0, SW_CAP0, FIX_COMPACT = 1 << 16, 1 << 12, 1 << 16      # initial node capacity, slide-window blocks, compaction floor (vxs_map.cu)

# worst observed error / tolerance per comparator family, and what each boundary case reached (printed at the end of the module, run with -s)
WORST, REACHED = {}, {}


def note(family, ratio):
    WORST[family] = max(WORST.get(family, 0.0), float(ratio))


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    if WORST:
        print("\nworst error/tolerance: " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(WORST.items())))
    for k, v in REACHED.items():
        print(f"{k}: {v}")


@pytest.fixture(scope="module")
def ctx():
    c = vx.Context(0)
    c.timing(True)
    yield c
    c.close()


# ------------------------------------------------------------------------------------------------ host rules of vxs_map.cu
def bits_for(v):
    """vxs_sortscan.cuh bits_for: the smallest b with 2^b > v, at least 1"""
    return max(int(v).bit_length(), 1)


def radix_passes(n_nodes):
    """accumulate_sorted sorts (leaf << 8 | slot) keys on bits_for(n_nodes) + 8 bits, 8 bits per k_radix_scatter pass"""
    return -(-(bits_for(n_nodes) + 8) // 8)


def node_capacity(ncap, need):
    """map_reserve_nodes: the node capacity after reserving `need` nodes"""
    if need <= ncap:
        return ncap
    nc = max(2 * ncap, NODE_CAP0)
    while nc < need:
        nc *= 2
    return nc


def accum_group(avg):
    """accumulate_sorted: lanes per node of k_map_accum from the average points per node"""
    return 32 if avg > 24.0 else (8 if avg > 3.0 else 1)


# ------------------------------------------------------------------------------------------------ scenes
def grid_cells(nx, ny, nz=1, origin=(0, 0, 0)):
    g = np.stack(np.meshgrid(np.arange(nx), np.arange(ny), np.arange(nz), indexing="ij"), -1).reshape(-1, 3)
    return g + np.asarray(origin)


def patch_points(cells, k, seed, level=LOW):
    """exactly k points in every cell: uniform in the plane over 0.05 ... 0.95 of the cell, at `level` +- 2/512 m along the cell's normal axis"""
    rng = np.random.default_rng(seed)
    cells = np.asarray(cells, dtype=np.int64).reshape(-1, 3)
    C = len(cells)
    u = rng.integers(26, 487, (C, k, 3)) / GRID
    axis = (cells[:, 0] + 2 * cells[:, 1] + 3 * cells[:, 2]) % 3              # the same normal in every scan
    u[np.arange(C), :, axis] = level + rng.integers(-2, 3, (C, k)) / GRID
    return (cells[:, None, :] + u).reshape(-1, 3)


def make_pose(seed):
    """signed permutation (det +1) and a translation on a 1/64 m grid: the body <-> world maps are exact"""
    rng = np.random.default_rng(seed)
    R = np.eye(3)[rng.permutation(3)] * rng.choice([-1.0, 1.0], 3)[:, None]
    if np.linalg.det(R) < 0:
        R[2] *= -1
    return np.concatenate([R.reshape(9), rng.integers(-256, 257, 3) / 64])


def records(world, pose):
    """pointVar records (body point | var) of world points seen from `pose`"""
    R, t = pose[:9].reshape(3, 3), pose[9:]
    return np.concatenate([(world - t) @ R, np.broadcast_to(VAR, (len(world), 9))], axis=1)


def scan(cells_k, seed, pose_seed=None, level=LOW):
    """one scan: (cells, k) groups -> (world points, true pose)"""
    world = np.concatenate([patch_points(c, k, seed + 7919 * j, level) for j, (c, k) in enumerate(cells_k)])
    return world, make_pose(seed if pose_seed is None else pose_seed)


def assert_exact_k(world, cells_k):
    """the scan holds exactly k points in every one of its cells (oracle voxel keys)"""
    cells, cnt = np.unique(oa.voxel_keys(world, 1.0)[0], axis=0, return_counts=True)
    got = dict(zip(map(tuple, cells), cnt))
    want = {}
    for c, k in cells_k:
        for cc in map(tuple, np.asarray(c).reshape(-1, 3)):
            want[cc] = want.get(cc, 0) + k
    assert got == want


def scene(W, scans, max_layer=2, max_points=100, **meta):
    for s in scans:
        assert_exact_k(s["world"], s["cells_k"])
    return dict(W=W, scans=scans, max_layer=max_layer, max_points=max_points, **meta)


def mkscan(cells_k, seed, level=LOW):
    w, p = scan(cells_k, seed, level=level)
    return dict(world=w, pose=p, cells_k=cells_k)


A64 = grid_cells(64, 64)                                   # 4096 cells


@functools.lru_cache(maxsize=None)
def node_growth_scene(first_roots):
    """case 1: a first scan on `first_roots` cells, then 61 440-point scans over those cells and new ones: n_nodes + n = first_roots + 61440"""
    A = np.concatenate([A64, [[64, 0, 0]]])[:first_roots]
    B = grid_cells(128, 128, 1, (0, 0, 3))[: 15360 - first_roots]
    scans = [mkscan([(A, 4)], 10)] + [mkscan([(A, 4), (B, 4)], 11 + i) for i in range(4)]
    return scene(3, scans, first_roots=first_roots, odom_cells=np.concatenate([A[::7], B[::11]]))


@functools.lru_cache(maxsize=None)
def recut_growth_scene():
    """case 2: four planar scans, a fifth that breaks every plane, then two planar scans into the children"""
    scans = [mkscan([(A64, 4)], 20 + i) for i in range(4)] + [mkscan([(A64, 4)], 24, level=HIGH)] + [mkscan([(A64, 4)], 25 + i) for i in range(2)]
    return scene(5, scans)


@functools.lru_cache(maxsize=None)
def radix_scene():
    """case 3: 65 535 roots, then 65 536"""
    G = grid_cells(256, 256)
    return scene(3, [mkscan([(G[:-1], 1)], 30), mkscan([(G, 1)], 31), mkscan([(G, 1)], 32)])


SW_A, SW_B, SW_C = grid_cells(60, 50), grid_cells(40, 25, 1, (0, 0, 10)), grid_cells(70, 50, 1, (0, 0, 20))


@functools.lru_cache(maxsize=None)
def sw_pool_scene():
    """case 4: area A (3000 roots) for a window, B (1000) until A leaves the slide map, one scan over B and 3500 new roots C, back to A, then A + C"""
    seq = [[(SW_A, 2)]] * 3 + [[(SW_B, 2)]] * 2 + [[(SW_B, 2), (SW_C, 2)]] + [[(SW_A, 2)]] * 2 + [[(SW_A, 2), (SW_C, 2)]]
    return scene(3, [mkscan(c, 40 + i) for i, c in enumerate(seq)], odom_cells=np.concatenate([SW_A[::5], SW_C[::5]]))


FX_X, FX_Y = A64, grid_cells(32, 16, 1, (0, 0, 5))


@functools.lru_cache(maxsize=None)
def fix_pool_scene():
    """case 5, max_points = 20: X (4096 roots, 8 points per scan) fills its point_fix to 24 and then loses it; Y (512 roots, 2 per scan) keeps
    its point_fix; after the compaction a scan breaks Y's planes, so the compacted point_fix is subdivided"""
    seq = [([(FX_X, 8), (FX_Y, 2)], LOW)] * 6 + [([(FX_X, 8), (FX_Y, 4)], None), ([(FX_X, 8), (FX_Y, 2)], LOW)]
    scans = []
    for i, (c, lv) in enumerate(seq):
        if lv is None:     # Y's points on the far plane of their cell
            s = mkscan([c[0]], 50 + i)
            y = mkscan([c[1]], 150 + i, level=HIGH)
            s = dict(world=np.concatenate([s["world"], y["world"]]), pose=s["pose"], cells_k=c)
        else:
            s = mkscan(c, 50 + i, level=lv)
        scans.append(s)
    return scene(3, scans, max_points=20, odom_cells=np.concatenate([FX_X[::9], FX_Y]))


ACCUM = [(3, 1), (4, 8), (24, 8), (25, 32)]


@functools.lru_cache(maxsize=None)
def accum_scene(k):
    """case 6: 256 roots, exactly k points per (root, scan)"""
    C = grid_cells(16, 16, 1, (-8, -3, -1))
    return scene(4, [mkscan([(C, k)], 60 + i) for i in range(6)], k=k)


@functools.lru_cache(maxsize=None)
def window_scene(W):
    """case 7: small scans; W = 250 fills its window and slides 10 times"""
    if W == 250:
        C = grid_cells(8, 5, 1, (-4, 2, 0))
        return scene(W, [mkscan([(C, 2)], 1000 + i) for i in range(W + 10)])
    C = grid_cells(20, 10, 1, (3, -5, 2))
    return scene(W, [mkscan([(C, 6)], 70 + 20 * W + i) for i in range(8)])


@functools.lru_cache(maxsize=None)
def w50_scene():
    """case 7, W = 50: 2500 roots, 8 points each per scan (20 000 points), 60 scans; the estimated poses are off by up to 3/256 m"""
    C = grid_cells(50, 50, 1, (-20, -20, 0))
    scans = [mkscan([(C, 8)], 300 + i) for i in range(60)]
    rng = np.random.default_rng(5)
    for i, s in enumerate(scans):
        s["est"] = s["pose"].copy()
        if i:
            s["est"][9:] += rng.integers(-3, 4, 3) / 256
    return scene(50, scans, ba_iters=1)


# ------------------------------------------------------------------------------------------------ one sequence, device and oracle side by side
def kernel_calls(ctx):
    return {k: v[1] for k, v in ctx.timing_read().items()}


def check_margins(so, mp, tag):
    """every leaf the next recut decides on (slide root, window, N > min_point) keeps its plane and tras_opt decisions a relative MARGIN from
    their thresholds, so that eigensolver rounding cannot flip one"""
    a, lay = so["pcr_add"], so["layer"]
    mpt = np.array([mp.min_point[min(l, 3)] for l in lay]) if len(lay) else np.zeros(0)
    live = so["in_slide"] & so["has_sw"] & so["isexist"] & (a[:, 9] > mpt)
    if not live.any():
        return
    a, lay = a[live], lay[live]
    n = a[:, 9]
    P = np.stack([a[:, [0, 1, 2]], a[:, [1, 3, 4]], a[:, [2, 4, 5]]], 1) / n[:, None, None]
    m = a[:, 6:9] / n[:, None]
    lam = np.linalg.eigvalsh(P - m[:, :, None] * m[:, None, :])
    thre = np.array([mp.plane_thre[min(l, 3)] for l in lay])
    mev = mp.min_eigen_value
    r02, r01 = lam[:, 0] / lam[:, 2], lam[:, 0] / lam[:, 1]
    assert np.all(np.abs(lam[:, 0] - mev) > MARGIN * mev), (tag, "min eigenvalue")
    assert np.all(np.abs(r02 - thre) > MARGIN * thre), (tag, "plane ratio")
    plane = (lam[:, 0] < mev) & (r02 < thre)
    assert np.all(np.abs(r01[plane] - 0.12) > MARGIN * 0.12), (tag, "tras_opt ratio")


OPEN = []


@pytest.fixture(autouse=True)
def _close_runs():
    """every device map is destroyed before its context, also when a case fails"""
    yield
    while OPEN:
        OPEN.pop().close()


class Run:
    """one sequence through vx.LocalMap and oa.SlidingSim (the device side is skipped when ctx is None)"""

    def __init__(self, ctx, sc):
        self.ctx, self.sc, self.W = ctx, sc, sc["W"]
        self.mp = vx.MapParams.make(voxel_size=1.0, max_layer=sc["max_layer"])
        self.sim = oa.SlidingSim(self.mp, self.W, 1, max_points=sc["max_points"])
        self.dm = vx.LocalMap(ctx, self.mp, self.W, max_points=sc["max_points"]) if ctx else None
        self.f = vx.Factor(ctx, self.W) if ctx else None
        self.ba = sc.get("ba_iters", 0)
        self.tol = 1e-10 if self.ba == 0 else 1e-8
        self.x_buf = []
        self.push_calls, self.margi_calls = {}, {}
        if ctx:
            OPEN.append(self)

    def step(self, i, compare=True):
        s = self.sc["scans"][i]
        pose = s.get("est", s["pose"])
        pv = records(s["world"], s["pose"])
        self.x_buf.append(pose)
        full = len(self.x_buf) >= self.W
        if self.dm is not None:
            self.ctx.timing_reset()
            self.dm.push_scan(pv, np.stack(self.x_buf), self.f)
            self.push_calls, self.margi_calls = kernel_calls(self.ctx), {}
        self.sim.add_scan_pv(pv, pose, ba_iters=self.ba)
        if self.dm is not None and compare and self.ba == 0:
            compare_factor(self.f, self.sim.factor(), self.W)          # the oracle's margi only reads the factor tras_opt extracted
            note("factor", factor_ratio(self.f, self.sim.factor(), self.W))
        if full:
            if self.dm is not None:
                if self.ba > 0 and self.f.counts()[0] >= 2:
                    o = self.ctx.lidar_ba(self.f, np.stack(self.x_buf), max_iter=self.ba, thd_num=2, want_hess=False)
                    self.x_buf = list(o["poses"])
                self.ctx.timing_reset()
                self.dm.margi(np.stack(self.x_buf), self.f, mgsize=1)
                self.margi_calls = kernel_calls(self.ctx)
            self.x_buf = self.x_buf[1:]
        so = self.sim.state()
        check_margins(so, self.mp, i)
        if self.dm is not None and compare:
            if self.ba > 0 and len(so["poses"]):
                assert np.max(np.abs(np.stack(self.x_buf) - so["poses"])) < 1e-8, i
            sg = self.dm.leaves()
            compare_leaves(sg, so, i, tol=self.tol)
            note("leaf sums", leaf_ratio(sg, so) / self.tol)
        return so

    def close(self):
        if self.dm is not None:
            self.dm.close(); self.f.close()
            self.dm = None


def leaf_ratio(sg, so):
    kg, ko = leaf_key(sg), leaf_key(so)
    r = 0.0
    for f in ("pcr_add", "pcr_fix", "slots"):
        x, y = sg[f][kg], so[f][ko]
        if x.size:
            r = max(r, float(np.max(np.abs(x - y) / (np.abs(y) + 1e-6))))
    return r


def factor_ratio(f_gpu, of, W):
    """the largest relative sum error of compare_factor over its tolerance (1e-10), and eigenvalue error over 1e-7"""
    ex = of.export()
    ptr, fr, cl, fx, co = f_gpu.read_structure()
    eig, s = f_gpu.read_back()
    if len(s) == 0:
        return 0.0
    kg, ko = np.lexsort(np.round(s[:, [8, 7, 6, 9]], 7).T), np.lexsort(np.round(ex["sum10"][:, [8, 7, 6, 9]], 7).T)
    dense = np.zeros((len(s), W, 10))
    dense[np.repeat(np.arange(len(s)), np.diff(ptr)), fr] = cl
    r = max(float(np.max(np.abs(a[kg] - b[ko]) / (np.abs(b[ko]) + 1e-6))) for a, b in ((dense, ex["clusters10"]), (s, ex["sum10"]), (fx, ex["fix10"])))
    lo = ex["eig12"][ko][:, :3]
    return max(r / 1e-10, float(np.max(np.abs(eig[kg][:, :3] - lo) / np.max(np.abs(lo), axis=1, keepdims=True))) / 1e-7)


def check_odometry(run, cells, seed):
    """one association pass of the odometry EKF against the resident map: flags bit-exact, HTH / HTz / nnt to 1e-9"""
    world = patch_points(cells, 2, seed)
    pose = make_pose(seed)
    pv = records(world, pose)
    rng = np.random.default_rng(seed)
    A = rng.standard_normal((3, 3)) * 1e-3; B = rng.standard_normal((3, 3)) * 1e-2
    og = run.dm.odom_accumulate(pv, pose, A @ A.T, B @ B.T)
    oo = run.sim.odom_accumulate(pv, pose, A @ A.T, B @ B.T)
    assert oo["n"] > len(world) // 4 and og["n"] == oo["n"] and np.array_equal(og["flags"], oo["flags"]), (og["n"], oo["n"])
    for k in ("HTH", "HTz", "nnt"):
        err = np.max(np.abs(og[k] - oo[k])) / np.max(np.abs(oo[k]))
        note("odometry", err / 1e-9)
        assert err < 1e-9, k
    return oo["n"]


def compare_planes(run):
    """the plane table plane_update left behind, tolerances of test_gpu_localmap.py"""
    pg, po = run.dm.planes(), run.sim.planes()
    assert len(pg["N"]) == len(po["N"]) > 0
    kg, ko = np.lexsort(np.round(pg["voxel_center"], 9).T), np.lexsort(np.round(po["voxel_center"], 9).T)
    assert np.array_equal(pg["voxel_center"][kg], po["voxel_center"][ko]) and np.array_equal(pg["N"][kg], po["N"][ko])
    dc = np.max(np.abs(pg["center"][kg] - po["center"][ko]))
    dn = np.max(np.abs(np.abs(np.sum(pg["normal"][kg] * po["normal"][ko], axis=1)) - 1))
    sgn = np.sign(np.sum(pg["normal"][kg] * po["normal"][ko], axis=1))
    Vo = po["plane_var"][ko].copy(); Vo[:, :3, 3:] *= sgn[:, None, None]; Vo[:, 3:, :3] *= sgn[:, None, None]
    dv = np.max(np.abs(pg["plane_var"][kg] - Vo) / np.max(np.abs(Vo), axis=(1, 2), keepdims=True))
    note("planes", max(dc / 1e-9, dn / 1e-8, dv / 1e-5))
    assert dc < 1e-9 and dn < 1e-8 and dv < 1e-5, (dc, dn, dv)


# ------------------------------------------------------------------------------------------------ oracle-side facts of every scene
@functools.lru_cache(maxsize=None)
def fix_pool_trace():
    """the device's point_fix pool predicted from the oracle's per-leaf n_point_fix: entries are appended at margi, die when their leaf drops its
    point_fix, and the pool is compacted to its live entries when it holds more than 2^16 entries and more than half are dead.  Returns per
    scan (pool entries, dead entries before the compaction check, compacted, live entries)."""
    sc = fix_pool_scene()
    run = Run(None, sc)
    prev, pool, dead, out = {}, 0, 0, []
    for i in range(len(sc["scans"])):
        so = run.step(i)
        cur = {(tuple(np.round(c, 9)), l): n for c, l, n in zip(so["voxel_center"], so["layer"], so["n_point_fix"])}
        assert not np.any(so["n_point_fix"][so["layer"] >= sc["max_layer"]])     # no entry is dropped by a subdivision to max_layer
        # a leaf that keeps existing and loses its point_fix lost it to the margi kill; a subdivided leaf hands its entries to its children
        killed = sum(n for key, n in prev.items() if n > 0 and cur.get(key, -1) == 0)
        live = sum(cur.values())
        pool += live - sum(prev.values()) + killed           # appended = live change + killed
        dead += killed
        compact = pool > FIX_COMPACT and 2 * dead > pool
        out.append((pool, dead, compact, live))
        if compact:
            pool, dead = live, 0
        prev = cur
    return out


SCENES = {
    "node-growth-65536": lambda: node_growth_scene(4096), "node-growth-65537": lambda: node_growth_scene(4097), "recut-growth": recut_growth_scene,
    "radix": radix_scene, "sw-pool": sw_pool_scene, "fix-pool": fix_pool_scene, **{f"accum-k{k}": functools.partial(accum_scene, k) for k, _ in ACCUM},
    "W1": functools.partial(window_scene, 1), "W2": functools.partial(window_scene, 2), "W250": functools.partial(window_scene, 250), "W50": w50_scene,
}


@pytest.mark.parametrize("name", list(SCENES))
def test_scenes_cross_their_boundaries(name):
    """oracle alone: the recut margins after every scan (inside Run.step) and the boundary each scene is built for"""
    sc = SCENES[name]()
    run = Run(None, sc)
    states = [run.step(i) for i in range(len(sc["scans"]))]
    n = [len(s["world"]) for s in sc["scans"]]
    if name.startswith("node-growth"):
        r1 = sc["first_roots"]
        assert len(states[0]["layer"]) == r1 and np.all(states[0]["layer"] == 0)                # n_nodes = r1 after the first push
        assert r1 + n[1] == (NODE_CAP0 if r1 == 4096 else NODE_CAP0 + 1)
        assert all(len(s["layer"]) == 15360 and np.all(s["layer"] == 0) for s in states[1:])   # no subdivision: 15 360 nodes
        assert node_capacity(node_capacity(NODE_CAP0, n[0]), r1 + n[1]) == (NODE_CAP0 if r1 == 4096 else 2 * NODE_CAP0)
    elif name == "recut-growth":
        assert all(len(s["layer"]) == 4096 and np.all(s["layer"] == 0) for s in states[:4])
        assert 4096 + n[4] <= NODE_CAP0 < 4096 + sum(n[:5])               # no growth at push start; the recut flags every window point
        assert np.all(states[4]["layer"] == 1) and len(np.unique(np.floor(states[4]["voxel_center"]), axis=0)) == 4096
    elif name == "radix":
        assert [len(s["layer"]) for s in states] == [65535, 65536, 65536] and all(np.all(s["layer"] == 0) for s in states)
        assert [radix_passes(len(s["layer"])) for s in states] == [3, 4, 4]
    elif name == "sw-pool":
        held = [int(np.sum(s["has_sw"])) for s in states]
        assert held[5] == 4500 > SW_CAP0 and max(held[:5]) <= SW_CAP0                        # the pool grows on scan 5
        a = np.isin(np.floor(states[4]["voxel_center"])[:, 2], [0])
        assert not states[4]["in_slide"][a].any() and np.all(states[4]["pcr_fix"][a][:, 9] == 6)
        a6 = np.floor(states[6]["voxel_center"])[:, 2] == 0
        assert states[6]["in_slide"][a6].all() and np.all(states[6]["pcr_fix"][a6][:, 9] == 6) and a6.sum() == 3000
    elif name == "fix-pool":
        tr = fix_pool_trace()
        k = [i for i, t in enumerate(tr) if t[2]]
        assert k == [5], tr                                                 # one compaction, in the margi of scan 5
        pool, dead, _, live = tr[5]
        assert pool > FIX_COMPACT and 2 * dead > pool and live == 4096
        assert max(t[0] for t in tr[:5]) > FIX_COMPACT                     # the pool grew past 2^16 with content
        assert np.any((states[6]["layer"] == 1) & (states[6]["n_point_fix"] > 0))    # the compacted point_fix was subdivided
    elif name.startswith("accum"):
        k = sc["k"]
        assert all(len(s["layer"]) == 256 and np.all(s["layer"] == 0) for s in states)      # every accumulation: 256 nodes x k points
        assert accum_group(float(k)) == dict(ACCUM)[k]
    elif name == "W250":
        assert states[-1]["win_count"] == 249 and states[248]["win_count"] == 249


# ------------------------------------------------------------------------------------------------ GPU cases
@pytest.mark.gpu
@pytest.mark.parametrize("first_roots", [4096, 4097], ids=["nodes65536-no-growth", "nodes65537-grows-and-rehashes"])
def test_node_growth_at_push_start(ctx, first_roots):
    """the node table grows at push start when n_nodes + n exceeds its capacity; with nodes in it, the root hash is rebuilt.  At 65 536 the
    second push fits and the table grows one push later (15 360 + 61 440 nodes), at 65 537 it grows in the second push."""
    sc = node_growth_scene(first_roots)
    run = Run(ctx, sc)
    ncap, nodes, rehashed = NODE_CAP0, 0, []
    for i in range(len(sc["scans"])):
        need = nodes + len(sc["scans"][i]["world"])
        grows = need > ncap
        ncap = node_capacity(ncap, need)
        run.step(i)
        assert run.push_calls.get("k_map_rehash", 0) == int(grows and nodes > 0), i
        if grows:
            rehashed.append(i)
        nodes = run.dm.counts()["nodes"]
        assert nodes == (first_roots if i == 0 else 15360)
    assert rehashed == ([2] if first_roots == 4096 else [1])
    REACHED[f"node growth {first_roots}"] = dict(nodes=nodes, capacity=ncap, rehash_at_scan=rehashed)          # 4096: the second push (n_nodes + n = 65536) did not rehash
    check_odometry(run, sc["odom_cells"], 90 + first_roots)
    compare_planes(run)
    run.close()


@pytest.mark.gpu
def test_node_growth_inside_recut(ctx):
    sc = recut_growth_scene()
    run = Run(ctx, sc)
    for i in range(4):
        run.step(i)
        assert run.dm.counts()["nodes"] == 4096 and run.push_calls.get("k_map_rehash", 0) == 0
    run.step(4)
    c = run.push_calls
    assert 4096 + len(sc["scans"][4]["world"]) <= NODE_CAP0                  # no growth at push start ...
    assert c.get("k_map_rehash", 0) == 1 and c.get("k_map_subdiv_assign", 0) >= 2   # ... so the rehash ran between subdivision passes
    assert run.dm.counts()["nodes"] > 4096
    REACHED["recut growth"] = dict(nodes_at_push_start=4096, points_flagged=5 * 4096 * 4, nodes_after=run.dm.counts()["nodes"])
    for i in range(5, 7):
        run.step(i)
    run.close()


@pytest.mark.gpu
def test_radix_width_crosses_2_pow_16(ctx):
    sc = radix_scene()
    run = Run(ctx, sc)
    for i, nodes in enumerate([65535, 65536, 65536]):
        run.step(i)
        assert run.dm.counts()["nodes"] == nodes
        assert run.push_calls["k_radix_scatter"] == radix_passes(nodes) == (3 if nodes < 65536 else 4)
    run.close()


@pytest.mark.gpu
def test_slide_window_pool_grows_with_free_blocks(ctx):
    sc = sw_pool_scene()
    run = Run(ctx, sc)
    held, left, back = [], False, False
    for i in range(len(sc["scans"])):
        so = run.step(i)
        held.append(int(np.sum(so["has_sw"])))
        a = np.floor(so["voxel_center"])[:, 2] == 0
        left = left or (not so["in_slide"][a].any() and np.all(so["pcr_fix"][a][:, 9] > 0))
        back = back or (left and so["in_slide"][a].all() and np.all(so["pcr_fix"][a][:, 9] > 0))
    assert max(held) > SW_CAP0 and left and back
    REACHED["slide-window pool"] = dict(windows_held_per_scan=held)
    check_odometry(run, sc["odom_cells"], 94)
    run.close()


@pytest.mark.gpu
def test_point_fix_growth_and_compaction(ctx):
    sc = fix_pool_scene()
    tr = fix_pool_trace()
    run = Run(ctx, sc)
    for i in range(len(sc["scans"])):
        so = run.step(i)
        pool, dead, compact, live = tr[i]
        assert run.margi_calls.get("k_map_fix_compact", 0) == (1 if compact else 0), i
        assert run.dm.counts()["fix_points"] == (live if compact else pool) == (int(np.sum(so["n_point_fix"])) if compact else pool), i
        if i == 6:
            assert run.push_calls.get("k_map_subdiv_assign", 0) >= 2
    REACHED["point_fix pool"] = dict(entries_per_scan=[t[0] for t in tr], dead=[t[1] for t in tr], live=[t[3] for t in tr])
    check_odometry(run, sc["odom_cells"], 95)
    compare_planes(run)
    run.close()


@pytest.mark.gpu
@pytest.mark.parametrize("k,G", ACCUM, ids=[f"k{k}-G{g}" for k, g in ACCUM])
def test_accumulation_group_width(ctx, k, G):
    sc = accum_scene(k)
    assert accum_group(float(k)) == G
    run = Run(ctx, sc)
    for i in range(len(sc["scans"])):
        run.step(i)
        assert run.dm.counts()["nodes"] == 256 and run.push_calls["k_map_accum"] == 1          # one accumulation, average exactly k
    run.close()


@pytest.mark.gpu
@pytest.mark.parametrize("W", [1, 2, 250], ids=["W1-margi-every-scan", "W2", "W250-full-window-and-10-slides"])
def test_window_sizes(ctx, W):
    sc = window_scene(W)
    run = Run(ctx, sc)
    for i in range(len(sc["scans"])):
        run.step(i, compare=(W < 250 or i % 25 == 0 or i >= W - 1))
        assert run.dm.counts()["win_count"] == min(i + 1, W - 1 if i >= W - 1 else W)
    run.close()


@pytest.mark.gpu
def test_window_size_limits(ctx):
    mp = vx.MapParams.make(voxel_size=1.0, max_layer=2)
    for W in (0, 251):
        with pytest.raises(vx.VxsError) as e:
            vx.LocalMap(ctx, mp, W)
        assert e.value.code == VXS_ERR_ARG


@pytest.mark.gpu
def test_window_50_with_ba():
    """W = 50, 20 000 points per scan, 60 scans, one LM iteration between push and margi.  Its own context: the BA's kernels do not crowd the
    timer table that the other cases read."""
    c = vx.Context(0)
    sc = w50_scene()
    try:
        run = Run(c, sc)
        for i in range(len(sc["scans"])):
            run.step(i)
        assert run.dm.counts()["win_count"] == 49
    finally:
        while OPEN:
            OPEN.pop().close()
        c.close()


@pytest.mark.gpu
def test_negative_control_point_across_a_cell_face(ctx):
    """one point moved into the neighbouring cell in the oracle's copy only: compare_leaves must fail, and pass without the move"""
    sc = accum_scene(4)
    run = Run(ctx, sc)
    moved = oa.SlidingSim(run.mp, run.W, 1, max_points=sc["max_points"])
    for i in range(2):
        run.step(i)
        w = sc["scans"][i]["world"].copy()
        if i == 1:
            w[0, 0] += 1.0
        moved.add_scan_pv(records(w, sc["scans"][i]["pose"]), sc["scans"][i]["pose"])
    with pytest.raises(AssertionError):
        compare_leaves(run.dm.leaves(), moved.state(), "moved")
    run.close()
