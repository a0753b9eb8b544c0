"""The odometry association (voxelslam.cpp:876-918, OctoTree::match voxel_map.hpp:1335-1392, match :1674-1698) and var_init
(voxelslam.hpp:187-203) at their rounding edges, on both device paths:

  * the exported plane table (ctx.odom_set_planes + ctx.odom_accumulate) against the oracle's from-scratch map (oa.LocalMap);
  * the resident map (vx.LocalMap fed scan by scan, vxs_map_odom_accumulate) against the oracle's sliding-window simulator (oa.SlidingSim).

Random scenes almost never put a point within rounding of a decision, so the points here are built on the CPU from the oracle itself:
pairs of points one ulp apart in one coordinate that straddle the 3-sigma gate or the range gate, world points on root-cell faces and
octant faces and one ulp either side, and points that end in a missing root, a missing child, a non-plane leaf or outside the plane
table.  Per-point flags and the match count are bit-exact; HTH / HTz / nnt are held to 1e-9 (summation order, and sigma_l, which the
device forms from the upper triangle of plane_var).

The one-ulp gate pairs run on the exported table only: there the device holds the oracle's own plane rows, while the resident map forms
its rows with its own plane_update, equal to the oracle's to 1e-9 (centre) and 1e-5 (plane_var), so the oracle's gate is not the
resident map's gate to one ulp.  Both paths evaluate the gates in the same od_contribution (vxs_odom_math.cuh)."""
import numpy as np
import pytest

import oracle_api as oa
import scenes
import synth
import voxel_slam_b200 as vx
from parity_checks import compare_leaves, pv_records

L = 6.0
SHIFT = np.array([-2.95, -3.1, -3.3])      # puts the corner room across both signs of every axis and its edges off the octant splits
SCENES = {"vs1_l2": (1.0, 2), "vs05_l2": (0.5, 2), "vs1_l3": (1.0, 3), "vs1_l0": (1.0, 0)}
IDENT = np.concatenate([np.eye(3).ravel(), [-0.0, -0.0, -0.0]])     # R p + (-0) keeps a world coordinate of -0.0
POSE_B = np.concatenate([oa.so3_exp(np.array([0.31, -0.22, 0.57])).ravel(), [0.137, -0.291, 0.0733]])


def _rng_spd(rng, s):
    A = rng.standard_normal((3, 3)) * s
    return A @ A.T


_r = np.random.default_rng(2024)
COV_GROUPS = [(np.zeros((3, 3)), np.zeros((3, 3))), (_rng_spd(_r, 1e-3), np.zeros((3, 3))), (np.zeros((3, 3)), _rng_spd(_r, 1e-2)),
              (_rng_spd(_r, 1e-3), _rng_spd(_r, 1e-2)), (_rng_spd(_r, 3e-3), _rng_spd(_r, 5e-3))]


# ---------------------------------------------------------------- host restatement of the decisions (oracle order, no contraction)
def world(pose, b):
    R, t = pose[:9].reshape(3, 3), pose[9:]
    return ((R[:, 0] * b[:, [0]] + R[:, 1] * b[:, [1]]) + R[:, 2] * b[:, [2]]) + t


def quantise(w, vs):
    loc = (w / vs).astype(np.float32)
    loc = np.where(loc < 0, loc - np.float32(1), loc)
    return np.trunc(loc).astype(np.int64)


def split_centres(k, vs, depth, w):
    """centres of the nodes a world point passes on its way down from root cell k (voxel_map.hpp:1029-1040, 1530-1533)"""
    c = (0.5 + k.astype(np.float64)) * vs
    q = np.float32(vs / 4.0)
    out = []
    for _ in range(depth):
        out.append(c.copy())
        b = w > c
        c = c + (np.where(b, np.float32(1), np.float32(-1)) * q).astype(np.float32).astype(np.float64)
        q = np.float32(q / np.float32(2))
    return out


def octant_bits(w, vs, depth):
    k = quantise(w, vs)
    cs = split_centres(k, vs, depth, w)
    return np.stack([(w > c) @ np.array([4, 2, 1]) for c in cs], axis=1) if depth else np.zeros((len(w), 0), dtype=np.int64)


def range_gate(w, centre, normal, radius):
    """voxel_map.hpp:1340-1344 in float: |n.d|, d.d, d.d - |n.d|^2 <= 9 radius"""
    d = w - centre
    nd = (normal[:, 0] * d[:, 0] + normal[:, 1] * d[:, 1]) + normal[:, 2] * d[:, 2]
    dtp = np.abs(nd).astype(np.float32)
    dtc = ((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]).astype(np.float32)
    return (dtc - dtp * dtp) <= np.float32(9) * radius.astype(np.float32)


def body_of(pose, w):
    R, t = pose[:9].reshape(3, 3), pose[9:]
    return (w - t) @ R


def records(b, var):
    return np.concatenate([b, var.reshape(-1, 9)], axis=1)


# ---------------------------------------------------------------- the two oracle maps
class Scene:
    def __init__(self, path, name):
        self.path, self.name = path, name
        self.vs, self.ml = SCENES[name]
        self.mp = vx.MapParams.make(voxel_size=self.vs, max_layer=self.ml)
        if path == "table":
            tr, _ = scenes.poses_true_est(4, L, 5)
            pts, off = scenes.make_points(4, 6000, L, 5, tr)
            tr[:, 9:] += SHIFT
            self.lm = oa.LocalMap(self.mp, pts, off, tr, 1e-4, mgsize=1)
            P = self.lm.planes()
            self.leaf_state = None
        else:
            self.Wn, self.scans, self.x = 4, [], []
            self.sim = oa.SlidingSim(self.mp, self.Wn, 1, max_points=100)
            for i in range(self.Wn + 4):
                pose = synth.true_pose(L, i)
                est = synth.perturb_pose(pose, 700 + i, 1e-3, 5e-3) if i else pose.copy()
                est[9:] += SHIFT
                pv = pv_records(synth.gen_scan(L, i, 4000, pose, seed=0x5EED0000 + 61), 500 + i, True)
                self.scans.append(pv); self.x.append(est)
                self.sim.add_scan_pv(pv, est)
            P = self.sim.planes()
            self.leaf_state = self.sim.state()
        self.P = P
        self.P["layer"] = np.rint(np.log2(self.vs / (2.0 * P["half"]))).astype(np.int32)
        self.P["root"] = quantise(P["voxel_center"], self.vs)

    def oracle(self, pv, pose, rv, tv):
        if self.path == "table":
            return self.lm.odom_accumulate(pv, pose, rv, tv)
        return self.sim.odom_accumulate(pv, pose, rv, tv)

    def flags(self, b, var, pose, rv, tv):
        return self.oracle(records(b, var), pose, rv, tv)["flags"]


_SCENES = {}


def scene(path, name):
    if (path, name) not in _SCENES:
        _SCENES[(path, name)] = Scene(path, name)
    return _SCENES[(path, name)]


# ---------------------------------------------------------------- gate pairs
def _bisect_pairs(fl, b0, u, s_hi):
    """fl(b) -> oracle flags.  fl(b0) == 1, fl(b0 + s_hi u) == 0.  Returns (inside, outside): equal but for one coordinate, one ulp
    apart there, fl(inside) == 1, fl(outside) == 0."""
    lo, hi = np.zeros(len(b0)), s_hi.copy()
    for _ in range(1100):
        mid = 0.5 * (lo + hi)
        live = (mid != lo) & (mid != hi)
        if not live.any():
            break
        f = fl(b0 + mid[:, None] * u)
        lo = np.where(live & (f == 1), mid, lo)
        hi = np.where(live & (f == 0), mid, hi)
    A, B = b0 + lo[:, None] * u, b0 + hi[:, None] * u
    # walk from A to B one coordinate at a time: some step flips the flag and changes one coordinate only
    P = [A.copy()]
    for j in range(3):
        q = P[-1].copy(); q[:, j] = B[:, j]; P.append(q)
    F = np.stack([fl(p) for p in P], axis=1)
    j = np.argmax(F[:, :3] != F[:, 1:], axis=1)
    rows = np.arange(len(A))
    p0, p1 = np.stack(P, axis=1)[rows, j], np.stack(P, axis=1)[rows, j + 1]
    first_in = F[rows, j] == 1
    inside, outside = np.where(first_in[:, None], p0, p1), np.where(first_in[:, None], p1, p0)
    lo_v, hi_v = inside[rows, j].copy(), outside[rows, j].copy()
    for _ in range(80):
        adj = np.nextafter(lo_v, hi_v) == hi_v
        if adj.all():
            break
        mid = np.where(adj, lo_v, lo_v + 0.5 * (hi_v - lo_v))
        q = inside.copy(); q[rows, j] = mid
        f = fl(q)
        lo_v = np.where(~adj & (f == 1), mid, lo_v)
        hi_v = np.where(~adj & (f == 0), mid, hi_v)
    inside[rows, j], outside[rows, j] = lo_v, hi_v
    return inside, outside


def _cube_exit(w0, d, vc, half):
    """distance along unit d from w0 to the boundary of the cube vc +- half"""
    with np.errstate(divide="ignore", invalid="ignore"):
        t = np.where(d > 0, (vc + half[:, None] - w0) / d, np.where(d < 0, (vc - half[:, None] - w0) / d, np.inf))
    return np.min(t, axis=1)


def gate_pairs(sc, pose, seed):
    """For every plane leaf: a pair straddling the 3-sigma gate (moved along the normal from near the plane centre) and, where the leaf's
    cube allows it, a pair straddling range_dis <= 9 radius (moved in the plane from its centre).  Each plane gets its own point covariance
    and one of COV_GROUPS' rot_var / tsl_var (zero matrices included).  Returns a list of dicts, one per covariance group."""
    P = sc.P
    n = len(P["radius"])
    rng = np.random.default_rng(seed)
    var = np.stack([_rng_spd(rng, 10 ** rng.uniform(-3, -1.5)) + np.eye(3) * 1e-6 for _ in range(n)])
    grp = np.arange(n) % len(COV_GROUPS)
    c, nr, vc, half = P["center"], P["normal"], P["voxel_center"], P["half"]
    # normal direction: start a little off the centre in the plane, walk along +-n
    a = np.cross(nr, rng.standard_normal((n, 3))); a /= np.linalg.norm(a, axis=1, keepdims=True)
    w_n = c + 0.1 * half[:, None] * a
    d_n = nr * np.where(rng.uniform(size=n) < 0.5, -1.0, 1.0)[:, None]
    # in-plane direction: towards the farthest corner of the leaf cube, projected onto the plane
    corners = vc[:, None, :] + half[:, None, None] * np.array([[i, j, k] for i in (-1, 1) for j in (-1, 1) for k in (-1, 1)])[None]
    rel = corners - c[:, None, :]
    rel = rel - np.sum(rel * nr[:, None, :], axis=2, keepdims=True) * nr[:, None, :]
    t = rel[np.arange(n), np.argmax(np.linalg.norm(rel, axis=2), axis=1)]
    t /= np.maximum(np.linalg.norm(t, axis=1, keepdims=True), 1e-300)
    R = pose[:9].reshape(3, 3)
    out = []
    for g, (rv, tv) in enumerate(COV_GROUPS):
        ins, outs, plane = [], [], []
        for w0, d in ((w_n, d_n), (c, t)):
            m = grp == g
            s_hi = 0.999 * _cube_exit(w0[m], d[m], vc[m], half[m])
            b0, u = body_of(pose, w0[m]), d[m] @ R
            fl = lambda b, vv=var[m]: sc.flags(b, vv, pose, rv, tv)          # noqa: E731
            ok = np.isfinite(s_hi) & (fl(b0) == 1) & (fl(b0 + s_hi[:, None] * u) == 0)
            sel = np.flatnonzero(m)[ok]
            if len(sel) == 0:
                continue
            fl = lambda b, vv=var[sel]: sc.flags(b, vv, pose, rv, tv)        # noqa: E731
            i_, o_ = _bisect_pairs(fl, b0[ok], u[ok], s_hi[ok])
            ins.append(i_); outs.append(o_); plane.append(sel)
        plane = np.concatenate(plane)
        ins, outs = np.concatenate(ins), np.concatenate(outs)
        ci, no, ra = c[plane], nr[plane], P["radius"][plane]
        by_range = range_gate(world(pose, ins), ci, no, ra) & ~range_gate(world(pose, outs), ci, no, ra)
        out.append(dict(rv=rv, tv=tv, inside=ins, outside=outs, var=var[plane], by_range=by_range))
    return out


def interleave(a, b):
    x = np.empty((2 * len(a),) + a.shape[1:], dtype=a.dtype)
    x[0::2], x[1::2] = a, b
    return x


# ---------------------------------------------------------------- face and miss points (identity pose, world == body)
def face_points(sc):
    """world points (identity pose) -> (points, labels).  Root-cell faces at k vs and one ulp either side, values whose float(w / vs) rounds
    onto an integer, -0.0, octant faces (each node centre on the way down to every plane leaf of layer >= 1, per axis and on all axes
    at once, and one ulp either side).  Each point starts at a plane centre, so most of them are in reach of a plane."""
    P, vs = sc.P, sc.vs
    c, nr, layer = P["center"], P["normal"], P["layer"]
    pts, lab = [], []
    inf = np.inf
    for i in range(len(c)):
        axes = [a for a in range(3) if abs(nr[i, a]) < 0.5]
        for a in axes:
            k0 = int(np.floor(c[i, a] / vs))
            for k in (k0, k0 + 1):
                f = k * vs
                vals = [(np.nextafter(f, -inf), "face-"), (f, "face0"), (np.nextafter(f, inf), "face+")]
                if k != 0:
                    vals += [((k - 1e-9) * vs, "round-up"), ((k + 1e-9) * vs, "round-down")]
                for v, tag in vals:
                    p = c[i].copy(); p[a] = v; pts.append(p); lab.append(tag)
        if layer[i] >= 1:
            k = quantise(c[i:i + 1], vs)
            for depth, cen in enumerate(split_centres(k, vs, int(layer[i]), c[i:i + 1]), start=1):
                cen = cen[0]
                for a in range(3):
                    for v, s in ((np.nextafter(cen[a], -inf), "-"), (cen[a], "0"), (np.nextafter(cen[a], inf), "+")):
                        p = c[i].copy(); p[a] = v; pts.append(p); lab.append(f"octant{depth}{s}")
                for v, s in ((np.nextafter(cen, -inf), "-"), (cen, "0"), (np.nextafter(cen, inf), "+")):
                    pts.append(v.copy()); lab.append(f"octant{depth}{s}")
    for y in (-0.0, -1.5 * vs, 2.5 * vs):
        pts.append(np.array([-0.0, y, -0.0])); lab.append("zero")
    return np.array(pts), np.array(lab)


def miss_points(sc):
    """world points (identity pose) that cannot match: a root cell with no plane under it, an octant with no plane leaf under it (on the
    resident path: the oracle's missing children and non-plane leaves), just outside the plane table's bounding box on each side."""
    P, vs = sc.P, sc.vs
    root = P["root"]
    pts, lab = [], []
    roots = {tuple(r) for r in root}
    mn, mx = root.min(0), root.max(0)
    rng = np.random.default_rng(5)
    for _ in range(4000):
        k = rng.integers(mn, mx + 1)
        if tuple(k) not in roots:
            pts.append((k + rng.uniform(0.05, 0.95, 3)) * vs); lab.append("no-root")
            if sum(l_ == "no-root" for l_ in lab) >= 40:
                break
    if sc.ml >= 1:
        # octants of planed roots whose layer-1 subtree holds no plane leaf
        for r in sorted(roots)[:200]:
            r = np.array(r)
            sub = (root == r).all(1)
            if (P["layer"][sub] == 0).any():
                continue
            have = {tuple(o) for o in octant_bits(P["voxel_center"][sub], vs, 1)[:, 0:1]}
            c0 = (0.5 + r) * vs
            for o in range(8):
                if (o,) in have:
                    continue
                b = np.array([(o >> 2) & 1, (o >> 1) & 1, o & 1])
                pts.append(c0 + (2 * b - 1) * vs / 4); lab.append("no-child")
    if sc.leaf_state is not None:
        s = sc.leaf_state
        for i in np.flatnonzero(~s["is_plane"])[:60]:
            pts.append(s["voxel_center"][i] + 0.3 * s["half"][i]); lab.append("non-plane")
    # the plane table's bounding box, each side, from the plane centre nearest to that side: its face, one ulp either side, 0.3 cells either side
    bb = []
    for a in range(3):
        for side, kk in ((-1, mn[a]), (1, mx[a] + 1)):
            i = np.argmin(P["center"][:, a]) if side < 0 else np.argmax(P["center"][:, a])
            f = kk * vs
            for v in (f, np.nextafter(f, -np.inf), np.nextafter(f, np.inf), f - 0.3 * vs, f + 0.3 * vs):
                p = P["center"][i].copy(); p[a] = v; bb.append(p)
    bb = np.array(bb)
    q = quantise(bb, vs)
    inside = np.all((q >= mn) & (q <= mx), axis=1)
    pts += list(bb); lab += ["bbox-in" if t else "bbox-out" for t in inside]
    return np.array(pts), np.array(lab)


def point_var(n, seed):
    rng = np.random.default_rng(seed)
    A = rng.standard_normal((n, 3, 3)) * 0.01
    return A @ np.transpose(A, (0, 2, 1)) + np.eye(3) * 1e-5


# ---------------------------------------------------------------- checks
def check(g, o, tol=1e-9):
    assert g["n"] == o["n"], (g["n"], o["n"])
    assert np.array_equal(g["flags"], o["flags"]), np.flatnonzero(g["flags"] != o["flags"])[:20]
    for k in ("HTH", "HTz", "nnt"):
        assert np.max(np.abs(g[k] - o[k])) <= tol * max(np.max(np.abs(o[k])), 1e-300), k


class Device:
    """one of the two device paths, holding the same map as the scene's oracle"""

    def __init__(self, ctx, sc):
        self.ctx, self.sc = ctx, sc
        if sc.path == "table":
            self.load_table()
        else:
            self.dm = vx.LocalMap(ctx, sc.mp, sc.Wn, max_points=100)
            f = vx.Factor(ctx, sc.Wn)
            x = []
            for pv, est in zip(sc.scans, sc.x):
                x.append(est)
                self.dm.push_scan(pv, np.stack(x), f)
                if len(x) >= sc.Wn:
                    self.dm.margi(np.stack(x), f, mgsize=1)
                    x = x[1:]
            f.close()
            compare_leaves(self.dm.leaves(), sc.leaf_state, sc.name)

    def load_table(self):
        P = self.sc.P
        self.ctx.odom_set_planes(self.sc.mp, P["voxel_center"], P["layer"], P["center"], P["normal"], P["plane_var"], P["radius"])

    def __call__(self, pv, pose, rv, tv, n=None, want_flags=True):
        if self.sc.path == "table":
            return self.ctx.odom_accumulate(pv, pose, rv, tv, n=n, want_flags=want_flags)
        return self.dm.odom_accumulate(pv, pose, rv, tv, n=n, want_flags=want_flags)

    def close(self):
        if self.sc.path == "resident":
            self.dm.close()


PATHS = ("table", "resident")


# ---------------------------------------------------------------- CPU: the generator does what it claims
@pytest.mark.parametrize("path", PATHS)
def test_edge_generator(path):
    """every gate pair straddles the oracle's decision one ulp apart in one coordinate, inside one leaf; every face point is where it is meant to be"""
    n_range = n_normal = 0
    for name in SCENES:
        sc = scene(path, name)
        for pose, seed in ((IDENT, 1), (POSE_B, 2)) if path == "table" else ():
            for G in gate_pairs(sc, pose, seed):
                i_, o_ = G["inside"], G["outside"]
                diff = i_ != o_
                assert np.all(diff.sum(1) == 1)
                assert np.all(np.nextafter(i_[diff], o_[diff]) == o_[diff])
                f = sc.oracle(records(interleave(i_, o_), interleave(G["var"], G["var"])), pose, G["rv"], G["tv"])["flags"]
                assert np.array_equal(f, np.tile([1, 0], len(i_)))
                wi, wo = world(pose, i_), world(pose, o_)
                assert np.array_equal(quantise(wi, sc.vs), quantise(wo, sc.vs))
                assert np.array_equal(octant_bits(wi, sc.vs, sc.ml), octant_bits(wo, sc.vs, sc.ml))
                n_range += int(G["by_range"].sum()); n_normal += int((~G["by_range"]).sum())
        w, lab = face_points(sc)
        assert np.array_equal(world(IDENT, w), w)
        q, fl, r = quantise(w, sc.vs), (w / sc.vs).astype(np.float32), w / sc.vs
        # root-cell faces: (face-, face0, face+) triples one ulp apart around k vs; the quantisation of each is the reference's
        m = np.flatnonzero(lab == "face0")
        ax = np.argmax(w[m - 1] != w[m + 1], axis=1)
        v0, vm, vp = w[m, ax], w[m - 1, ax], w[m + 1, ax]
        k = np.rint(v0 / sc.vs)
        assert np.all(v0 == k * sc.vs) and np.all(np.nextafter(v0, -np.inf) == vm) and np.all(np.nextafter(v0, np.inf) == vp)
        assert (k < 0).any() and (k > 0).any()
        assert np.all(q[m, ax] == np.where(fl[m, ax] < 0, np.floor(fl[m, ax]) - 1, np.floor(fl[m, ax])))
        # float(w / vs) lands on an integer while w / vs is not one: the quantisation differs from floor(w / vs)
        for tag in ("round-up", "round-down"):
            i_, a_ = np.nonzero((lab == tag)[:, None] & (np.abs(r - np.rint(r)) > 0) & (np.abs(r - np.rint(r)) < 1e-8))
            assert len(i_) > 0 and np.all(fl[i_, a_] == np.rint(fl[i_, a_]))
        assert ((lab == "round-up")[:, None] & (q != np.floor(r))).any() and ((lab == "round-down")[:, None] & (q != np.floor(r))).any()
        assert np.any(np.signbit(world(IDENT, w[lab == "zero"])[:, 0]))
        # octant faces: the node centre and its lower neighbour go to the lower octant at that depth, the upper neighbour to the upper one
        for d in range(1, sc.ml + 1):
            m = np.flatnonzero(lab == f"octant{d}0")
            if (sc.P["layer"] >= d).any():
                assert len(m) > 0, d
            if len(m):
                bm, b0, bp = (octant_bits(w[m + s], sc.vs, d)[:, d - 1] for s in (-1, 0, 1))
                assert np.array_equal(bm, b0) and np.all(bp != b0) and np.all((bp & ~b0) == bp - b0), d
        wm, lm_ = miss_points(sc)
        f = sc.oracle(records(wm, point_var(len(wm), 3)), IDENT, *COV_GROUPS[3])["flags"]
        assert not f[lm_ != "bbox-in"].any()
        assert (lm_ == "no-root").sum() > 0 and (lm_ == "bbox-out").sum() >= 6 and (lm_ == "bbox-in").sum() >= 6
    assert path == "resident" or (n_normal > 400 and n_range > 40), (n_normal, n_range)
    layers = np.concatenate([scene(path, nm).P["layer"] for nm in SCENES])
    assert {0, 1, 2} <= set(layers.tolist())


# ---------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def ctx():
    c = vx.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def device(ctx):
    made = {}

    def get(path, name):
        if (path, name) not in made:
            made[(path, name)] = Device(ctx, scene(path, name))
        d = made[(path, name)]
        if path == "table":
            d.load_table()           # the ctx holds one plane table at a time
        return d
    yield get
    for d in made.values():
        d.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(SCENES))
def test_gate_pairs(device, name):
    sc, dev = scene("table", name), device("table", name)
    for pose, seed in ((IDENT, 1), (POSE_B, 2)):
        for G in gate_pairs(sc, pose, seed):
            pv = records(interleave(G["inside"], G["outside"]), interleave(G["var"], G["var"]))
            o = sc.oracle(pv, pose, G["rv"], G["tv"])
            assert o["n"] == len(G["inside"])
            check(dev(pv, pose, G["rv"], G["tv"]), o)


@pytest.mark.gpu
def test_gate_pairs_negative_control(device):
    """the flag check sees a one-ulp shift across the gate: the device fed every pair swapped fails it"""
    sc, dev = scene("table", "vs1_l2"), device("table", "vs1_l2")
    G = gate_pairs(sc, POSE_B, 2)[3]
    pv = records(interleave(G["inside"], G["outside"]), interleave(G["var"], G["var"]))
    sw = records(interleave(G["outside"], G["inside"]), interleave(G["var"], G["var"]))
    o = sc.oracle(pv, POSE_B, G["rv"], G["tv"])
    check(dev(pv, POSE_B, G["rv"], G["tv"]), o)
    with pytest.raises(AssertionError):
        check(dev(sw, POSE_B, G["rv"], G["tv"]), o)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(SCENES))
@pytest.mark.parametrize("path", PATHS)
def test_faces_and_misses(device, path, name):
    sc, dev = scene(path, name), device(path, name)
    w, lab = face_points(sc)
    wm, lm_ = miss_points(sc)
    for k, (rv, tv) in enumerate(COV_GROUPS[:3]):
        pv = records(w, point_var(len(w), 10 + k))
        o = sc.oracle(pv, IDENT, rv, tv)
        assert o["n"] > len(w) // 10
        check(dev(pv, IDENT, rv, tv), o)
        pm = records(wm, point_var(len(wm), 20 + k))
        om = sc.oracle(pm, IDENT, rv, tv)
        assert not om["flags"][lm_ != "bbox-in"].any()
        check(dev(pm, IDENT, rv, tv), om)


def _mixed(sc):
    """face points, led on the exported-table path by gate pairs (see the module docstring)"""
    w, _ = face_points(sc)
    b = body_of(POSE_B, w)
    if sc.path == "table":
        G = gate_pairs(sc, POSE_B, 2)[3]
        b = np.concatenate([interleave(G["inside"], G["outside"]), b])
    return records(b, point_var(len(b), 4)), COV_GROUPS[3][0], COV_GROUPS[3][1]


@pytest.mark.gpu
@pytest.mark.parametrize("path", PATHS)
def test_launch_shapes(device, path):
    """n = 0, 1 and partial warps / blocks around 32 and 256 (od_flush); want_flags=False gives the same sums; the resident scan re-used"""
    sc, dev = scene(path, "vs1_l2"), device(path, "vs1_l2")
    pv, rv, tv = _mixed(sc)
    assert len(pv) > 257
    for n in (0, 1, 31, 33, 255, 257):
        o = sc.oracle(pv[:n], POSE_B, rv, tv)
        g = dev(pv[:n], POSE_B, rv, tv)
        check(g, o)
        assert n < 255 or o["n"] > 30
        h = dev(None, POSE_B, rv, tv, n=n, want_flags=False)
        assert h["flags"] is None and h["n"] == g["n"]
        for k in ("HTH", "HTz", "nnt"):
            assert np.max(np.abs(h[k] - g[k])) <= 1e-12 * max(np.max(np.abs(g[k])), 1e-300), (n, k)


@pytest.mark.gpu
def test_resident_scan_after_the_table_is_replaced(ctx, device):
    """odom_accumulate(pv12=None) after odom_set_planes has swapped the plane table: the kept scan meets the new table"""
    a, b = scene("table", "vs1_l2"), scene("table", "vs05_l2")
    pv, rv, tv = _mixed(a)
    device("table", "vs1_l2")
    check(ctx.odom_accumulate(pv, POSE_B, rv, tv), a.oracle(pv, POSE_B, rv, tv))
    device("table", "vs05_l2")
    o = b.oracle(pv, POSE_B, rv, tv)
    assert o["n"] > 50
    check(ctx.odom_accumulate(None, POSE_B, rv, tv, n=len(pv)), o)


# ---------------------------------------------------------------- var_init with real extrinsics
EXTRINSICS = [(oa.so3_exp(np.array([0.02, -0.01, 0.03])), np.array([0.05, -0.02, 0.1])),
              (oa.so3_exp(np.array([0.013, -0.021, np.pi / 2 + 0.004])), np.array([-0.31, 0.12, 0.043])),
              (oa.so3_exp(np.array([0.7, -0.4, 0.25])), np.array([0.0131, 0.271, -0.193]))]


def lidar_scan(i, n, ext_R, ext_p):
    """a scan of the room in the sensor frame: body points taken back through the extrinsic, as float32 (what var_init reads)"""
    body = synth.gen_scan(L, i, n, synth.true_pose(L, i), seed=0x5EED0000 + 83)
    return ((body - ext_p) @ ext_R).astype(np.float32)


@pytest.mark.gpu
@pytest.mark.parametrize("e", range(len(EXTRINSICS)))
def test_var_init_points_bit_exact(ctx, e):
    ext_R, ext_p = EXTRINSICS[e]
    rng = np.random.default_rng(30 + e)
    pts = rng.uniform(-60, 60, (20000, 3)).astype(np.float32)
    pts[0] = (3.0, -2.0, 0.0)
    pts = np.concatenate([pts, lidar_scan(0, 5000, ext_R, ext_p)])
    g, o = ctx.var_init(pts, ext_R, ext_p, 0.02, 0.05), oa.var_init(pts, ext_R, ext_p, 0.02, 0.05)
    assert np.array_equal(g[:, :3], o[:, :3])
    assert np.max(np.abs(g[:, 3:] - o[:, 3:]) / np.max(np.abs(o[:, 3:]), axis=1, keepdims=True)) < 1e-11
    # negative control: one entry of the extrinsic one ulp off moves points
    bad = ext_R.copy(); bad[1, 2] = np.nextafter(bad[1, 2], np.inf)
    with pytest.raises(AssertionError):
        assert np.array_equal(ctx.var_init(pts, bad, ext_p, 0.02, 0.05)[:, :3], o[:, :3])


def _handover(ctx, ext_R, ext_p, from_oracle):
    """var_init -> pvec_update(None) -> push_scan(None) per scan, margi when full, then var_init -> map_odom_accumulate(None)"""
    Wn, n = 4, 3000
    mp = vx.MapParams.make(voxel_size=1.0, max_layer=2)
    dm, f = vx.LocalMap(ctx, mp, Wn), vx.Factor(ctx, Wn)
    rv, tv = np.eye(3) * 1e-6, np.eye(3) * 1e-4
    x = []
    try:
        for i in range(Wn + 3):
            pose = synth.true_pose(L, i)
            cloud = lidar_scan(i, n, ext_R, ext_p)
            x.append(pose)
            if from_oracle:
                ctx.pvec_update(oa.var_init(cloud, ext_R, ext_p, 0.02, 0.05), pose, rv, tv, want_pv=False, want_pwld=False)
            else:
                ctx.var_init(cloud, ext_R, ext_p, 0.02, 0.05, want_out=False)
                ctx.pvec_update(None, pose, rv, tv, n=n, want_pv=False, want_pwld=False)
            dm.push_scan(None, np.stack(x), f, n=n)
            if len(x) >= Wn:
                dm.margi(np.stack(x), f, mgsize=1)
                x = x[1:]
        cloud = lidar_scan(Wn + 3, 8000, ext_R, ext_p)
        pose = synth.perturb_pose(synth.true_pose(L, Wn + 3), 17, 1e-3, 5e-3)
        if from_oracle:
            od = dm.odom_accumulate(oa.var_init(cloud, ext_R, ext_p, 0.02, 0.05), pose, rv, tv)
        else:
            ctx.var_init(cloud, ext_R, ext_p, 0.02, 0.05, want_out=False)
            od = dm.odom_accumulate(None, pose, rv, tv, n=len(cloud))
        return dm.leaves(), od
    finally:
        dm.close(); f.close()


@pytest.mark.gpu
@pytest.mark.parametrize("e", [1, 2])
def test_var_init_handover_to_the_map(ctx, e):
    """the device hand-over from var_init into the resident map equals the same calls fed with the oracle's var_init output"""
    ext_R, ext_p = EXTRINSICS[e]
    a, oa_ = _handover(ctx, ext_R, ext_p, False)
    b, ob = _handover(ctx, ext_R, ext_p, True)
    ka = np.lexsort(np.concatenate([np.round(a["voxel_center"], 9), a["layer"][:, None]], axis=1).T)
    kb = np.lexsort(np.concatenate([np.round(b["voxel_center"], 9), b["layer"][:, None]], axis=1).T)
    assert len(ka) == len(kb) > 50
    for k in ("voxel_center", "layer", "is_plane", "pcr_add", "slots"):
        assert np.array_equal(a[k][ka], b[k][kb]), k
    assert ob["n"] > 1000
    check(oa_, ob)
