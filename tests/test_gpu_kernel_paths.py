"""Every Hessian, residual and LDL^T kernel path at its dispatch boundaries and in its A/B forms, CUDA vs the CPU oracle.

The host drivers pick kernels by shape (vxs_eval_hessian_dev, vxs_residual_stream_launch, vxs_solve_damped) and the context picks the SYRK
and LDL^T A/B forms from VXS_* environment variables at creation.  Each case here names its shape and switch in its id, checks with the kernel timers that the
intended kernel ran, and compares with the oracle (the as-written restatement of the reference) at the existing parity tolerances.

Factors of an exact shape are cut from one small synthetic window instead of big map builds: its fully observed voxels are replicated over
voxels and frames (replica frames get slightly perturbed poses), and the cached eigen-decomposition / point sums are recomputed by the oracle at
those poses so the factor is self-consistent.  Voxels with no entry at all are accepted by the oracle's push and are included in the Hessian
cases (the dense Jacobian kernels zero their rows explicitly); the residual of such a voxel is undefined without a fix cluster, so the residual
cases keep every voxel observed."""
import functools

import numpy as np
import pytest

import oracle_api as oa
import scenes
import synth
import voxel_slam_b200 as vx

pytestmark = pytest.mark.gpu

VXS_VARS = ("VXS_SYRK_WAVES", "VXS_LDLT_LOOKAHEAD_CTA", "VXS_HBA_ROUTE")

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
    with pytest.MonkeyPatch.context() as mp:      # the default forms, whatever the caller's environment holds
        for k in VXS_VARS:
            mp.delenv(k, raising=False)
        c = vx.Context(0)
    c.timing(True)
    yield c
    c.close()


@pytest.fixture
def env_ctx(monkeypatch):
    """env_ctx(VXS_X="1", ...) -> a fresh context created with exactly these VXS_* variables set; closed at teardown."""
    made = []

    def make(**env):
        for k in VXS_VARS:
            monkeypatch.delenv(k, raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, str(v))
        c = vx.Context(0)
        c.timing(True)
        made.append(c)
        return c

    yield make
    for c in made:
        c.close()


@functools.lru_cache(maxsize=None)
def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def ran_kernels(ctx):
    return {name for name, (_, calls) in ctx.timing_read().items() if calls > 0}


def relinf(a, b):
    return float(np.max(np.abs(np.asarray(a) - np.asarray(b))) / max(np.max(np.abs(b)), 1e-300))


# ------------------------------------------------------------------------------------------------ factors of an exact shape
@functools.lru_cache(maxsize=None)
def _base():
    sc = scenes.make_window(W=8, pts_per_scan=4000, L=6.0, seed=5)
    full = np.all(sc["clusters10"][:, :, 9] > 0, axis=1)
    assert full.sum() >= 100
    return sc["clusters10"][full], sc["poses_est"]


def window_poses(W, seed):
    """frame j reuses the body-frame clusters of base frame j % 8; replicas sit at slightly perturbed poses"""
    _, est = _base()
    return np.stack([est[j] if j < 8 else synth.perturb_pose(est[j % 8], 100003 * seed + j, 2e-3, 1e-2) for j in range(W)])


@functools.lru_cache(maxsize=None)
def case(W, V, obs="dense", seed=0, fix=True, coe=True, single=2, empty=1, k=0, stride=0, short=0):
    """Dense [V][W][10] factor arrays.  obs: which (voxel, frame) slots hold an entry
         dense   each slot with probability 0.7        full    every slot
         k       exactly k random slots per voxel        stride  slots 0, stride, 2 stride, ...
         mixed   first half of the voxels full, the rest strided
       then: `single` voxels observed by exactly one frame, `short` voxels lose one entry, `empty` voxels lose all entries (after the
       cache was computed, so their cached sums stay valid).  fix: a world-frame fix cluster on every third voxel; coe: random positive."""
    cl0, _ = _base()
    rng = np.random.default_rng(1000003 * seed + 1009 * W + V)
    if obs == "dense":
        m = rng.random((V, W)) < 0.7
    elif obs == "full":
        m = np.ones((V, W), bool)
    elif obs == "k":
        m = np.zeros((V, W), bool)
        for v in range(V):
            m[v, rng.choice(W, k, replace=False)] = True
    elif obs == "stride":
        m = np.zeros((V, W), bool)
        m[:, ::stride] = True
    elif obs == "mixed":
        m = np.zeros((V, W), bool)
        m[: V // 2] = True
        m[V // 2:, ::stride] = True
    else:
        raise ValueError(obs)
    for v in np.flatnonzero(~m.any(axis=1)):
        m[v, rng.integers(W)] = True
    for v in range(1, 1 + single if V > single + 1 else 1):
        m[v] = False
        m[v, rng.integers(W)] = True
    for v in range(V - short, V):
        m[v, rng.choice(np.flatnonzero(m[v]))] = False
    src = (np.arange(V) * 37 + seed) % cl0.shape[0]
    poses = window_poses(W, seed)
    cl = np.where(m[:, :, None], cl0[src][:, np.arange(W) % 8, :], 0.0)
    # A voxel seen by one frame only and without fixed points is invariant to that frame's pose: its Hessian terms cancel to rounding noise
    # of the as-written formula (two evaluation orders of the same block disagree at O(1) of its ~1e-16 scale), so such voxels carry a fix.
    # The fixed points are base frame 1's scan at its own estimated pose, so they never coincide with a window frame's points.
    lone = m.sum(axis=1) == 1
    assert fix or not lone.any()
    fix10 = None
    if fix:
        fix10 = np.zeros((V, 10))
        for v in np.flatnonzero((np.arange(V) % 3 == 0) | lone):
            fix10[v] = oa.cluster_transform(cl0[src[v], 1], _base()[1][1])
    co = rng.uniform(0.5, 2.0, V) if coe else None
    of = oa.OracleFactor.from_dense(W, cl, fix10, co, np.zeros((V, 12)), np.zeros((V, 10)))
    of.residual(poses)                                  # the cache (eig, pcr_add) the map build would leave at these poses
    ex = of.export()
    if empty and V >= 8:
        m[V // 2: V // 2 + empty] = False
        cl[V // 2: V // 2 + empty] = 0.0
    assert m.any(axis=1).sum() >= V - empty
    return dict(W=W, V=V, cl=cl, fix=fix10, coe=co, eig=ex["eig12"], sum=ex["sum10"], poses=poses, obs=m,
                key=(W, V, obs, seed, fix, coe, single, empty, k, stride, short))


def oracle_factor(c, cl=None):
    return oa.OracleFactor.from_dense(c["W"], c["cl"] if cl is None else cl, c["fix"], c["coe"], c["eig"], c["sum"])


def push(f, c, cl=None):
    f.push_voxels_dense(c["cl"] if cl is None else cl, c["eig"], c["sum"], fix10=c["fix"], coe=c["coe"])


def to_csr(c):
    m = c["obs"]
    ptr = np.concatenate([[0], np.cumsum(m.sum(axis=1))]).astype(np.int64)
    v, fr = np.nonzero(m)                                  # row-major: voxel by voxel, frames ascending
    return ptr, fr.astype(np.int32), c["cl"][v, fr]


_HREF = {}


def hessian_ref(c):
    if c["key"] not in _HREF:
        _HREF[c["key"]] = oracle_factor(c).hessian(c["poses"])
    return _HREF[c["key"]]


def hessian_on_reused_factor(ctx, c, async_push=False, cl=None):
    """Evaluate on a Factor whose workspaces first held a different, fully observed factor of the same W (more voxels): a zero-fill that
    misses a slot or a padding row then shows up as stale data instead of as fresh zeroed memory."""
    W = c["W"]
    f = vx.Factor(ctx, W)
    prime = case(W, c["V"] + 5, "full", seed=c["key"][3] + 77, single=0, empty=0)
    push(f, prime)
    ctx.evaluate_hessian(f, prime["poses"])
    f.clear()
    if async_push:
        ptr, fr, ent = to_csr(c)
        f.push_voxels_async(ptr, fr, ent, c["eig"], c["sum"], fix10=c["fix"], coe=c["coe"])
    else:
        push(f, c, cl)
    ctx.timing_reset()
    out = ctx.evaluate_hessian(f, c["poses"])
    ran = ran_kernels(ctx)
    f.close()
    return out, ran


def is_dense(c):
    V, W, E = c["V"], c["W"], int(c["obs"].sum())
    return V * W <= 4 * E


def pick_group(E, V):             # vxs_eval.cu pick_group: k_pairs<G>
    avg = E / V
    return 32 if avg > 16 else (16 if avg > 8 else 8)


def pick_group_jac(E, V, W):      # vxs_eval.cu pick_group_jac: k_jac<G, .>
    avg = E / V
    return 64 if (avg > 24 and W > 32) else pick_group(E, V)


def check_path(ran, c):
    assert "k_jac" in ran and "k_lambda_sum" in ran, ran
    if is_dense(c):
        assert "k_syrk" in ran and "k_pairs" not in ran, ran
    else:
        assert "k_pairs" in ran and "k_syrk" not in ran, ran


def check_hessian(got, ref, obs):
    """H, J, r against the oracle: relinf < 1e-9 (r 1e-12), every non-zero 6x6 block to 1e-7 of its own scale, blocks of frame pairs that
    share no voxel exactly zero, and H symmetric bit for bit outside the 6x6 diagonal blocks.  The diagonal blocks are not symmetric in the
    reference either: their rotation part carries -0.5 hat(J_rot) (voxel_map.hpp acc_evaluate2), and the oracle keeps that form."""
    H, J, r = got
    Hr, Jr, rr = ref
    W = obs.shape[1]
    offdiag = ~np.kron(np.eye(W, dtype=bool), np.ones((6, 6), dtype=bool))
    assert np.array_equal(H[offdiag], H.T[offdiag]), "H is not bitwise symmetric outside the diagonal blocks"
    er, ej, eh = abs(r - rr) / abs(rr), relinf(J, Jr), relinf(H, Hr)
    assert er < 1e-12, er
    assert ej < 1e-9, ej
    assert eh < 1e-9, eh
    Hb, Hrb = H.reshape(W, 6, W, 6), Hr.reshape(W, 6, W, 6)
    scale = np.max(np.abs(Hrb), axis=(1, 3))
    err = np.max(np.abs(Hb - Hrb), axis=(1, 3))
    nz = scale > 0
    eb = float(np.max(err[nz] / scale[nz])) if nz.any() else 0.0
    assert eb < 1e-7, eb
    assert np.all(err[~nz] == 0)
    shared = (obs.T.astype(np.int64) @ obs.astype(np.int64)) > 0
    assert np.all(np.max(np.abs(Hb), axis=(1, 3))[~shared] == 0), "non-zero block for a frame pair that shares no voxel"
    note("hessian", max(er / 1e-12, ej / 1e-9, eh / 1e-9, eb / 1e-7))


def check_same(got, base):
    """A/B form vs the default form on the same factor: only the summation order differs"""
    for a, b in zip(got, base):
        e = relinf(a, b) if np.ndim(a) else abs(a - b) / abs(b)
        assert e <= 1e-12, e
        note("hessian A/B vs default", e / 1e-12)


# ------------------------------------------------------------------------------------------------ 3. Hessian sweep
DENSE_W = [1, 2, 3, 7, 8, 9, 16, 17, 24, 63, 64, 65, 127, 128, 129, 136]


@pytest.mark.parametrize("W", DENSE_W, ids=[f"W{w}" for w in DENSE_W])
def test_hessian_dense(ctx, W):
    """sy_geom remainder groups / pair-count parity / diagonal tile masks, k_jac_slab<64|128>, slab vs k_jac<G,true> + k_syrk at 128/129"""
    c = case(W, 150, "dense", seed=1)
    assert is_dense(c)
    got, ran = hessian_on_reused_factor(ctx, c)
    check_path(ran, c)
    check_hessian(got, hessian_ref(c), c["obs"])


VMOD = [(W, V) for W in (9, 65, 129) for V in (40, 41, 42, 43, 1, 3)]


@pytest.mark.parametrize("W,V", VMOD, ids=[f"W{w}-V{v}" for w, v in VMOD])
def test_hessian_voxel_count_mod4(ctx, W, V):
    """the last voxel group of 4 partly padding (slab zero-fill for W <= 128, memset above)"""
    c = case(W, V, "dense", seed=2)
    assert is_dense(c)
    got, ran = hessian_on_reused_factor(ctx, c)
    check_path(ran, c)
    check_hessian(got, hessian_ref(c), c["obs"])


# (W, entries per voxel) -> k_jac<G,false> / k_pairs<G>
SPARSE = [(30, 5, 8, 8), (60, 12, 16, 16), (100, 20, 32, 32), (120, 28, 64, 32)]


@pytest.mark.parametrize("W,k,gj,gp", SPARSE, ids=[f"W{w}-k{k}-jac{gj}-pairs{gp}" for w, k, gj, gp in SPARSE])
def test_hessian_sparse_groups(ctx, W, k, gj, gp):
    c = case(W, 200, "k", seed=3, k=k)
    E, V = int(c["obs"].sum()), c["V"]
    assert not is_dense(c) and pick_group_jac(E, V, W) == gj and pick_group(E, V) == gp
    got, ran = hessian_on_reused_factor(ctx, c)
    check_path(ran, c)
    check_hessian(got, hessian_ref(c), c["obs"])


def test_hessian_sparse_strided_window(ctx):
    """frames embedded with a stride into a wider window: most frame pairs share no voxel"""
    c = case(60, 150, "stride", seed=4, stride=10)
    assert not is_dense(c)
    got, ran = hessian_on_reused_factor(ctx, c)
    check_path(ran, c)
    check_hessian(got, hessian_ref(c), c["obs"])


@pytest.mark.parametrize("short,dense", [(0, True), (1, False)], ids=["VW-eq-4E-dense", "VW-gt-4E-sparse"])
def test_hessian_dense_sparse_switch(ctx, short, dense):
    """V*W = 4E is still dense; one entry fewer is sparse"""
    c = case(40, 100, "k", seed=5, k=10, single=0, empty=0, short=short)
    E = int(c["obs"].sum())
    assert E == 1000 - short and is_dense(c) == dense
    got, ran = hessian_on_reused_factor(ctx, c)
    check_path(ran, c)
    check_hessian(got, hessian_ref(c), c["obs"])


def test_hessian_no_fix_unit_coe(ctx):
    c = case(65, 90, "dense", seed=6, fix=False, coe=False, single=0)
    got, ran = hessian_on_reused_factor(ctx, c)
    check_path(ran, c)
    check_hessian(got, hessian_ref(c), c["obs"])


# ------------------------------------------------------------------------------------------------ 4. A/B equivalence of the SYRK forms
FORMS = {"waves1": dict(VXS_SYRK_WAVES=1), "waves3": dict(VXS_SYRK_WAVES=3), "waves24": dict(VXS_SYRK_WAVES=24)}
AB_SHAPES = ["W37", "W50", "W129", "W50-many-groups"]


def ab_case(shape):
    if shape == "W50-many-groups":
        return case(50, 32 * sm_count() + 5, "dense", seed=8)
    return case(int(shape[1:]), 150, "dense", seed=7)


def syrk_groups_per_cta(W, V, waves):   # vxs_eval.cu launch_syrk, one upload chunk: voxel groups of 4 per k_syrk CTA
    r0 = W % 8 or 8
    nbp = ((W - r0) // 8 + 2) // 2
    ntiles = nbp * (nbp + 1) // 2
    ng = (V + 3) // 4
    nchunks = max(1, min(sm_count() * 2 * waves // ntiles, (ng + 7) // 8))
    return -(-ng // nchunks)


@pytest.mark.parametrize("form", list(FORMS))
@pytest.mark.parametrize("shape", AB_SHAPES)
def test_syrk_ab_forms(ctx, env_ctx, shape, form):
    c = ab_case(shape)
    if shape == "W50-many-groups":
        assert syrk_groups_per_cta(50, c["V"], 1) > 8        # at one wave the CTA target, not the 8-groups-per-chunk floor, sets the chunks
    base, _ = hessian_on_reused_factor(ctx, c)
    got, ran = hessian_on_reused_factor(env_ctx(**FORMS[form]), c)
    check_path(ran, c)
    check_hessian(got, hessian_ref(c), c["obs"])
    check_same(got, base)


@pytest.mark.parametrize("W", [64, 65])
def test_chunked_first_build_after_async_push(ctx, W):
    """vxs_factor_push_voxels_async: the first build runs the Jacobian + SYRK chunk by chunk behind the upload events (V % 4 != 0)"""
    c = case(W, 257, "dense", seed=9)
    base, _ = hessian_on_reused_factor(ctx, c)
    got, ran = hessian_on_reused_factor(ctx, c, async_push=True)
    check_path(ran, c)
    check_hessian(got, hessian_ref(c), c["obs"])
    check_same(got, base)


# ------------------------------------------------------------------------------------------------ 5. residual sweep
def resid_plan(V, W):
    """vxs_resid.cu vxs_residual_stream_launch: (vbcap, SP) — the batch accumulator rows per CTA and whether the [12][W] pose table fits in the
    per-CTA shared memory of 3 CTAs per SM next to the 2 stages of 256 entries"""
    import torch
    G = 3 * sm_count()
    m = max(1, (V + G * 48) // (G * 96))
    VB = -(-V // (G * m))
    while VB > 256:
        m += 1
        VB = -(-V // (G * m))
    vbcap = (max(VB, 1) + 7) & ~7
    base = 2 * (10 * 258 * 8 + 256 * 4) + vbcap * 80 + (vbcap + 8) * 4 + 256 * 8 + 2 * 2 * 8 + 128
    budget = torch.cuda.get_device_properties(0).shared_memory_per_block_optin // 3 - 1024
    return vbcap, base + 12 * W * 8 <= budget


@functools.lru_cache(maxsize=None)
def csr_case(W, V, k, seed):
    """A residual factor in CSR form (what push_voxels_async takes), for voxel counts whose dense [V][W][10] arrays would not fit in host
    memory: each voxel is seen by k frames spread over the window, entry (v, j) is the body-frame cluster of base frame j % 8 of a fully
    observed base voxel, a world-frame fix cluster on every third voxel, random positive coe."""
    cl0, est = _base()
    rng = np.random.default_rng(1000003 * seed + 1009 * W + V)
    fr = np.sort((rng.integers(W, size=V)[:, None] + np.arange(k) * (W // k)) % W, axis=1)
    src = (np.arange(V) * 37 + seed) % cl0.shape[0]
    fix10 = np.zeros((V, 10))
    for v in range(0, V, 3):
        fix10[v] = oa.cluster_transform(cl0[src[v], 1], est[1])
    return dict(W=W, V=V, ptr=np.arange(0, V * k + 1, k, dtype=np.int64), fr=fr.ravel().astype(np.int32), ent=cl0[src[:, None], fr % 8].reshape(-1, 10),
                fix=fix10, coe=rng.uniform(0.5, 2.0, V), poses=window_poses(W, seed))


def csr_clusters(c, a, b):
    """dense [b - a][W][10] clusters of voxels [a, b) of a csr_case"""
    ptr, lo, hi = c["ptr"], c["ptr"][a], c["ptr"][b]
    out = np.zeros((b - a, c["W"], 10))
    out[np.repeat(np.arange(b - a), np.diff(ptr[a:b + 1])), c["fr"][lo:hi]] = c["ent"][lo:hi]
    return out


def band_w196(): return csr_case(196, 144 * 3 * sm_count() - 1, 4, 15)      # vbcap 144: the smallest W whose pose table can miss


def band_w256(): return csr_case(256, 80 * 3 * sm_count(), 4, 16)            # vbcap 80


RESID_SHAPES = {
    "W20-sp": lambda: case(20, 300, "dense", seed=10, empty=0),
    "W136-full-sp": lambda: case(136, 60, "full", seed=11, single=0, empty=0),      # 136 entries per voxel: more than a 128-entry tile
    "W300-mixed-sp": lambda: case(300, 80, "mixed", seed=12, stride=10, empty=0),   # > 256 entries (> one tile), and a 28.8 KB pose table
    "W520-mixed-gmem": lambda: case(520, 40, "mixed", seed=13, stride=7, empty=0),  # > 256 entries, poses from global memory
    "W16-V7-sp": lambda: case(16, 7, "dense", seed=14, empty=0),                    # fewer voxels than CTAs
    "W196-V144G-gmem": band_w196,
    "W256-V80G-gmem": band_w256,
    "W256-V300-sp": lambda: csr_case(256, 300, 4, 17),
}


def eval_poses(c):
    W = c["W"]
    return np.stack([synth.perturb_pose(p, 7 * W + j, 1e-3, 5e-3) for j, p in enumerate(c["poses"])])


def residual_ref(c, poses, chunk=2048):
    """the oracle's evaluate_only_residual and the cache (eig, pcr_add) it leaves, voxel slice by voxel slice so that a slice's dense
    [n][W][10] arrays stay small; the cache the factor is pushed with does not enter the residual"""
    r, eig, s = 0.0, [], []
    for a in range(0, c["V"], chunk):
        b = min(c["V"], a + chunk)
        if "ptr" in c:
            dense = csr_clusters(c, a, b)
        else:
            dense = c["cl"][a:b]
        of = oa.OracleFactor.from_dense(c["W"], dense, None if c["fix"] is None else c["fix"][a:b], None if c["coe"] is None else c["coe"][a:b],
                                        np.zeros((b - a, 12)), np.zeros((b - a, 10)))
        r += of.residual(poses)
        ex = of.export()
        eig.append(ex["eig12"])
        s.append(ex["sum10"])
    return r, np.concatenate(eig), np.concatenate(s)


def check_eig(e_gpu, e_ref, tol):
    assert relinf(e_gpu[:, :3], e_ref[:, :3]) < tol
    Ug, Ur = e_gpu[:, 3:].reshape(-1, 3, 3), e_ref[:, 3:].reshape(-1, 3, 3)
    lam = e_ref[:, :3]
    worst = relinf(e_gpu[:, :3], e_ref[:, :3]) / tol
    for k in range(3):       # eigenvectors up to sign, only where the eigenvalue gap makes them well defined
        gap = np.min(np.abs(lam - lam[:, [k]]) + np.eye(3)[k] * 1e300, axis=1) / np.max(np.abs(lam), axis=1)
        ok = gap > 1e-3
        d = np.abs(np.abs(np.sum(Ug[ok, :, k] * Ur[ok, :, k], axis=1)) - 1.0)
        assert d.size == 0 or d.max() < 1e-8
        worst = max(worst, (d.max() if d.size else 0.0) / 1e-8)
    return worst


def check_residual(r_gpu, eig, s, ref):
    """residual to 1e-10, cached sums to 1e-12, eigenvalues to 1e-7 of lambda_max, eigenvectors to 1e-8 (as test_gpu_ba)"""
    rr, eig_ref, sum_ref = ref
    er = abs(r_gpu - rr) / abs(rr)
    assert er < 1e-10, er
    es = relinf(s, sum_ref)
    assert es < 1e-12, es
    ee = check_eig(eig, eig_ref, 1e-7)
    note("residual", max(er / 1e-10, es / 1e-12, ee))


@pytest.mark.parametrize("shape", list(RESID_SHAPES))
def test_residual_shapes(ctx, shape):
    c = RESID_SHAPES[shape]()
    assert resid_plan(c["V"], c["W"])[1] == shape.endswith("-sp")
    if shape == "W196-V144G-gmem":
        assert resid_plan(c["V"], c["W"])[0] == 144 and resid_plan(c["V"], 195)[1]
    if shape == "W256-V80G-gmem":
        assert resid_plan(c["V"], c["W"])[0] == 80
    poses = eval_poses(c)
    f = vx.Factor(ctx, c["W"])
    if "ptr" in c:
        f.push_voxels_async(c["ptr"], c["fr"], c["ent"], np.zeros((c["V"], 12)), np.zeros((c["V"], 10)), fix10=c["fix"], coe=c["coe"])
    else:
        push(f, c)
    ctx.timing_reset()
    r1 = ctx.evaluate_residual(f, poses)
    assert "k_residual_stream" in ran_kernels(ctx)
    e1, s1 = f.read_back()
    check_residual(r1, e1, s1, residual_ref(c, poses))
    # the streaming kernel's reduction order depends only on the factor and the launch shape
    r2 = ctx.evaluate_residual(f, poses)
    e2, s2 = f.read_back()
    assert r2 == r1 and np.array_equal(e2, e1) and np.array_equal(s2, s1)
    f.close()


# ------------------------------------------------------------------------------------------------ 6. LDL^T sweep
def ldlt_system(n, kind, gauge, seed):
    """(H, g) before the gauge fix.  kinds: spd; indef (diagonal of random sign, |d| in [2, 3], small coupling); scaled (unit-diagonal SPD
    scaled to a diagonal spanning 1e-10 .. 1e10); ties (all |diag| = 1, random signs); zero (SPD with zero rows / columns outside the gauge,
    a frame that observes no voxel)."""
    rng = np.random.default_rng(seed)

    def sym_noise(c):
        G = rng.standard_normal((n, n))
        return (G + G.T) * (0.5 * c / np.sqrt(n))

    g = rng.standard_normal(n)
    if kind in ("spd", "zero", "scaled"):
        R = rng.standard_normal((n, n))
        A = R @ R.T / n + np.eye(n)
        if kind == "scaled":
            d = np.sqrt(np.diag(A))
            A = A / np.outer(d, d)
            s = np.sqrt(np.logspace(-10, 10, n))[rng.permutation(n)]
            A = A * np.outer(s, s)
        if kind == "zero":
            rows = np.array([n // 2, n - 1]) if n < 12 else np.r_[6 * ((n // 6) // 2):6 * ((n // 6) // 2) + 6, n - 1]
            rows = rows[rows >= gauge]
            assert rows.size > 0
            A[rows, :] = 0.0
            A[:, rows] = 0.0
            g[rows] = 0.0
    elif kind == "indef":
        A = sym_noise(0.5)
        A[np.diag_indices(n)] = rng.choice([-1.0, 1.0], n) * rng.uniform(2.0, 3.0, n)
    elif kind == "ties":
        A = sym_noise(0.5)
        A[np.diag_indices(n)] = rng.choice([-1.0, 1.0], n)
    else:
        raise ValueError(kind)
    A = (A + A.T) * 0.5
    return A, g


def damped_system(H, g, gauge, u):
    """the LM step's system: Hess.topRows/leftCols(gauge) = 0, identity block, JacT.head(gauge) = 0; A = Hess + u diag(Hess), b = -JacT"""
    A = H.copy()
    A[:gauge, :] = 0.0
    A[:, :gauge] = 0.0
    A[:gauge, :gauge] = np.eye(gauge)
    A[np.diag_indices_from(A)] += u * np.diag(A)
    b = -g.copy()
    b[:gauge] = 0.0
    return A, b


def backward_error(A, x, b):
    A, x, b = (np.asarray(a, dtype=np.longdouble) for a in (A, x, b))
    r = np.max(np.abs(A @ x - b))
    return 0.0 if r == 0 else float(r / (np.max(np.sum(np.abs(A), axis=1)) * np.max(np.abs(x)) + np.max(np.abs(b))))


def check_ldlt(dx, sing, H, g, gauge, u):
    """vs the oracle's Eigen-ordered LDL^T: singular flag = oracle status, dx = 0 in the zero-pivot and gauge rows, solution to 1e-10 relative
    after symmetric diagonal equilibration (every system here is well conditioned once equilibrated); and a backward error in long double,
    independent of both LDL^T implementations, below max(10 x the oracle's, 10 n 2^-53)."""
    A, b = damped_system(H, g, gauge, u)
    n = A.shape[0]
    x_ref, rc = oa.ldlt_solve(A, b)
    assert bool(sing) == (rc != 0), (sing, rc)
    zero = np.diag(A) == 0.0
    assert np.all(dx[zero] == 0.0) and np.all(x_ref[zero] == 0.0)
    assert np.all(dx[:gauge] == 0.0)
    s = np.where(zero, 1.0, np.sqrt(np.abs(np.diag(A))))
    ex = relinf(dx * s, x_ref * s)
    assert ex < 1e-10, ex
    bg, bo = backward_error(A, dx, b), backward_error(A, x_ref, b)
    bound = max(10.0 * bo, 10.0 * n * 2.0 ** -53)
    assert bg < bound, (bg, bo)
    note("ldlt vs oracle", ex / 1e-10)
    note("ldlt backward error", bg / bound)
    return A, x_ref


# (n, kind, gauge, u): every n of the sweep with two or three systems; gauge / u / kind combinations sampled, not the full product
LDLT_CASES = [
    (1, "spd", 0, 0.0), (1, "indef", 0, 1e-2),
    (6, "ties", 0, 1e-4), (6, "zero", 0, 0.0), (6, "spd", 6, 1e-2),
    (31, "indef", 6, 1e-4), (31, "scaled", 0, 1e-2),
    (32, "spd", 15, 0.0), (32, "ties", 6, 1e-2), (32, "zero", 6, 1e-4),
    (33, "scaled", 6, 1e-4), (33, "indef", 15, 0.0),
    (63, "ties", 15, 1e-4), (63, "spd", 0, 1e-2),
    (64, "indef", 0, 0.0), (64, "scaled", 15, 1e-2),
    (65, "zero", 15, 1e-2), (65, "spd", 6, 1e-4),
    (95, "scaled", 0, 0.0), (95, "ties", 6, 1e-2),
    (96, "indef", 6, 1e-2), (96, "zero", 0, 1e-4),
    (127, "spd", 15, 1e-4), (127, "ties", 0, 0.0),
    (128, "zero", 6, 0.0), (128, "scaled", 6, 1e-4),
    (129, "indef", 15, 1e-2), (129, "spd", 0, 1e-4),
    (480, "ties", 6, 1e-4), (480, "scaled", 15, 0.0),
    (960, "indef", 6, 1e-4), (960, "zero", 15, 1e-2),
    (992, "spd", 6, 1e-2), (992, "scaled", 0, 1e-4),
    (1025, "ties", 15, 1e-2), (1025, "indef", 0, 1e-4),
    (1500, "zero", 6, 1e-4), (1500, "scaled", 15, 1e-2),
    (2394, "spd", 6, 1e-4), (2394, "scaled", 6, 1e-2), (2394, "zero", 6, 0.0),
]


def ldlt_id(t):
    n, kind, gauge, u = t
    return f"n{n}-{kind}-g{gauge}-u{u:g}"


def run_ldlt(cx, n, kind, gauge, u):
    H, g = ldlt_system(n, kind, gauge, seed=n * 31 + len(kind) + gauge)
    cx.timing_reset()
    dx, sing = cx.solve_damped(H, g, gauge, u)
    assert "k_ldlt_all" in ran_kernels(cx)
    check_ldlt(dx, sing, H, g, gauge, u)
    assert sing == (1 if kind == "zero" else 0)


@pytest.mark.parametrize("n,kind,gauge,u", LDLT_CASES, ids=[ldlt_id(t) for t in LDLT_CASES])
def test_ldlt(ctx, n, kind, gauge, u):
    run_ldlt(ctx, n, kind, gauge, u)


LDLT_NO_LA = [(33, "indef", 6, 1e-4), (65, "spd", 6, 1e-2), (480, "scaled", 6, 1e-4), (992, "ties", 6, 1e-2), (1025, "zero", 15, 1e-4),
              (2394, "indef", 6, 1e-2)]


@pytest.mark.parametrize("n,kind,gauge,u", LDLT_NO_LA, ids=[ldlt_id(t) for t in LDLT_NO_LA])
def test_ldlt_without_lookahead_cta(env_ctx, n, kind, gauge, u):
    run_ldlt(env_ctx(VXS_LDLT_LOOKAHEAD_CTA=0), n, kind, gauge, u)


# ------------------------------------------------------------------------------------------------ 7. negative controls
def drop_one_entry(c):
    """the dense clusters with one (voxel, frame) entry removed from a voxel that keeps other entries"""
    v = int(np.flatnonzero(c["obs"].sum(axis=1) >= 3)[0])
    j = int(np.flatnonzero(c["obs"][v])[1])
    cl = c["cl"].copy()
    cl[v, j] = 0.0
    return cl


def test_negative_control_hessian(ctx):
    c = case(65, 150, "dense", seed=1)
    got, _ = hessian_on_reused_factor(ctx, c, cl=drop_one_entry(c))
    with pytest.raises(AssertionError):
        check_hessian(got, hessian_ref(c), c["obs"])


def test_negative_control_residual(ctx):
    c = RESID_SHAPES["W20-sp"]()
    poses = eval_poses(c)
    f = vx.Factor(ctx, c["W"])
    push(f, c, drop_one_entry(c))
    r = ctx.evaluate_residual(f, poses)
    e, s = f.read_back()
    f.close()
    with pytest.raises(AssertionError):
        check_residual(r, e, s, residual_ref(c, poses))


def test_negative_control_ldlt(ctx):
    n, gauge, u = 480, 6, 1e-4
    H, g = ldlt_system(n, "spd", gauge, seed=11)
    dx, sing = ctx.solve_damped(H, g, gauge, u)
    A, x_ref = check_ldlt(dx, sing, H, g, gauge, u)
    k = gauge + int(np.argmax(np.abs(np.diag(A) * x_ref)[gauge:]))
    Hp = H.copy()
    Hp[k, k] *= 1.0 + 1e-9                                 # one pivot off by 1e-9 relative
    dxp, singp = ctx.solve_damped(Hp, g, gauge, u)
    with pytest.raises(AssertionError):
        check_ldlt(dxp, singp, H, g, gauge, u)
