"""The warp-per-chain row kernels against the float32 oracle in every row size class, for HMC and NUTS.

The row kernels are templates over the row size class (csrc/bjx_launch.cuh ``size_class_for``); every class is separately
compiled code.  NUTS also changes its code path with the row: rows of 16 and 32 slots per lane (V4, V8) keep only the
moving trajectory endpoint in registers and go through the workspace for the other one and the momentum sum, and the
U-turn checkpoints live in shared or global memory depending on the row size and the depth (csrc/bjx_api.cu
``ckpt_in_smem``).  The case lists below are checked at import to reach every class at both of its edges and every
NUTS class with both checkpoint homes.

Tolerances (DESIGN section 4): one step from identical inputs within 1e-5 relative; discrete decisions identical except
where the deciding float comparison sits within rounding of a tie (|u - p_accept| < 1e-5, NUTS: the oracle's margins).
"""
import numpy as np
import pytest
import torch

import blackjax_b200 as bj
from blackjax_b200 import _engine, targets as T
from blackjax_b200.mcmc import integrators as I
from blackjax_b200.mcmc.metrics import gaussian_euclidean_low_rank
from oracle import adaptation as oadapt
from oracle import hmc as ohmc
from oracle import nuts as onuts
from oracle import prng as oprng
from oracle import targets as otargets
from test_gpu_parity import close, make_target, npy, tf, tk

pytestmark = pytest.mark.gpu
F = np.float32
DEV = "cuda:0"


# ---------------------------------------------------------------------------------------------------------------------
# the coverage table, restated from the C++ and checked at import
# ---------------------------------------------------------------------------------------------------------------------
def size_class_for(D):
    """csrc/bjx_launch.cuh size_class_for, warp-kernel classes only (None: the CTA-per-chain rows)."""
    if D % 4 == 0 and D <= 1024:
        return "V1" if D <= 128 else "V2" if D <= 256 else "V4" if D <= 512 else "V8"
    if D <= 32:
        return "S1"
    if D <= 128:
        return "S4"
    return None


SLOTS = {"S1": 1, "S4": 4, "V1": 4, "V2": 8, "V4": 16, "V8": 32}   # float slots per lane (R::NS)
CLASS_EDGES = {"S1": ({1, 3}, 31), "S4": ({33}, 127), "V1": ({4}, 128), "V2": ({132}, 256), "V4": ({260}, 512),
               "V8": ({516}, 1024)}
MAX_TREE_DEPTH = 30                       # bjx_create's bound on max_tree_depth


def ckpt_in_smem(D, depth, row_slice):
    """csrc/bjx_api.cu ckpt_in_smem: 4 warps x 2 rows x depth x D floats of checkpoints, plus one row slice per warp when
    the metric is small dense or low rank (or the target dense / user-defined), must fit in 40 KB."""
    return 4 * 4 * 2 * depth * D + (4 * 4 * D if row_slice else 0) <= 40 * 1024


def check_edges(dims, name):
    by_class = {}
    for D in dims:
        by_class.setdefault(size_class_for(D), set()).add(D)
    for sc, (low, high) in CLASS_EDGES.items():
        got = by_class.get(sc, set())
        assert got & low and high in got, f"{name}: class {sc} needs dims {sorted(low)} (one of) and {high}, has {sorted(got)}"


def check_homes(cases, name):
    homes = {}
    for D, depth, row_slice in cases:
        homes.setdefault(size_class_for(D), set()).add(ckpt_in_smem(D, depth, row_slice))
    for sc, (_, high) in CLASS_EDGES.items():
        # S1 rows are too short for any depth to push the checkpoints out of shared memory
        want = {True} if ckpt_in_smem(high, MAX_TREE_DEPTH, True) else {True, False}
        assert homes.get(sc) == want, f"{name}: class {sc} has checkpoint homes {homes.get(sc)}, needs {want}"


# row kernels: (D, metric); metric in diag / per_chain / dense (small dense, D <= 128) / low_rank (D <= 512)
ROW_DIMS = [1, 3, 31, 33, 127, 4, 128, 132, 256, 260, 512, 516, 1024]
ROW_CASES = [(D, m) for D in ROW_DIMS for m in ("diag", "per_chain", "dense", "low_rank")
             if not (m == "dense" and D > 128) and not (m == "low_rank" and (D > 512 or D < 4))]
check_edges(ROW_DIMS, "ROW_CASES")
assert {size_class_for(D) for D, m in ROW_CASES if m == "dense"} == {"S1", "S4", "V1"}
assert {size_class_for(D) for D, m in ROW_CASES if m == "low_rank"} == {"S1", "S4", "V1", "V2", "V4"}

# step-wise NUTS against the oracle: (target, D, C, step size, metric, engine max_tree_depth, max_num_doublings, per-chain
# step size).  The engine's depth decides the checkpoint home.
NUTS_CASES = [
    ("diag", 1, 64, 0.5, "ones", 10, 10, False),
    ("funnel", 31, 64, 0.2, "diag", 10, 10, False),
    ("diag", 33, 64, 0.3, "diag", 10, 10, True),
    ("funnel", 127, 48, 0.1, "ones", 11, 10, False),       # 4064 B per doubling: global at depth 11
    ("diag", 127, 40, 0.25, "dense", 10, 10, False),       # small dense metric, global
    ("diag", 33, 40, 0.25, "dense", 10, 10, False),        # small dense metric, shared memory
    ("funnel", 128, 64, 0.1, "ones", 10, 10, False),       # exactly 40 KB: shared memory
    ("diag", 128, 48, 0.2, "diag", 11, 10, False),         # global
    ("diag", 4, 64, 0.4, "per_chain", 10, 10, True),
    ("diag", 128, 40, 0.2, "dense", 10, 8, False),         # small dense metric at V1, global
    ("diag", 132, 48, 0.06, "diag", 10, 10, False),        # V2, global, deeper than the fused doublings
    ("funnel", 256, 48, 0.03, "ones", 5, 5, False),        # V2 at exactly 40 KB: the fifth doubling is its own launch
    ("diag", 256, 40, 0.08, "low_rank", 10, 10, False),
    ("std", 512, 40, 1e-3, "ones", 10, 10, False),         # V4: every tree 1023 leaves, global checkpoints
    ("diag", 260, 48, 0.3, "diag", 4, 4, False),           # V4, shared memory
    ("funnel", 512, 48, 0.04, "per_chain", 10, 10, True),  # per-chain step size and diagonal metric at V4
    ("diag", 512, 40, 0.08, "low_rank", 10, 10, False),
    ("diag", 512, 40, 0.3, "low_rank", 2, 2, False),       # low rank at exactly 40 KB: shared memory
    ("diag", 1024, 40, 0.05, "diag", 10, 10, False),       # V8, global, deeper than the fused doublings
    ("funnel", 516, 40, 0.05, "ones", 1, 1, False),        # V8, shared memory
    ("diag", 1024, 40, 0.06, "per_chain", 10, 10, True),   # per-chain step size and diagonal metric at V8
    ("diag", 1024, 40, 1e3, "ones", 10, 10, False),        # diverges on the first leaf
]


def _row_slice(target, metric):
    return metric in ("dense", "low_rank") or target == "dense"


check_edges([c[1] for c in NUTS_CASES], "NUTS_CASES")
check_homes([(c[1], c[5], _row_slice(c[0], c[4])) for c in NUTS_CASES], "NUTS_CASES")

# NUTS on trajectories that float32 represents exactly: (D, engine max_tree_depth), max_num_doublings 3
EXACT_CASES = [(3, 10), (31, 10), (33, 10), (127, 11), (4, 10), (128, 11), (132, 10), (256, 5), (260, 4), (512, 10),
               (516, 2), (1024, 10)]
check_edges([D for D, _ in EXACT_CASES], "EXACT_CASES")
check_homes([(D, depth, False) for D, depth in EXACT_CASES], "EXACT_CASES")


# ---------------------------------------------------------------------------------------------------------------------
# setup shared by the tests below
# ---------------------------------------------------------------------------------------------------------------------
def make_metric(kind, D, C, rs):
    """(device metric, oracle metric) of one kind."""
    if kind == "ones":
        imm = np.ones(D, F)
        return tf(imm), ohmc.Metric(imm)
    if kind == "diag":
        imm = np.exp(rs.uniform(-0.5, 0.5, D)).astype(F)
        return tf(imm), ohmc.Metric(imm)
    if kind == "per_chain":
        imm = np.exp(rs.uniform(-0.5, 0.5, (C, D))).astype(F)
        return tf(imm), oadapt._PerChainDiag(imm)
    if kind == "dense":
        A = rs.standard_normal((D, D))
        imm = (A @ A.T / D + np.eye(D)).astype(F)
        return tf(imm), ohmc.Metric(imm)
    if kind == "low_rank":
        k = min(8, D - 1)
        U, _ = np.linalg.qr(rs.standard_normal((D, k)))
        sigma = np.exp(rs.uniform(-0.5, 0.5, D)).astype(F)
        lam = np.exp(rs.uniform(-1.0, 1.0, k)).astype(F)
        U = U.astype(F)
        return gaussian_euclidean_low_rank(tf(sigma), tf(U), tf(lam)), ohmc.LowRankMetric(sigma, U, lam)
    raise ValueError(kind)


def exact_metric(kind, D, C, rs):
    """A metric of the kind whose products with small integer vectors are exact in float32, and whose M^-1 keeps a
    vector's support inside its group (row_group): dyadic diagonals, 2 x 2 integer blocks, coordinate-axis low rank.
    Returns (device metric, oracle metric, M^-1 as float64 [C, D, D])."""
    if kind in ("diag", "per_chain"):
        imm = (2.0 ** rs.integers(-2, 3, (C, D) if kind == "per_chain" else D)).astype(F)
        full = np.broadcast_to(np.eye(D) * imm[..., None, :], (C, D, D))
        return tf(imm), (oadapt._PerChainDiag(imm) if kind == "per_chain" else ohmc.Metric(imm)), full
    if kind == "dense":
        imm = np.eye(D, dtype=F) * 2
        for b in range(0, D - 1, 2):
            imm[b, b + 1] = imm[b + 1, b] = 1
        return tf(imm), ohmc.Metric(imm), np.broadcast_to(imm.astype(np.float64), (C, D, D))
    k = min(4, D)
    sigma = (2.0 ** rs.integers(-1, 2, D)).astype(F)
    U = np.eye(D, k, dtype=F)
    lam = np.arange(2, 2 + k).astype(F)
    full = np.diag(sigma) @ (np.eye(D) + U @ np.diag(lam - 1) @ U.T) @ np.diag(sigma)
    return (gaussian_euclidean_low_rank(tf(sigma), tf(U), tf(lam)), ohmc.LowRankMetric(sigma, U, lam),
            np.broadcast_to(full, (C, D, D)))


def row_group(kind, D):
    """Coordinates split into two groups that M^-1 of exact_metric never mixes (the dense blocks are pairs)."""
    i = np.arange(D)
    return (i // 2) % 2 == 0 if kind == "dense" else i % 2 == 0


def engine(D, C, tgt, metric, depth=10):
    eng = _engine.Engine(DEV, C, D, tgt, max_tree_depth=depth)
    eng.set_metric(metric)
    return eng


# ---------------------------------------------------------------------------------------------------------------------
# row kernels per class
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D, metric", ROW_CASES)
def test_row_building_blocks_match_oracle(D, metric):
    rs = np.random.default_rng(D * 7 + len(metric))
    C = 37
    tgt, otgt = make_target("diag", D, rs)          # the funnel's kernels are checked through NUTS below
    dm, om = make_metric(metric, D, C, rs)
    eng = engine(D, C, tgt, dm)
    q = (0.4 * rs.standard_normal((C, D))).astype(F)
    dq = tf(q)
    logp, g = eng.init_state(dq)
    lp0, g0 = otgt(q)
    close(npy(logp), lp0, rtol=1e-5, scale=np.max(np.abs(lp0)) + 1)
    close(npy(g), g0, rtol=1e-5)
    keys = oprng.split(oprng.key(D + 3), C)
    p_ref = om.sample_momentum(keys, D)
    close(npy(eng.sample_momentum(tk(keys))), p_ref, rtol=1e-5)
    e_ref = (-lp0 + om.kinetic_energy(p_ref)).astype(F)
    close(npy(eng.energy(tf(p_ref), logp)), e_ref, rtol=1e-5, scale=np.max(np.abs(lp0)) + D)
    # velocity Verlet and McLachlan, three steps each from identical inputs
    for coef, ocoef in ((I.velocity_verlet, ohmc.VELOCITY_VERLET), (I.mclachlan, ohmc.MCLACHLAN)):
        eng.set_integrator(coef)
        dq, dp = tf(q), tf(p_ref)
        lg, gg = eng.init_state(dq)
        eng.leapfrog_(dq, dp, lg, gg, 0.05, 3)
        q1, p1, lp1, g1 = ohmc.static_integration(otgt, om, q, p_ref, lp0, g0, F(0.05), 3, ocoef)
        close(npy(dq), q1, rtol=1e-5)
        close(npy(dp), p1, rtol=1e-5)
        close(npy(gg), g1, rtol=1e-5)
        close(npy(lg), lp1, rtol=1e-5, scale=np.max(np.abs(lp1)) + 1)
    eng.set_integrator(I.velocity_verlet)
    # one HMC and one multinomial-HMC transition with per-chain step sizes
    eps = (0.08 * np.exp(rs.uniform(-0.3, 0.3, C))).astype(F)
    for multinomial in (False, True):
        okern = ohmc.mhmc_kernel if multinomial else ohmc.hmc_kernel
        onew, oinfo = okern(keys, ohmc.init(q, otgt), otgt, eps, om, 5)
        alg = bj.mhmc if multinomial else bj.hmc
        new, info = alg.build_kernel(full_info=True)(tk(keys), alg.init(tf(q), tgt), tgt, tf(eps), dm, 5)
        torch.cuda.synchronize()
        close(npy(info.momentum), oinfo.momentum, rtol=1e-5)
        assert (npy(info.is_divergent) == oinfo.is_divergent).all()
        if not multinomial:
            close(npy(info.proposal.position), oinfo.proposal[0], rtol=1e-5)
            close(npy(info.proposal.momentum), oinfo.proposal[1], rtol=1e-5)
            close(npy(info.energy), oinfo.energy, rtol=1e-5, scale=np.max(np.abs(oinfo.energy)) + D)
            close(npy(info.acceptance_rate), oinfo.acceptance_rate, rtol=1e-4, scale=1.0)
            u = oprng.uniform(oprng.split(keys, 2)[:, 1])
            acc = npy(info.is_accepted)
            assert ((acc == oinfo.is_accepted) | (np.abs(u - oinfo.acceptance_rate) < 1e-5)).all()
            same = acc == oinfo.is_accepted
        else:
            # the selected leaf: identical except where one of the progressive draws sat on a tie
            same = np.all(np.isclose(npy(new.position), onew.position, rtol=1e-4, atol=1e-5), axis=1)
            assert same.mean() >= 0.97
            close(npy(info.acceptance_rate)[same], oinfo.acceptance_rate[same], rtol=1e-4, scale=1.0)
            close(npy(info.energy)[same], oinfo.energy[same], rtol=1e-5, scale=np.max(np.abs(oinfo.energy)) + D)
        # the state after five leapfrogs (multinomial: the selected leaf, up to five of them)
        rtol = 1e-4 if multinomial else 1e-5
        close(npy(new.position)[same], onew.position[same], rtol=rtol)
        close(npy(new.logdensity_grad)[same], onew.logdensity_grad[same], rtol=rtol)
        close(npy(new.logdensity)[same], onew.logdensity[same], rtol=1e-5, scale=np.max(np.abs(onew.logdensity)) + 1)
    eng.close()


@pytest.mark.parametrize("D, metric", ROW_CASES)
def test_is_turning_matches_oracle_with_exact_ties(D, metric):
    """metrics.is_turning (<=, OR) through bjx_is_turning.  First on small-integer momenta whose U-turn products are
    exactly zero, positive or negative in float32 in any summation order (the momenta and the rho vector live in the
    two coordinate groups M^-1 never mixes), then on random momenta."""
    rs = np.random.default_rng(D * 11 + len(metric))
    C = 64
    tgt = T.StdNormal(D)
    dm, om, full = exact_metric(metric, D, C, rs)
    eng = engine(D, C, tgt, dm)
    a = row_group(metric, D)
    ints = lambda: (2 * rs.integers(-3, 4, (C, D))).astype(F)
    pl, pr, rho = ints(), ints(), ints()
    pattern = np.arange(C) % 4                        # 0: left product zero, 1: right zero, 2: both, 3: random signs
    on_a = np.where(a, 1, 0).astype(F)
    pl[pattern % 2 == 0] *= on_a                      # left momentum in group a, rho in group b: dl == 0
    pr[(pattern == 1) | (pattern == 2)] *= on_a
    rho[pattern < 3] *= 1 - on_a
    ps = (rho + (pl + pr) / 2).astype(F)
    dl = np.einsum("cij,cj,ci->c", full, pl.astype(np.float64), rho)
    dr = np.einsum("cij,cj,ci->c", full, pr.astype(np.float64), rho)
    assert (dl[pattern % 2 == 0] == 0).all() and (dr[(pattern == 1) | (pattern == 2)] == 0).all()
    assert D == 1 or ((dl > 0) & (dr > 0)).any()      # the zeros decide: some chains have only positive products
    want = (dl <= 0) | (dr <= 0)
    got = npy(eng.is_turning(tf(pl), tf(pr), tf(ps)))
    np.testing.assert_array_equal(got, want)
    np.testing.assert_array_equal(om.is_turning(pl, pr, ps), want)
    # random momenta, compared where no product is within rounding of zero
    # rho = a pl + b pr + noise with random signs a, b: each product takes the sign of its coefficient at every D
    pl, pr = rs.standard_normal((2, C, D)).astype(F)
    a, b = rs.choice([-1.0, 1.0], (2, C, 1))
    rho = a * pl + b * pr + 0.3 * rs.standard_normal((C, D))
    ps = (rho + (pl + pr) / 2).astype(F)
    dm, om = make_metric(metric, D, C, rs)
    eng.set_metric(dm)
    got = npy(eng.is_turning(tf(pl), tf(pr), tf(ps)))
    want = om.is_turning(pl, pr, ps)
    decided = om.turning_margin(pl, pr, ps) > 1e-5
    np.testing.assert_array_equal(got[decided], want[decided])
    assert decided.mean() > 0.9 and want.any() and not want.all()
    eng.close()


# ---------------------------------------------------------------------------------------------------------------------
# step-wise NUTS per class
# ---------------------------------------------------------------------------------------------------------------------
def compare_nuts(new, info, onew, oinfo, margins, min_match=0.97):
    """The protocol of test_nuts_disagreements_sit_on_ties with full_info: returns the agreeing chains."""
    same = ((npy(info.num_integration_steps) == oinfo.num_integration_steps)
            & (npy(info.num_trajectory_expansions) == oinfo.num_trajectory_expansions)
            & (npy(info.is_turning) == oinfo.is_turning) & (npy(info.is_divergent) == oinfo.is_divergent)
            & np.all(np.isclose(npy(new.position), onew.position, rtol=1e-4, atol=1e-5), axis=1))
    print(f"{same.mean():.4f} of chains identical; margins of the others {np.sort(margins[~same])[:6]}; tree sizes "
          f"{np.unique(oinfo.num_integration_steps)}")
    assert same.mean() >= min_match
    assert (margins[~same] < 1e-5 * 64).all(), np.sort(margins[~same])[-3:]
    assert same[margins > 1e-2].all()
    ok = same
    close(npy(info.energy)[ok], oinfo.energy[ok], rtol=1e-5, scale=np.max(np.abs(oinfo.energy[ok]), initial=0) + 1)
    close(npy(info.acceptance_rate)[ok], oinfo.acceptance_rate[ok], rtol=1e-4, scale=1.0)
    close(npy(new.logdensity_grad)[ok], onew.logdensity_grad[ok], rtol=1e-4)
    for side, oside in ((info.trajectory_leftmost_state, oinfo.trajectory_leftmost_state),
                        (info.trajectory_rightmost_state, oinfo.trajectory_rightmost_state)):
        close(npy(side.position)[ok], oside[0][ok], rtol=1e-4)
        close(npy(side.momentum)[ok], oside[1][ok], rtol=1e-4)
    return same


@pytest.mark.parametrize("kind, D, C, eps, metric, depth, md, pce", NUTS_CASES)
def test_nuts_matches_oracle_per_class(kind, D, C, eps, metric, depth, md, pce):
    rs = np.random.default_rng(D + C + md)
    tgt, otgt = make_target(kind, D, rs)
    dm, om = make_metric(metric, D, C, rs)
    q = (0.5 * rs.standard_normal((C, D))).astype(F)
    if kind == "funnel":
        q[:, 0] = rs.uniform(-1.0, 1.0, C)
    eps_np = (eps * np.exp(rs.uniform(-0.4, 0.4, C))).astype(F) if pce else F(eps)
    keys = oprng.split(oprng.key(D * 3 + md), C)
    margins = np.full(C, np.inf)
    onew, oinfo = onuts.nuts_kernel(keys, ohmc.init(q, otgt), otgt, eps_np, om, md, margins=margins)
    kern = bj.nuts.build_kernel(full_info=True, max_tree_depth=depth)
    new, info = kern(tk(keys), bj.nuts.init(tf(q), tgt), tgt, tf(eps_np) if pce else float(eps_np), dm, md)
    torch.cuda.synchronize()
    compare_nuts(new, info, onew, oinfo, margins)
    n, d = oinfo.num_integration_steps, oinfo.num_trajectory_expansions
    if eps >= 100:                                       # the divergent case: every chain stops on its first leaf
        assert (n == 1).all() and oinfo.is_divergent.all()
    elif SLOTS[size_class_for(D)] >= 8 and md > 4:       # past the fused doublings: the compacted-list launches run
        assert d.max() > 4
    if kind == "std":
        assert (n == 2 ** md - 1).all()


@pytest.mark.parametrize("D, depth", EXACT_CASES)
def test_nuts_exact_trajectories_every_chain_identical(D, depth):
    """NUTS on trajectories that float32 represents exactly, so that every U-turn product is computed without rounding
    on both sides and chains may not disagree on a tie.  At step size 1 the Gaussian coordinates of precision 2 rotate
    (q, p) -> (p, -q) and those of precision 1 follow p_{n+2} = p_{n+1} - p_n: integer and quarter-integer values only.
    Coordinates of precision 2 start at q = 0 and those of precision 1 at p = 0, so the momentum at leaf 3 in either
    direction is exactly zero while no U-turn has fired before it: a checkpoint U-turn product that is exactly 0, which
    the reference's `<=` counts as a turn (termination.py:96-103)."""
    rs = np.random.default_rng(D)
    C, md = 64, 3
    x = np.arange(D) % 2 == 0
    prec = np.where(x, 2.0, 1.0)
    tgt, otgt = T.DiagGaussian(1.0 / np.sqrt(prec)), otargets.DiagGaussian(1.0 / np.sqrt(prec))
    assert (otgt.inv_var == prec).all()
    active = (np.arange(D) < 6) | (np.arange(D) >= D - 2)   # a few coordinates: first and last slots of the row
    k = rs.integers(1, 4, (C, D)) * rs.choice([-1, 1], (C, D)) * active
    p0 = np.where(x, k, 0).astype(F)
    q0 = np.where(x, 0, 4 * k).astype(F)
    keys = oprng.split(oprng.key(D + 1), C)
    margins = np.full(C, np.inf)
    imm = np.ones(D, F)
    onew, oinfo = onuts.nuts_kernel(keys, ohmc.init(q0, otgt), otgt, F(1.0), imm, md, momentum=p0, key_integrator=keys,
                                    margins=margins)
    kern = bj.nuts.build_kernel(full_info=True, max_tree_depth=depth)
    new, info = kern(None, bj.nuts.init(tf(q0), tgt), tgt, 1.0, tf(imm), md, _momentum=tf(p0), _key_integrator=tk(keys))
    torch.cuda.synchronize()
    assert (margins == 0).mean() > 0.3                   # exact U-turn ties do decide trees here
    np.testing.assert_array_equal(npy(info.num_integration_steps), oinfo.num_integration_steps)
    np.testing.assert_array_equal(npy(info.num_trajectory_expansions), oinfo.num_trajectory_expansions)
    np.testing.assert_array_equal(npy(info.is_turning), oinfo.is_turning)
    np.testing.assert_array_equal(npy(new.position), onew.position)
    np.testing.assert_array_equal(npy(info.trajectory_leftmost_state.momentum), oinfo.trajectory_leftmost_state[1])
    np.testing.assert_array_equal(npy(info.trajectory_rightmost_state.momentum), oinfo.trajectory_rightmost_state[1])


# ---------------------------------------------------------------------------------------------------------------------
# more than 10 doublings, and the decoupled sampler
# ---------------------------------------------------------------------------------------------------------------------
def stepwise(key, st0, tgt, eps, imm, T_, md, depth, thin=1):
    """T_ calls of the step-wise kernel with run_inference_algorithm's step keys: (final state, history, acceptance
    rates, tree sizes)."""
    kern = bj.nuts.build_kernel(max_tree_depth=depth)
    keys = bj.random.split(key, T_)
    st = bj.nuts.init(st0.position.clone(), tgt)
    hist, acc, n_int = [], [], []
    for t in range(T_):
        st, info = kern(keys[t], st, tgt, eps, imm, md)
        if (t + 1) % thin == 0:
            hist.append(st.position)
        acc.append(info.acceptance_rate)
        n_int.append(info.num_integration_steps)
    return st, torch.stack(hist), torch.stack(acc), torch.stack(n_int)


def assert_native_equals_stepwise(key, st0, tgt, eps, imm, T_, md, depth, thin=1):
    fin, hist, acc, n_int = bj.sample_nuts_native(key, st0, tgt, eps, imm, T_, max_num_doublings=md, thin=thin)
    st, shist, sacc, sn = stepwise(key, st0, tgt, eps, imm, T_, md, depth, thin)
    assert torch.equal(n_int, sn) and torch.equal(acc, sacc) and torch.equal(hist, shist)
    assert torch.equal(fin.position, st.position) and torch.equal(fin.logdensity, st.logdensity)
    assert torch.equal(fin.logdensity_grad, st.logdensity_grad)
    return sn


@pytest.mark.parametrize("md", [11, 12])
def test_nuts_beyond_ten_doublings(md):
    """Trees of 2^11 - 1 and 2^12 - 1 leaves: step-wise against the oracle, and the decoupled sampler (whose key schedule
    covers 10 doublings per call) bit for bit against the step-wise calls."""
    D, C, eps = 8, 16, 5e-4
    rs = np.random.default_rng(md)
    tgt, otgt = T.StdNormal(D), otargets.StdNormal(D)
    q = rs.standard_normal((C, D)).astype(F)
    imm = np.ones(D, F)
    keys = oprng.split(oprng.key(md), C)
    margins = np.full(C, np.inf)
    onew, oinfo = onuts.nuts_kernel(keys, ohmc.init(q, otgt), otgt, F(eps), imm, md, margins=margins)
    assert (oinfo.num_integration_steps == 2 ** md - 1).all()
    new, info = bj.nuts.build_kernel(full_info=True, max_tree_depth=md)(tk(keys), bj.nuts.init(tf(q), tgt), tgt, eps,
                                                                         tf(imm), md)
    torch.cuda.synchronize()
    compare_nuts(new, info, onew, oinfo, margins)
    n = assert_native_equals_stepwise(bj.random.key(md, DEV), bj.nuts.init(tf(q), tgt), tgt, eps, tf(imm), 4, md, md)
    assert int(n.min()) == 2 ** md - 1


@pytest.mark.parametrize("D, C, T_, md, depth, thin, pce, metric", [
    (512, 37, 4, 6, 10, 1, False, "diag"),       # C not a multiple of 4
    (1024, 3001, 4, 5, 10, 1, False, "diag"),    # more chains than resident warps: warps take several from the queue
    (512, 301, 6, 6, 10, 2, True, "per_chain"),  # thin > 1, per-chain step size and metric
    (1024, 66, 5, 7, 10, 3, True, "diag"),
    (512, 130, 4, 2, 10, 1, False, "diag"),      # step-wise checkpoints global (engine depth 10), native in shared memory
])
def test_native_nuts_sampler_wide_rows(D, C, T_, md, depth, thin, pce, metric):
    if md == 2:   # bjx_nuts_sample applies the rule with max_num_doublings, bjx_nuts_step with the engine's depth
        assert ckpt_in_smem(D, md, False) and not ckpt_in_smem(D, depth, False)
    rs = np.random.default_rng(C)
    tgt = T.Funnel(D)
    q = (0.3 * rs.standard_normal((C, D))).astype(F)
    q[:, 0] = rs.uniform(-1, 1, C)
    dm, _ = make_metric(metric, D, C, rs)
    eps = tf((0.1 * np.exp(rs.uniform(-0.5, 0.5, C))).astype(F)) if pce else 0.1
    n = assert_native_equals_stepwise(bj.random.key(D + C, DEV), bj.nuts.init(tf(q), tgt), tgt, eps, dm, T_, md, depth,
                                      thin)
    assert len(torch.unique(n)) >= min(3, md)
