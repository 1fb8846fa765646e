"""Slice sampling on the GPU: one teacher-forced transition against the float32 oracle (oracle/slice_sampling.py) in
every row size class and on the CTA rows; the caps; the bounded Gaussian; the native loops bit-identical to step calls on
both routes; chain_offset and plug-in bit identity; the rejections; and moments within 5 MCSE.

is_accepted, num_expansions and num_shrink must match the oracle exactly except on chains where one of the oracle's
in-slice tests was a tie (the oracle's margin covers every eager evaluation): |logp - level| below TIE_REL * (1 + |level| + D), twice that with a dense scale.  The
direction's norm is summed in another order on the device (and the dense scale's matvec too), which moves the points
x + t d, and so their log-densities, by about 1e-7 to 1e-6 of the size of their terms."""
import numpy as np
import pytest
import torch

import blackjax_b200 as bj
from blackjax_b200 import _lib
from blackjax_b200.mcmc import slice as sl
from oracle import prng as oprng
from oracle import slice_sampling as osl
from oracle import targets as otargets
from test_gpu_parity import close, make_target, npy, tf, tk

pytestmark = pytest.mark.gpu
F = np.float32
TIE_REL = 3e-6
INTERVALS = {"doubling": sl.doubling, "stepping_out": sl.stepping_out}


def make_scale(kind, D, rs):
    if kind == "scalar":
        return F(1.7)
    if kind == "vec":
        return np.exp(rs.uniform(-0.5, 0.5, D)).astype(F)
    A = rs.standard_normal((D, D))
    return np.linalg.cholesky(A @ A.T / D + 0.5 * np.eye(D)).astype(F)


def run_step(tgt, q, keys, scale, width, interval, me=10, ms=100, inplace=False):
    st = sl.init(tf(q), tgt)
    l0 = npy(st.logdensity)
    s = scale if np.ndim(scale) == 0 else tf(scale)
    w = width if np.ndim(width) == 0 else tf(width)
    kern = sl.build_kernel(INTERVALS[interval], me, ms, inplace=inplace)
    new, info = kern(tk(keys), st, tgt, sl.direction_proposal(s), w)
    torch.cuda.synchronize()
    if inplace:
        assert new.position.data_ptr() == st.position.data_ptr()
    return npy(new.position), npy(new.logdensity), {k: npy(v) for k, v in info._asdict().items()}, l0


def compare(keys, q, l0, otgt, scale, width, interval, got, me=10, ms=100, dense=False):
    qd, ld, info, _ = got
    C, D = q.shape
    (qo, lo), oi = osl.step(keys, q, l0, otgt, scale, width, interval, me, ms)
    with np.errstate(divide="ignore"):
        lvl = np.abs(l0.astype(np.float64) + np.log(oprng.uniform(oprng.split(oprng.split(keys)[:, 1], 3)[:, 0])))
    tie = TIE_REL * (2.0 if dense else 1.0) * (1.0 + np.where(np.isfinite(lvl), lvl, 0.0) + D)
    ok = oi["margin"] > tie
    # the oracle's margins cover every eager evaluation, decisive or not, so they flag more chains than can differ
    assert ok.mean() >= 0.6, f"{(~ok).sum()} of {C} chains tie"
    for k in ("num_expansions", "num_shrink"):
        np.testing.assert_array_equal(info[k][ok], oi[k][ok], err_msg=k)
    np.testing.assert_array_equal(info["is_accepted"][ok], oi["is_accepted"][ok])
    close(info["bracket_left"][ok], oi["bracket_left"][ok], scale=1.0)
    close(info["bracket_right"][ok], oi["bracket_right"][ok], scale=1.0)
    for c in np.nonzero(ok)[0]:
        close(qd[c], qo[c])
    close(ld[ok], lo[ok], scale=np.abs(lo[ok]).max() + D)
    return oi, ok


# (target, D, scale, interval, width, in place): every row size class and the CTA rows
CASES = [("std", 1, "scalar", "doubling", "scalar", False), ("banana", 2, "dense", "stepping_out", "chain", True),
         ("funnel", 3, "vec", "doubling", "chain", False), ("diag", 31, "dense", "doubling", "scalar", True),
         ("funnel", 33, "vec", "stepping_out", "scalar", False), ("dense", 127, "dense", "doubling", "chain", False),
         ("diag", 4, "scalar", "stepping_out", "scalar", False), ("dense", 128, "vec", "doubling", "scalar", True),
         ("diag", 128, "dense", "stepping_out", "chain", False), ("funnel", 132, "vec", "doubling", "scalar", False),
         ("diag", 256, "scalar", "stepping_out", "chain", True), ("std", 260, "vec", "doubling", "scalar", False),
         ("funnel", 512, "vec", "doubling", "chain", False), ("diag", 516, "scalar", "stepping_out", "scalar", False),
         ("diag", 1024, "vec", "doubling", "scalar", True), ("funnel", 1024, "scalar", "stepping_out", "chain", False),
         ("diag", 1028, "vec", "doubling", "chain", False), ("funnel", 2048, "scalar", "stepping_out", "scalar", True),
         ("std", 18432, "vec", "doubling", "scalar", False)]


def start(kind, D, rs):
    q = (0.5 * rs.standard_normal((1, D))).astype(F)
    if kind == "funnel":
        q[:, 0] = 0.0
    return q


@pytest.mark.parametrize("kind, D, scale_kind, interval, width_kind, inplace", CASES)
def test_single_transition_matches_oracle(kind, D, scale_kind, interval, width_kind, inplace):
    rs = np.random.default_rng(D + len(kind))
    C = 128 if D <= 1024 else 24
    tgt, otgt = make_target(kind, D, rs)
    scale = make_scale(scale_kind, D, rs)
    width = F(1.3) if width_kind == "scalar" else rs.uniform(0.5, 2.0, C).astype(F)
    q = np.concatenate([start(kind, D, rs) for _ in range(C)])
    keys = oprng.split(oprng.key(D), C)
    got = run_step(tgt, q, keys, scale, width, interval, inplace=inplace)
    compare(keys, q, got[3], otgt, scale, width, interval, got, dense=scale_kind == "dense")


def test_hier_logit_10000_matches_oracle():
    C, D = 6, 10000
    x, bits = bj.targets.HierLogit.synthetic_data(D - 4, seed=1)
    tgt, otgt = bj.targets.HierLogit(x, bits), otargets.HierLogit(x, bits)
    rs = np.random.default_rng(3)
    q = (0.3 * rs.standard_normal((C, D))).astype(F)
    keys = oprng.split(oprng.key(4), C)
    scale = np.full(D, 0.5, F)
    got = run_step(tgt, q, keys, scale, F(0.5), "doubling")
    compare(keys, q, got[3], otgt, scale, F(0.5), "doubling", got)


@pytest.mark.parametrize("me, ms", [(0, 100), (1, 100), (10, 0), (10, 1), (0, 1)])
@pytest.mark.parametrize("D, interval", [(64, "doubling"), (64, "stepping_out"), (2048, "doubling")])
def test_caps_match_oracle(me, ms, D, interval):
    """With max_shrinkage 0 or 1 many chains find no point: they keep their state bit for bit and report
    is_accepted = 0."""
    rs = np.random.default_rng(7)
    C = 128 if D <= 1024 else 16
    tgt, otgt = bj.targets.DiagGaussian(np.full(D, 0.3)), otargets.DiagGaussian(np.full(D, 0.3))
    q = (0.3 * rs.standard_normal((C, D))).astype(F)
    keys = oprng.split(oprng.key(9), C)
    got = run_step(tgt, q, keys, F(1.0), F(2.0), interval, me, ms)
    compare(keys, q, got[3], otgt, F(1.0), F(2.0), interval, got, me, ms)
    ex = ~got[2]["is_accepted"].astype(bool)
    if ms == 0:
        assert ex.all() and (got[2]["num_shrink"] == 0).all()
    np.testing.assert_array_equal(got[0][ex], q[ex])
    np.testing.assert_array_equal(got[1][ex], got[3][ex])


def test_bounded_gaussian_plugin():
    """The box at +-2: NaN log-densities outside are never in the slice, no chain leaves the box, and the truncated
    normal's moments come out within 5 MCSE."""
    from blackjax_b200 import plugin
    from scipy import stats
    D, C, T_ = 2, 4096, 200
    B = 2.0
    tgt = bj.targets.UserTarget(D, plugin.read_example("bounded_gaussian"), np.array([B], F), name="bounded_gaussian")
    q = tf(np.zeros((C, D), F))
    st = sl.init(q, tgt)
    _, hist, _, _ = bj.sample_slice_sampling_native(tk(oprng.key(3)), st, tgt, T_, width=3.0)
    h = npy(hist)
    assert np.all(np.abs(h) < B)
    # the density exp(-x^2/2) (B - |x|) per axis, by quadrature
    xs = np.linspace(-B, B, 200001)
    w = np.exp(-0.5 * xs ** 2) * (B - np.abs(xs))
    w /= w.sum()
    var = float(np.sum(w * xs ** 2))
    mcse_check(hist[20:].contiguous(), np.zeros(D), np.full(D, var), tgt)


def stepwise(key, st, tgt, scale, width, interval, T_, thin, chain_offset):
    kern = sl.build_kernel(INTERVALS[interval], chain_offset=chain_offset)
    prop = sl.direction_proposal(scale)
    hist, ne, ns = [], [], []
    for t, k in enumerate(oprng.split(key, T_)):
        st, info = kern(tk(k), st, tgt, prop, width)
        ne.append(npy(info.num_expansions))
        ns.append(npy(info.num_shrink))
        if (t + 1) % thin == 0:
            hist.append(npy(st.position))
    return st, np.stack(hist), np.stack(ne), np.stack(ns)


@pytest.mark.parametrize("D, scale_kind, interval", [(100, "vec", "doubling"), (64, "dense", "stepping_out"),
                                                     (2048, "vec", "doubling"), (1028, "scalar", "stepping_out")])
def test_native_loop_bit_identical_to_steps(D, scale_kind, interval):
    rs = np.random.default_rng(5)
    C, T_, thin, off = 40, 10, 3, 7
    tgt, _ = make_target("diag", D, rs)
    scale = make_scale(scale_kind, D, rs)
    scale = scale if np.ndim(scale) == 0 else tf(scale)
    width = tf(rs.uniform(0.5, 2.0, C).astype(F))
    q = tf((0.5 * rs.standard_normal((C, D))).astype(F))
    key = oprng.key(21)
    st0 = sl.init(q, tgt)
    ref, h_ref, e_ref, s_ref = stepwise(key, st0, tgt, scale, width, interval, T_, thin, off)
    ev = torch.zeros(1, dtype=torch.uint64, device="cuda")
    fin, hist, ne, ns = bj.sample_slice_sampling_native(tk(key), st0, tgt, T_, scale=scale, width=width,
                                                        interval=INTERVALS[interval], thin=thin, chain_offset=off,
                                                        evaluations=ev)
    np.testing.assert_array_equal(npy(fin.position), npy(ref.position))
    np.testing.assert_array_equal(npy(fin.logdensity), npy(ref.logdensity))
    np.testing.assert_array_equal(npy(hist), h_ref)
    np.testing.assert_array_equal(npy(ne), e_ref)
    np.testing.assert_array_equal(npy(ns), s_ref)
    n_ev = int(ev.cpu().item())
    lo = int(s_ref.sum()) + (2 * C * T_ if interval == "doubling" else 0)
    assert n_ev >= lo, (n_ev, lo)


def test_chain_offset_split_matches_one_handle():
    rs = np.random.default_rng(8)
    D, C = 96, 64
    tgt, _ = make_target("diag", D, rs)
    q = tf((0.5 * rs.standard_normal((C, D))).astype(F))
    key = tk(oprng.key(3))
    whole = bj.sample_slice_sampling_native(key, sl.init(q, tgt), tgt, 6)
    for lo in (0, 32):
        part = bj.sample_slice_sampling_native(key, sl.init(q[lo:lo + 32].clone(), tgt), tgt, 6, chain_offset=lo)
        assert torch.equal(part[0].position, whole[0].position[lo:lo + 32])
        assert torch.equal(part[1], whole[1][:, lo:lo + 32])
        assert torch.equal(part[2], whole[2][:, lo:lo + 32]) and torch.equal(part[3], whole[3][:, lo:lo + 32])


def test_plugins_match_builtin():
    from blackjax_b200 import plugin
    for D, src in ((100, "diag_gaussian"), (2048, "diag_gaussian_big")):
        C = 32
        user = bj.targets.UserTarget(D, plugin.read_example(src), np.ones(D, F), name=src)
        builtin = bj.targets.StdNormal(D)
        q = tf(np.random.default_rng(D).standard_normal((C, D)).astype(F))
        key = tk(oprng.key(5))
        a = bj.sample_slice_sampling_native(key, sl.init(q.clone(), builtin), builtin, 6, scale=0.8)
        b = bj.sample_slice_sampling_native(key, sl.init(q.clone(), user), user, 6, scale=0.8)
        assert torch.equal(a[0].position, b[0].position) and torch.equal(a[1], b[1]) and torch.equal(a[2], b[2])


def test_rejections():
    from blackjax_b200._engine import get_engine
    C = 4
    k = tk(oprng.split(oprng.key(0), C))
    tgt = bj.targets.StdNormal(8)
    st = sl.init(tf(np.zeros((C, 8), F)), tgt)
    eng = get_engine(st.position, tgt)
    with pytest.raises(_lib.BjxError, match="needs a direction scale"):
        eng.slice_step(k, *st, 1.0, 0, 10, 100)
    eng.ensure_slice_scale(1.0)
    for args, msg in (((0.0, 0, 10, 100), "width"), ((float("inf"), 0, 10, 100), "width"),
                      ((1.0, 0, -1, 100), ">= 0"), ((1.0, 0, 10, -1), ">= 0"), ((1.0, 2, 10, 100), "interval")):
        with pytest.raises(_lib.BjxError, match=msg):
            eng.slice_step(k, *st, *args)
    D = 132  # a dense scale beyond 128 dims
    tgt = bj.targets.StdNormal(D)
    st = sl.init(tf(np.zeros((C, D), F)), tgt)
    with pytest.raises(_lib.BjxError, match="dim <= 128"):
        sl.build_kernel()(k, st, tgt, sl.direction_proposal(tf(np.eye(D, dtype=F))))
    D = 256  # the tensor-core dense target path
    A = np.random.default_rng(1).standard_normal((D, D))
    tgt = bj.targets.DenseGaussian(A @ A.T / D + np.eye(D))
    st = sl.init(tf(np.zeros((C, D), F)), tgt)
    with pytest.raises(_lib.BjxError, match="tensor-core dense target path"):
        sl.build_kernel()(k, st, tgt, sl.direction_proposal())


def mcse_check(h, mean, var, tgt):
    from blackjax_b200.diagnostics import effective_sample_size
    x = h.double()
    mt = torch.as_tensor(np.array(mean), device=x.device).double()
    d2 = (x - mt) ** 2
    ess = effective_sample_size(h, tgt).double()
    ess2 = effective_sample_size(d2.float().contiguous(), tgt).double()
    zm = ((x.mean(dim=(0, 1)) - mt).abs() / (x.std(dim=(0, 1)) / ess.sqrt())).cpu().numpy()
    zv = ((d2.mean(dim=(0, 1)) - torch.as_tensor(np.array(var), device=x.device).double()).abs()
          / (d2.std(dim=(0, 1)) / ess2.sqrt())).cpu().numpy()
    assert zm.max() < 5, zm.max()
    assert zv.max() < 5, zv.max()


@pytest.mark.parametrize("interval", ["doubling", "stepping_out"])
def test_moments_std_normal_and_correlated(interval):
    C, T_ = 2048, 200
    tgt = bj.targets.StdNormal(3)
    st = sl.init(tf(np.random.default_rng(0).standard_normal((C, 3)).astype(F)), tgt)
    _, h, _, _ = bj.sample_slice_sampling_native(tk(oprng.key(1)), st, tgt, T_, interval=INTERVALS[interval])
    mcse_check(h, np.zeros(3), np.ones(3), tgt)
    sigma = np.array([[1.0, 0.8], [0.8, 1.0]])
    tgt = bj.targets.DenseGaussian(np.linalg.inv(sigma))
    x0 = np.random.default_rng(1).standard_normal((C, 2)) @ np.linalg.cholesky(sigma).T
    st = sl.init(tf(x0.astype(F)), tgt)
    _, h, _, _ = bj.sample_slice_sampling_native(tk(oprng.key(2)), st, tgt, T_,
                                                 scale=tf(np.linalg.cholesky(sigma).astype(F)),
                                                 interval=INTERVALS[interval])
    mcse_check(h, np.zeros(2), np.ones(2), tgt)


def test_funnel_neck_128():
    """Neal's funnel at D = 128 from exact draws: the neck variable v ~ N(0, 9) and x_i | v ~ N(0, e^v)."""
    C, T_, D = 4096, 100, 128
    rs = np.random.default_rng(4)
    v = 3.0 * rs.standard_normal(C)
    x = rs.standard_normal((C, D - 1)) * np.exp(v / 2)[:, None]
    q = np.concatenate([v[:, None], x], axis=1).astype(F)
    tgt = bj.targets.Funnel(D)
    st = sl.init(tf(q), tgt)
    _, h, _, _ = bj.sample_slice_sampling_native(tk(oprng.key(6)), st, tgt, T_)
    mcse_check(h[:, :, :1].contiguous(), np.zeros(1), np.full(1, 9.0), bj.targets.StdNormal(1))
