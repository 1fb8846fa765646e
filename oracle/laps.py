"""NumPy restatement of LAPS (blackjax/adaptation/laps.py, laps_burn_in.py, eca.py, bisection_monotonic_fn of
adaptation/step_size.py:262-304), batched over chains, on top of the MCLMC and MAMS oracles (oracle/mclmc.py,
oracle/adjusted_mclmc.py) and oracle/prng.py.  Ensemble averages are float64 sums divided by N, rounded to float32."""
import numpy as np

from . import adjusted_mclmc as oa
from . import mclmc as om
from . import prng as oprng

F = np.float32
VV = (0.5, 1.0, 0.5)


def sampling_keys(phase_key, N, T, t, chain_offset=0):
    """split(key_sampling, (N, T))[:, t] with key_sampling = split(phase_key)[0]."""
    ks = oprng.split(phase_key, 2)[0]
    return oprng.fold_in(ks, (np.arange(N, dtype=np.uint64) + chain_offset) * T + t)


def adaptation_key(phase_key, t):
    return oprng.fold_in(oprng.split(phase_key, 2)[1], t)


def rademacher(key, shape):
    """jax.random.rademacher = 2 bernoulli(key, 0.5, shape) - 1."""
    return (2 * (oprng.uniform(key, shape) < F(0.5)).astype(np.int32) - 1).astype(F)


def initialize(q, target):
    """laps_burn_in.initialize after sample_init: (q, u, logp, g), and the signs."""
    q = np.asarray(q, F)
    logp, g = target(q)
    n = np.sqrt(np.sum(g.astype(np.float64) ** 2, axis=1)).astype(F)
    u = np.where((n > F(1e-13))[:, None], g / n[:, None], g).astype(F)
    E = np.mean((-q * g).astype(np.float64), axis=0).astype(F)
    signs = (F(-2.0) * (E < F(1.0)) + F(1.0)).astype(F)
    return (q, (u * signs).astype(F), logp, g), signs


class BurnIn:
    """The burn-in's adaptation state (laps_burn_in.py:256-272) with a history of save_num rows, newest first."""

    def __init__(self, D, save_num):
        self.D, self.save_num = D, save_num
        self.L, self.eps = F(np.inf), F(F(0.01) * np.sqrt(F(D)))
        self.count = 0
        self.hist = np.zeros((save_num, D), F)
        self.w = np.zeros(save_num, F)


def burn_in_kernel(keys, state, target, L, eps):
    """sequential_kernel (laps_burn_in.py:54-76): MCLMC with velocity Verlet, M^-1 = 1, then nan_reject."""
    new, info = om.mclmc_kernel(keys, state, target, np.ones(state[0].shape[1], F), L, eps, VV)
    ok = info.nonans
    kept = tuple(np.where(ok[:, None] if n.ndim == 2 else ok, n, o).astype(F) for n, o in zip(new, state))
    return kept, info


def summaries(state, info):
    """Etheta without equipartition_fullrank: the ensemble means of the summary statistics."""
    q, _, _, g = state
    ok = info.nonans.astype(F)
    E = (info.energy_change * ok).astype(F)
    m = lambda x: np.mean(np.asarray(x, np.float64), axis=0).astype(F)
    return {"equipartition_diagonal": m(-q * g), "x": m(q), "xsq": m(q * q), "E": m(E), "Esq": m(E * E),
            "nans": m(1 - ok), "entropy": m(-(info.logdensity * ok))}


def equi_full(state, key):
    """equipartition_fullrank_loss of the ensemble mean of Z + (Z g) x^T (float64)."""
    q, _, _, g = (np.asarray(x, np.float64) for x in state)
    Z = rademacher(key, (100, q.shape[1])).astype(np.float64)
    M = Z + (Z @ g.T) @ q / q.shape[0]
    return float(np.mean(M * M) / q.shape[1])


def contract_history(theta, weights):
    theta, weights = np.asarray(theta, np.float64), np.asarray(weights, np.float64)
    a = np.sum(theta * weights[:, None], 0) / weights.sum()
    a2 = np.sum(theta * theta * weights[:, None], 0) / weights.sum()
    r = (a2 - a * a) / (a * a)
    return np.array([np.max(r), np.mean(r)])


def update_history(new, history):
    return np.concatenate([np.asarray(new)[None], history[:-1]])


def update(ad, Et, alpha, C, bias_type, equi_full_value=np.nan):
    """Adaptation.update (laps_burn_in.py:292-364); returns (info row, imm) and updates ad in place."""
    D = ad.D
    equi_diag = float(np.mean((1.0 - np.float64(Et["equipartition_diagonal"])) ** 2))
    ad.hist = update_history(Et["x"], ad.hist)
    ad.w = update_history(F(1), ad.w)
    r_max, r_avg = contract_history(ad.hist, ad.w)
    imm = (Et["xsq"] - (Et["x"] * Et["x"]).astype(F)).astype(F)  # float32, as the reference forms them
    L = alpha * np.sqrt(np.mean(imm, dtype=np.float64)) * np.sqrt(D)
    eevpd = np.float64((Et["Esq"] - (Et["E"] * Et["E"]).astype(F)).astype(F)) / D
    bias = [r_max, r_avg, equi_full_value, equi_diag][bias_type]
    wanted = C * bias ** 0.375
    with np.errstate(invalid="ignore", divide="ignore"):
        f = (wanted / eevpd) ** (1.0 / 6.0)
    f = np.nan if np.isnan(f) else min(max(f, 0.3), 3.0)
    if Et["nans"] > 0:
        f = 0.5
    row = {"L": ad.L, "step_size": ad.eps, "EEVPD_wanted": wanted, "EEVPD": eevpd, "equi_diag": equi_diag,
           "equi_full": equi_full_value, "r_max": r_max, "r_avg": r_avg, "entropy": float(Et["entropy"])}
    ad.L, ad.eps, ad.count = F(L), F(ad.eps * f), ad.count + 1
    return row, imm.astype(F)


def stop_index(r_max, save_num, r_end, num_steps):
    """Number of burn-in steps run (eca.py:119-156, laps_burn_in.py:366-368).  r_max[t] is step t's; the loop's first
    condition is evaluated on a probe of step 0, which decides alone when save_num = 0."""
    cond = lambda r, t: (r > r_end) or (t < save_num)
    if not cond(r_max[0], 0):
        return 0
    for t in range(num_steps):
        if not cond(r_max[t], t):
            return t + 1
    return num_steps


def bisection(target, shift=np.log(2.0), tol=0.03):
    """bisection_monotonic_fn (step_size.py:262-304) in float64: update(state, eps, acc) -> (state, eps)."""

    def upd(state, exp_x, acc):
        (lo, hi), term = state
        x = np.log(exp_x)
        if acc > target:
            lo = max(lo, x)
            xn = lo + shift
        else:
            hi = min(hi, x)
            xn = hi - shift
        if np.isfinite(lo) and np.isfinite(hi):
            xn = (lo + hi) / 2
        eps = term * exp_x + (1 - term) * np.exp(xn)
        return ((lo, hi), bool(abs(acc - target) < tol) or term), eps

    return upd


def adjusted_kernel(keys, state, target, imm, eps, steps_per_sample, coefficients):
    return oa.adjusted_mclmc_kernel(keys, state, target, imm, eps, steps_per_sample, coefficients, L_proposal_factor=1.25)
