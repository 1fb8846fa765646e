"""Barker's proposal (blackjax/mcmc/barker.py:73-159,230-282, metrics.py:306-344,701-729, util.py:66-91) restated in
float32 NumPy for a batch of chains, with the decision margins: |u - p_accept| per chain and min_i |u_i - p_i| over the
sign draws."""
import numpy as np

from . import prng

F = np.float32


def log1pexp(a):
    """barker.py:285-286, naive: inf when exp overflows."""
    with np.errstate(over="ignore"):
        return np.log1p(np.exp(a)).astype(F)


class Metric:
    """gaussian_euclidean's scale (metrics.py:306-344): M^1/2 and M^-1/2 of an inverse mass matrix [D], [C, D] (one
    diagonal per chain) or [D, D] (dense: M^-1/2 = L = chol(M^-1), M^1/2 = L^-T)."""

    def __init__(self, inverse_mass_matrix, n_chains):
        imm = np.asarray(inverse_mass_matrix, F)
        self.imm = imm
        self.dense = imm.ndim == 2 and imm.shape[0] == imm.shape[1] and imm.shape[0] != n_chains
        if self.dense:
            L = np.linalg.cholesky(imm.astype(np.float64))
            self.inv_sqrt = L.astype(F)
            self.sqrt = np.linalg.solve(L.T, np.eye(L.shape[0])).astype(F)
        else:
            self.inv_sqrt = np.sqrt(imm).astype(F)
            self.sqrt = (F(1.0) / self.inv_sqrt).astype(F)

    def scale(self, v, inv, trans):
        m = self.inv_sqrt if inv else self.sqrt
        if self.dense:
            m = m.T if trans else m
            return (v @ m.T).astype(F)
        return (m * v).astype(F)

    def kinetic(self, v):
        vel = (v @ self.imm.T).astype(F) if self.dense else (self.imm * v).astype(F)
        return (F(0.5) * np.sum(vel * v, axis=-1, dtype=F)).astype(F)


def sample(keys, x, g, step_size, metric):
    """_barker_sample (barker.py:230-282) for every chain: (proposal, the sign draws' margins |u_i - p_i| [C, D])."""
    C, D = x.shape
    eps = np.broadcast_to(np.asarray(step_size, F), (C,)).astype(F)[:, None]
    k = prng.split(keys)                            # key1, key2
    z = (eps * prng.normal(k[:, 0], (D,))).astype(F)
    c = metric.scale(g, inv=False, trans=True)
    with np.errstate(over="ignore"):
        p = np.exp(-log1pexp((-c * z).astype(F))).astype(F)
    u = prng.uniform(prng.split(k[:, 1], 1)[:, 0], (D,))
    b = u < p
    bz = np.where(b, z, -z).astype(F)
    y = (x + metric.scale(bz, inv=False, trans=False)).astype(F)
    return y, np.abs(u - p)


def log_p_accept(x, logp_x, g_x, y, logp_y, g_y, metric):
    """_compute_acceptance_probability (barker.py:80-128) in the reference's order, NaN kept."""
    D = x.shape[-1]
    with np.errstate(all="ignore"):
        y_minus_x = (y - x).astype(F)
        x_minus_y = -y_minus_x
        zt_xy = metric.scale(y_minus_x, inv=True, trans=True)
        zt_yx = metric.scale(x_minus_y, inv=True, trans=True)
        c_x = metric.scale(g_x, inv=False, trans=True)
        c_y = metric.scale(g_y, inv=False, trans=True)
        s_yx = np.sum(log1pexp((-zt_yx * c_y).astype(F)), axis=-1, dtype=F)
        s_xy = np.sum(log1pexp((-zt_xy * c_x).astype(F)), axis=-1, dtype=F)
        n = F(D)
        ratio = ((((n * metric.kinetic(x_minus_y)).astype(F) - s_yx).astype(F) - (n * metric.kinetic(y_minus_x)).astype(F))
                 .astype(F) + s_xy).astype(F)
        return ((logp_y - logp_x).astype(F) + ratio).astype(F)


def step(keys, q, logp, g, logdensity_fn, step_size, inverse_mass_matrix=None):
    """One transition of every chain.  keys [C, 2]; step_size scalar or [C]; inverse_mass_matrix None (ones), [D],
    [C, D] or dense [D, D].  Returns ((q, logp, g), info) with acceptance_rate, is_accepted, the proposal (position,
    logdensity, grad), margin = |u - p_accept|, sign_margins = |u_i - p_i| and sign_margin = their minimum."""
    q, logp, g = (np.asarray(a, F) for a in (q, logp, g))
    C, D = q.shape
    metric = Metric(np.ones(D, F) if inverse_mass_matrix is None else inverse_mass_matrix, C)
    ks = prng.split(keys)                              # key_sample, key_rmh  barker.py:147
    y, sign_margins = sample(ks[:, 0], q, g, step_size, metric)
    logp_y, g_y = logdensity_fn(y)
    logp_y, g_y = np.asarray(logp_y, F), np.asarray(g_y, F)
    la = log_p_accept(q, logp, g, y, logp_y, g_y, metric)
    with np.errstate(all="ignore"):
        p = np.where(np.isnan(la), F(np.nan), np.minimum(np.exp(la), F(1.0))).astype(F)  # clip keeps NaN
    u = prng.uniform(ks[:, 1])
    acc = u < p
    out = (np.where(acc[:, None], y, q), np.where(acc, logp_y, logp), np.where(acc[:, None], g_y, g))
    return out, dict(acceptance_rate=p, is_accepted=acc, proposal=(y, logp_y, g_y), margin=np.abs(u - p),
                     sign_margin=sign_margins.min(axis=-1), sign_margins=sign_margins)
