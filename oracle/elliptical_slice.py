"""Elliptical slice sampling (blackjax/mcmc/elliptical_slice.py:76-262, util.py:66-91) restated in float32 NumPy for a
batch of chains, with the sub-iteration cap of the device kernels (``max_subiter``), and for every chain the smallest
margin |logL(p) - logy| over its loop decisions, so that a test can tell a disagreement from a tie."""
import numpy as np

from . import prng

F = np.float32
TWO_PI = F(2 * np.pi)  # 2 * jnp.pi is weakly typed: the float32 6.2831855


def prior_scale(cov):
    """sqrt(cov) of a 1-D cov, chol(cov) of a 2-D one (formed in float64, as the host does), else the reference's
    ValueError (elliptical_slice.py:94-105)."""
    cov = np.asarray(cov)
    if cov.ndim == 1:
        return np.sqrt(cov.astype(F)).astype(F)
    if cov.ndim == 2:
        return np.linalg.cholesky(cov.astype(F).astype(np.float64)).astype(F)
    raise ValueError("The mass matrix has the wrong number of dimensions:"
                     f" expected 1 or 2, got {cov.ndim}.")


def momentum(keys, mean, scale, D):
    """nu = mean + S normal(key_momentum, (D,)) with key_momentum = split(key, 4)[1] (util.py:66-91)."""
    z = prng.normal(prng.split(keys, 4)[:, 1], (D,))
    if scale.ndim == 1:
        lz = (scale * z).astype(F)
    else:
        lz = (z.astype(np.float64) @ scale.astype(np.float64).T).astype(F)
    return (mean + lz).astype(F)


def ellipse(a, b, mean, theta):
    """(a - mean) cos(theta) + (b - mean) sin(theta) + mean, per chain theta [C] (elliptical_slice.py:265-300)."""
    c = np.cos(theta.astype(F)).astype(F)[:, None]
    s = np.sin(theta.astype(F)).astype(F)[:, None]
    return ((((a - mean).astype(F) * c).astype(F) + ((b - mean).astype(F) * s).astype(F)).astype(F) + mean).astype(F)


def step(keys, x, logl, loglik_fn, mean, scale, max_subiter=1000):
    """One transition of every chain.  keys [C, 2]; x [C, D]; logl [C]; loglik_fn maps [C, D] to ([C], grad);
    mean [D]; scale = prior_scale(cov).  Returns ((x, logl), info) with info momentum, theta, subiter, exhausted,
    margin (the smallest |logL(p) - logy| over the chain's loop decisions) and nu."""
    x, logl = np.asarray(x, F), np.asarray(logl, F)
    C, D = x.shape
    mean = np.broadcast_to(np.asarray(mean, F), (D,)).astype(F)
    ks = prng.split(keys, 4)
    key_slice = ks[:, 0]
    nu = momentum(keys, mean, scale, D)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        logy = (logl + np.log(prng.uniform(ks[:, 2]))).astype(F)
    theta = (TWO_PI * prng.uniform(ks[:, 3])).astype(F)
    theta_min, theta_max = (theta - TWO_PI).astype(F), theta.copy()
    p = ellipse(x, nu, mean, theta)
    lp = np.asarray(loglik_fn(p)[0], F)
    subiter = np.ones(C, np.int32)
    margin = np.full(C, np.inf)

    def note(active):
        with np.errstate(invalid="ignore", over="ignore"):
            m = np.abs(lp.astype(np.float64) - logy.astype(np.float64))
        m = np.where(np.isnan(m), np.inf, m)
        margin[active] = np.minimum(margin[active], m[active])

    with np.errstate(invalid="ignore"):
        active = lp <= logy
    note(np.ones(C, bool))
    active &= subiter < max_subiter
    while active.any():
        f = prng.uniform(prng.fold_in(key_slice, subiter.astype(np.uint32)))
        t_new = np.maximum(theta_min, (f * (theta_max - theta_min).astype(F)).astype(F) + theta_min).astype(F)
        theta = np.where(active, t_new, theta)
        p_new = ellipse(x, nu, mean, theta)
        p = np.where(active[:, None], p_new, p)
        lp_new = np.asarray(loglik_fn(p_new)[0], F)
        lp = np.where(active, lp_new, lp)
        theta_min = np.where(active & (theta < 0), theta, theta_min)
        theta_max = np.where(active & (theta > 0), theta, theta_max)
        subiter = np.where(active, subiter + 1, subiter).astype(np.int32)
        note(active)
        with np.errstate(invalid="ignore"):
            active = active & (lp <= logy) & (subiter < max_subiter)
    with np.errstate(invalid="ignore"):
        exhausted = lp <= logy
    c = np.cos(theta).astype(F)[:, None]
    s = np.sin(theta).astype(F)[:, None]
    m = ((((nu - mean).astype(F) * c).astype(F) - ((x - mean).astype(F) * s).astype(F)).astype(F) + mean).astype(F)
    m = np.where(exhausted[:, None], nu, m)
    x_new = np.where(exhausted[:, None], x, p)
    l_new = np.where(exhausted, logl, lp).astype(F)
    info = dict(momentum=m, theta=np.where(exhausted, F(0), theta).astype(F), subiter=subiter, exhausted=exhausted,
                margin=margin, nu=nu)
    return (x_new, l_new), info
