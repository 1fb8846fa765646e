"""Analytic ``value_and_grad`` of the named targets (float32, batched over chains).

TEST INFRASTRUCTURE (see oracle/__init__.py).  The reference differentiates arbitrary
JAX callables with ``jax.value_and_grad`` (blackjax/mcmc/hmc.py:91,
integrators.py:189,204); without JAX the named models are differentiated by hand:

* ``StdNormal`` / ``DiagGaussian``  tests/fixtures.py:60-78 ``std_normal_logdensity``
* ``Funnel``                        tests/fixtures.py:81-98 ``neal_funnel_logdensity``
* ``DenseGaussian``                 tests/mcmc/test_mclmc_lrd.py:68-90,
                                    tests/adaptation/test_staged_adaptation.py:1029-1040
* ``Banana``                        tests/mcmc/test_trajectory.py:79-80
* ``NormLogpdf``                    tests/mcmc/test_trajectory.py:27 (jax.scipy.stats.norm.logpdf)
* ``LinearRegression``              tests/mcmc/test_sampling.py:103-111 ``regression_logprob``
* ``Rosenbrock``                    builder-defined neighbour-coupled model (blackjax_b200/user_targets/rosenbrock.cuh)
* ``BoundedGaussian``               tests/mcmc/test_mclmc_nan_fix_969.py:45-47 (the bounded target of issue #969)

Each target maps ``q: f32[C, D]`` to ``(logp: f32[C], grad: f32[C, D])``.
"""
import numpy as np

F = np.float32


class DiagGaussian:
    """logp = -1/2 sum (x_i/s_i)^2 ; grad_i = -x_i / s_i^2   (scale scalar or [D])."""

    kind = "diag_gaussian"

    def __init__(self, scale=1.0, dim=None, mean=None, logp_offset=0.0):
        s = np.asarray(scale, np.float64)
        if s.ndim == 0:
            assert dim is not None
            s = np.full((dim,), float(s))
        self.scale = s.astype(F)
        # same constant the device path receives: 1/s^2 rounded once to f32
        self.inv_var = (1.0 / (s * s)).astype(F)
        self.dim = self.scale.shape[0]
        self.mean = None if mean is None else np.broadcast_to(np.asarray(mean, F), (self.dim,)).copy()
        self.logp_offset = F(logp_offset)

    def __call__(self, q):
        q = np.asarray(q, F)
        d = q if self.mean is None else (q - self.mean).astype(F)
        t = d * self.inv_var
        logp = F(-0.5) * np.sum(d * t, axis=-1, dtype=F) + self.logp_offset
        return logp.astype(F), (-t).astype(F)


def StdNormal(dim):
    return DiagGaussian(1.0, dim)


class Funnel:
    """Neal's funnel: y=x[0]~N(0,3^2), x[1:]~N(0,e^y).

    logp = -1/2 (y/3)^2 - 1/2 e^{-y} sum v^2 - 1/2 n y
    d/dy = -y/9 + 1/2 e^{-y} sum v^2 - n/2 ;  d/dv_i = -e^{-y} v_i
    """

    kind = "funnel"

    def __init__(self, dim):
        self.dim = dim

    def __call__(self, q):
        q = np.asarray(q, F)
        y = q[..., 0]
        v = q[..., 1:]
        n = F(self.dim - 1)
        with np.errstate(over="ignore", invalid="ignore"):
            ey = np.exp(-y).astype(F)
            ss = np.sum(v * v, axis=-1, dtype=F)
            t = y / F(3.0)
            logp = F(-0.5) * (t * t) + (F(-0.5) * ey * ss - F(0.5) * n * y)
            g = np.empty_like(q)
            g[..., 0] = -y / F(9.0) + F(0.5) * ey * ss - F(0.5) * n
            g[..., 1:] = -(ey[..., None] * v)
        return logp.astype(F), g.astype(F)


class DenseGaussian:
    """logp = -1/2 x^T P x ; grad = -P x   (P symmetric precision, [D, D])."""

    kind = "dense_gaussian"

    def __init__(self, precision, const=0.0):
        self.precision = np.asarray(precision, F)
        self.dim = self.precision.shape[0]
        self.const = F(const)

    def __call__(self, q):
        q = np.asarray(q, F)
        Pq = (q @ self.precision.T).astype(F)
        logp = F(-0.5) * np.sum(q * Pq, axis=-1, dtype=F) + self.const
        return logp.astype(F), (-Pq).astype(F)


class Banana:
    """logp = -(1-x0)^2 - 1.5 (x1 - x0^2)^2   (tests/mcmc/test_trajectory.py:79-80)."""

    kind = "banana"
    dim = 2

    def __call__(self, q):
        q = np.asarray(q, F)
        x0, x1 = q[..., 0], q[..., 1]
        r = x1 - x0 * x0
        logp = -((F(1.0) - x0) ** 2) - F(1.5) * r * r
        g = np.stack([F(2.0) * (F(1.0) - x0) + F(6.0) * r * x0, F(-3.0) * r], axis=-1)
        return logp.astype(F), g.astype(F)


class NormLogpdf:
    """sum_i norm.logpdf(x_i) = -1/2 x^2 - 1/2 log(2 pi) (normalised standard normal)."""

    kind = "norm_logpdf"

    def __init__(self, dim=1):
        self.dim = dim

    def __call__(self, q):
        q = np.asarray(q, F)
        logp = np.sum(F(-0.5) * q * q - F(0.5 * np.log(2 * np.pi)), axis=-1, dtype=F)
        return logp.astype(F), (-q).astype(F)


def correlated_gaussian(dim, seed=0, lo=-1.0, hi=1.0):
    """BASELINE config 2 target: Sigma = Q diag(logspace(lo,hi,dim)) Q^T, Q from QR of a
    default_rng(seed) normal matrix (recipe of tests/mcmc/test_mclmc_lrd.py:68-90).
    Returns (cov f32, precision f32), both symmetrised in float64 before the cast."""
    rng = np.random.default_rng(seed)
    Q, _ = np.linalg.qr(rng.standard_normal((dim, dim)))
    eigs = np.logspace(lo, hi, dim)
    cov = (Q * eigs) @ Q.T
    prec = (Q / eigs) @ Q.T
    cov = 0.5 * (cov + cov.T)
    prec = 0.5 * (prec + prec.T)
    return cov.astype(F), prec.astype(F)


class HierLogit:
    """Hierarchical logistic regression, BASELINE config 5 (builder-defined; see blackjax_b200/targets.py HierLogit).
    x = [mu, log_tau, beta0, beta1, alpha_0..alpha_{G-1}]; covariates [G,8,2]; outcomes: bit k of byte g."""

    kind = "hier_logit"

    def __init__(self, covariates, outcomes_bits):
        self.x = np.asarray(covariates, F)
        bits = np.asarray(outcomes_bits, np.uint8)
        self.y = ((bits[:, None] >> np.arange(8, dtype=np.uint8)) & 1).astype(F)      # [G, 8]
        self.G = self.x.shape[0]
        self.dim = 4 + self.G

    def __call__(self, q):
        q = np.asarray(q, F)
        mu, lt, b0, b1 = q[..., 0], q[..., 1], q[..., 2], q[..., 3]
        alpha = q[..., 4:]                                                             # [C, G]
        with np.errstate(over="ignore", invalid="ignore"):
            e2 = np.exp(F(-2.0) * lt).astype(F)
            d = (alpha - mu[..., None]).astype(F)
            eta = (alpha[..., None] + b0[..., None, None] * self.x[:, :, 0] + b1[..., None, None] * self.x[:, :, 1]).astype(F)
            sig = (F(1.0) / (F(1.0) + np.exp(-eta))).astype(F)
            softplus = (np.maximum(eta, F(0.0)) + np.log1p(np.exp(-np.abs(eta)))).astype(F)
            r = (self.y - sig).astype(F)
            ll = np.sum(self.y * eta - softplus, axis=(-1, -2), dtype=F)
            sd = np.sum(d, axis=-1, dtype=F)
            sd2 = np.sum(d * d, axis=-1, dtype=F)
            logp = (F(-0.005) * mu * mu - F(0.5) * lt * lt - F(0.08) * (b0 * b0 + b1 * b1)
                    + (F(-0.5) * e2 * sd2 - F(self.G) * lt) + ll)
            g = np.empty_like(q)
            g[..., 0] = F(-0.01) * mu + e2 * sd
            g[..., 1] = -lt + e2 * sd2 - F(self.G)
            g[..., 2] = F(-0.16) * b0 + np.sum(r * self.x[:, :, 0], axis=(-1, -2), dtype=F)
            g[..., 3] = F(-0.16) * b1 + np.sum(r * self.x[:, :, 1], axis=(-1, -2), dtype=F)
            g[..., 4:] = -d * e2[..., None] + np.sum(r, axis=-1, dtype=F)
        return logp.astype(F), g.astype(F)


class LinearRegression:
    """``regression_logprob`` of the reference's sampling tests (tests/mcmc/test_sampling.py:103-111), K coefficients:

        scale = exp(log_scale)
        logp  = expon.logpdf(scale, 0, 1) + log_scale + sum_k norm.logpdf(coefs_k, 0, 5)
              + sum_n norm.logpdf(y_n, X_n . coefs, scale)

    position = [log_scale, coefs_0 .. coefs_{K-1}].  The gradient is what ``jax.grad`` of that expression gives,
    written out:  d/d log_scale = -scale + 1 - N + sum_n r_n^2 / scale^2,  d/d coefs_k = -coefs_k/25 + sum_n r_n X_nk / scale^2
    (r_n = y_n - X_n . coefs).  Checked against central differences of the float64 density in tests/test_oracle_kat.py."""

    kind = "linear_regression"

    def __init__(self, x, y):
        x = np.asarray(x, F)
        self.x = x[:, None] if x.ndim == 1 else x
        self.y = np.asarray(y, F).reshape(-1)
        self.N, self.K = self.x.shape
        self.dim = 1 + self.K

    def logp64(self, q):
        """The reference's expression in float64 (jax.scipy.stats formulas), for gradient checks."""
        q = np.asarray(q, np.float64)
        ls, c = q[..., 0], q[..., 1:]
        scale = np.exp(ls)
        r = self.y.astype(np.float64) - c @ self.x.astype(np.float64).T
        prior = -scale + ls + np.sum(-c * c / 50.0 - np.log(5.0) - 0.5 * np.log(2 * np.pi), axis=-1)
        lik = np.sum(-r * r / (2.0 * scale[..., None] ** 2) - ls[..., None] - 0.5 * np.log(2 * np.pi), axis=-1)
        return prior + lik

    def __call__(self, q):
        q = np.asarray(q, F)
        ls, c = q[..., 0], q[..., 1:]
        with np.errstate(over="ignore", invalid="ignore"):
            scale = np.exp(ls).astype(F)
            w = np.exp(F(-2.0) * ls).astype(F)
            r = (self.y - (c @ self.x.T).astype(F)).astype(F)                    # [C, N]
            ss = np.sum(r * r, axis=-1, dtype=F)
            rx = (r @ self.x).astype(F)                                          # [C, K]
            cc = np.sum(c * c, axis=-1, dtype=F)
            k0 = F(np.log(5.0)) + F(0.5 * np.log(2 * np.pi))
            logp = (ls - scale) - (cc / F(50.0) + F(self.K) * k0) - (F(0.5) * w * ss + F(self.N) * (ls + F(0.5 * np.log(2 * np.pi))))
            g = np.empty_like(q)
            g[..., 0] = (w * ss - scale) + (F(1.0) - F(self.N))
            g[..., 1:] = w[..., None] * rx - c / F(25.0)
        return logp.astype(F), g.astype(F)


class Rosenbrock:
    """logp(x) = -beta * sum_{i<D-1} [a (x_{i+1} - x_i^2)^2 + (1 - x_i)^2]; the neighbour-coupled user-defined target of
    blackjax_b200/user_targets/rosenbrock.cuh (builder-defined: not in the reference)."""

    kind = "rosenbrock"

    def __init__(self, dim, a=5.0, beta=0.05):
        self.dim, self.a, self.beta = dim, F(a), F(beta)

    def logp64(self, q):
        q = np.asarray(q, np.float64)
        t = q[..., 1:] - q[..., :-1] ** 2
        return -float(self.beta) * np.sum(float(self.a) * t * t + (1.0 - q[..., :-1]) ** 2, axis=-1)

    def __call__(self, q):
        q = np.asarray(q, F)
        a, beta = self.a, self.beta
        with np.errstate(over="ignore", invalid="ignore"):
            xi = q[..., :-1]
            t = (q[..., 1:] - xi * xi).astype(F)
            o = (F(1.0) - xi).astype(F)
            logp = -beta * np.sum(a * t * t + o * o, axis=-1, dtype=F)
            d = np.zeros_like(q)
            d[..., :-1] = F(-4.0) * a * xi * t - F(2.0) * o
            d[..., 1:] += F(2.0) * a * t
        return logp.astype(F), (-beta * d).astype(F)


class BoundedGaussian:
    """The bounded target of tests/mcmc/test_mclmc_nan_fix_969.py:45-47: -1/2 sum x^2 + sum log(B - |x|)."""

    def __init__(self, dim, bound=5.0):
        self.dim, self.bound = dim, F(bound)

    def __call__(self, q):
        q = np.asarray(q, F)
        with np.errstate(invalid="ignore", divide="ignore"):
            r = (self.bound - np.abs(q)).astype(F)
            logp = (F(-0.5) * np.sum(q * q, axis=-1, dtype=F) + np.sum(np.log(r), axis=-1, dtype=F)).astype(F)
            g = (-q - np.where(q >= 0, F(1), F(-1)) / r).astype(F)
        return logp, g
