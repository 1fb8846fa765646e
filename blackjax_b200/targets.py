"""Log-density targets with a fused device ``value_and_grad``.

BlackJAX accepts any JAX callable as ``logdensity_fn`` and differentiates it with
``jax.value_and_grad`` (blackjax/mcmc/hmc.py:91, integrators.py:189).  Without a tracing compiler the
H100 path takes a *target descriptor* in the ``logdensity_fn`` slot instead: one of the named models
below, each with a hand-derived gradient fused into the leapfrog kernels
(blackjax_b200/csrc/bjx_row.cuh ``Ctx::value_and_grad``), or a ``UserTarget``: the user's own fused
``value_and_grad`` as CUDA source, compiled into a plug-in that holds every kernel of the path
(include/bjx_user_target.h, blackjax_b200/plugin.py).
"""
import numpy as np
import torch

from . import _lib


class Target:
    kind = None
    dim = None

    def _desc(self, device):
        raise NotImplementedError

    def desc(self, device):
        """bjx_target_desc for ``device`` (parameter tensors are cached per device)."""
        return self._desc(torch.device(device))

    def _cached(self, name, host_array, device):
        cache = self.__dict__.setdefault("_dev", {})
        k = (name, str(device))
        if k not in cache:
            cache[k] = torch.as_tensor(np.ascontiguousarray(host_array, dtype=np.float32)).to(device)
        return cache[k]


class DiagGaussian(Target):
    """``std_normal_logdensity(x, scale)`` (tests/fixtures.py:60-78): -1/2 sum ((x-mean)/scale)^2 + offset."""

    kind = _lib.TARGET_DIAG_GAUSSIAN

    def __init__(self, scale=1.0, dim=None, mean=None, logp_offset=0.0):
        s = np.asarray(scale, np.float64)
        if s.ndim == 0:
            if dim is None:
                raise ValueError("dim is required with a scalar scale")
            s = np.full((dim,), float(s))
        self.scale = s
        self.dim = int(s.shape[0])
        self.inv_var = (1.0 / (s * s)).astype(np.float32)
        self.mean = None if mean is None else np.broadcast_to(np.asarray(mean, np.float32), (self.dim,)).copy()
        self.logp_offset = float(logp_offset)

    def _desc(self, device):
        d = _lib.TargetDesc()
        d.kind, d.dim = self.kind, self.dim
        d.inv_var = self._cached("inv_var", self.inv_var, device).data_ptr()
        d.mean = None if self.mean is None else self._cached("mean", self.mean, device).data_ptr()
        d.precision = None
        d.logp_offset = self.logp_offset
        return d


def StdNormal(dim):
    return DiagGaussian(1.0, dim)


class Funnel(Target):
    """``neal_funnel_logdensity`` (tests/fixtures.py:81-98)."""

    kind = _lib.TARGET_FUNNEL

    def __init__(self, dim):
        if dim < 2:
            raise ValueError("funnel needs dim >= 2")
        self.dim = int(dim)

    def _desc(self, device):
        d = _lib.TargetDesc()
        d.kind, d.dim = self.kind, self.dim
        d.logp_offset = 0.0
        return d


class DenseGaussian(Target):
    """-1/2 x^T P x + offset (tests/mcmc/test_mclmc_lrd.py:86-88)."""

    kind = _lib.TARGET_DENSE_GAUSSIAN

    def __init__(self, precision, logp_offset=0.0):
        p = np.asarray(precision, np.float32)
        if p.ndim != 2 or p.shape[0] != p.shape[1]:
            raise ValueError("precision must be a square matrix")
        # the kernels evaluate grad = -P x, which is the gradient of -1/2 x^T P x (what autodiff of the reference's
        # logdensity gives: -1/2 (P + P^T) x) only for a symmetric P
        asym = float(np.max(np.abs(p - p.T))) if p.size else 0.0
        if asym > 1e-6 * max(float(np.max(np.abs(p))), 1e-30):
            raise ValueError("precision must be symmetric (the fused value_and_grad computes -P x); "
                             "pass 0.5 * (P + P.T) for a general quadratic form")
        self.precision = p
        self.dim = int(p.shape[0])
        self.logp_offset = float(logp_offset)

    def _desc(self, device):
        d = _lib.TargetDesc()
        d.kind, d.dim = self.kind, self.dim
        d.precision = self._cached("precision", self.precision, device).data_ptr()
        d.logp_offset = self.logp_offset
        return d


class Banana(Target):
    """-(1-x0)^2 - 1.5 (x1 - x0^2)^2 (tests/mcmc/test_trajectory.py:79-80)."""

    kind = _lib.TARGET_BANANA
    dim = 2

    def _desc(self, device):
        d = _lib.TargetDesc()
        d.kind, d.dim = self.kind, 2
        d.logp_offset = 0.0
        return d


class HierLogit(Target):
    """Hierarchical logistic regression (BASELINE config 5; builder-defined, not in the reference).

    x = [mu, log_tau, beta0, beta1, alpha_0 .. alpha_{G-1}];  G groups, 8 Bernoulli-logit observations per group
    with two covariates:  eta_gk = alpha_g + beta . x_gk,  alpha_g ~ N(mu, tau^2),  mu ~ N(0, 10^2),
    log_tau ~ N(0, 1) (density on log_tau itself),  beta_j ~ N(0, 2.5^2).

      logp = -mu^2/200 - lt^2/2 - (b0^2+b1^2)/12.5 + sum_g [-(alpha_g-mu)^2 e^{-2 lt}/2 - lt]
             + sum_gk [y_gk eta_gk - softplus(eta_gk)]
    """

    kind = _lib.TARGET_HIER_LOGIT

    def __init__(self, covariates, outcomes_bits):
        x = np.ascontiguousarray(covariates, np.float32)
        y = np.ascontiguousarray(outcomes_bits, np.uint8)
        if x.ndim != 3 or x.shape[1:] != (8, 2) or y.shape != (x.shape[0],):
            raise ValueError("covariates must be [G, 8, 2] and outcomes_bits uint8 [G]")
        self.x, self.y = x, y
        self.n_groups = int(x.shape[0])
        self.dim = 4 + self.n_groups

    @staticmethod
    def synthetic_data(n_groups, seed=1):
        """Covariates ~ N(0,1) and outcomes drawn from the model at mu=0.5, tau=0.7, beta=(1,-0.5); default_rng(seed)."""
        rng = np.random.default_rng(seed)
        x = rng.standard_normal((n_groups, 8, 2)).astype(np.float32)
        alpha = 0.5 + 0.7 * rng.standard_normal(n_groups)
        eta = alpha[:, None] + x[:, :, 0] * 1.0 + x[:, :, 1] * (-0.5)
        y = rng.uniform(size=(n_groups, 8)) < 1.0 / (1.0 + np.exp(-eta))
        bits = (y.astype(np.uint8) << np.arange(8, dtype=np.uint8)).sum(axis=1).astype(np.uint8)
        return x, bits

    def _desc(self, device):
        d = _lib.TargetDesc()
        d.kind, d.dim = self.kind, self.dim
        d.data_x = self._cached("x", self.x, device).data_ptr()
        cache = self.__dict__.setdefault("_dev", {})
        k = ("y", str(device))
        if k not in cache:
            cache[k] = torch.as_tensor(self.y).to(device)
        d.data_y = cache[k].data_ptr()
        d.n_groups = self.n_groups
        d.logp_offset = 0.0
        return d


class UserTarget(Target):
    """A model of the user's own: ``source`` is CUDA text defining the device struct ``bjx_user::Model`` (contract:
    include/bjx_user_target.h); ``params`` is the float32 parameter block the function reads as ``u.theta`` (data,
    hyper-parameters).  This is the slot of BlackJAX's arbitrary ``logdensity_fn`` (mcmc/hmc.py:91): the gradient comes
    from the author instead of from autodiff, everything downstream (HMC / multinomial / generalized HMC, NUTS, window
    adaptation, ChEES, MEADS, every metric and integrator of the warp kernels) is the same code as for the built-in
    targets.  The plug-in is compiled by nvcc on first use and cached in-tree (blackjax_b200/_plugins/)."""

    kind = _lib.TARGET_USER

    def __init__(self, dim, source, params=None, name="user", logp_offset=0.0, dense_metric=True,
                 general_integrators=True):
        from . import plugin
        self.dim = int(dim)
        plugin.size_class(self.dim)  # validates the row size
        self.source = source
        self.name = name
        self.params = None if params is None else np.ascontiguousarray(params, np.float32).reshape(-1)
        self.logp_offset = float(logp_offset)
        self.build_options = dict(dense_metric=bool(dense_metric), general_integrators=bool(general_integrators))
        self._plugin_path = None

    def plugin_path(self):
        """Build the plug-in if it is not cached yet and return its path."""
        from . import plugin
        if self._plugin_path is None:
            self._plugin_path = plugin.build_plugin(self.source, self.dim, self.name, **self.build_options)
        return self._plugin_path

    def _desc(self, device):
        from . import plugin
        d = _lib.TargetDesc()
        d.kind, d.dim = self.kind, self.dim
        d.logp_offset = self.logp_offset
        d.user_plugin = plugin.load_plugin(self.plugin_path())
        if self.params is not None and self.params.size:
            d.user_params = self._cached("params", self.params, device).data_ptr()
            d.n_user_params = int(self.params.size)
        return d


class LinearRegression(UserTarget):
    """The regression posterior of the reference's sampling tests (tests/mcmc/test_sampling.py:103-111
    ``regression_logprob``; position = [log_scale, coefs_0 .. coefs_{K-1}]) as a user-defined target:
    blackjax_b200/user_targets/linear_regression.cuh.  ``x`` is [N, K] (K <= 16), ``y`` is [N]."""

    def __init__(self, x, y, **build_options):
        from . import plugin
        x = np.ascontiguousarray(x, np.float32)
        y = np.ascontiguousarray(y, np.float32).reshape(-1)
        if x.ndim == 1:
            x = x[:, None]
        if x.ndim != 2 or x.shape[0] != y.shape[0] or not (1 <= x.shape[1] <= 16):
            raise ValueError("x must be [N, K] with 1 <= K <= 16 and y [N]")
        if x.shape[0] >= 1 << 24:
            raise ValueError("N must be below 2^24 (it travels as a float)")
        self.x, self.y = x, y
        theta = np.concatenate([np.asarray([x.shape[0], x.shape[1]], np.float32), x.reshape(-1), y])
        super().__init__(1 + x.shape[1], plugin.read_example("linear_regression"), theta, name="linear_regression",
                         **build_options)


class Rosenbrock(UserTarget):
    """-beta * sum_{i<D-1} [a (x_{i+1} - x_i^2)^2 + (1 - x_i)^2]: a neighbour-coupled model shipped as a user-defined target
    (blackjax_b200/user_targets/rosenbrock.cuh; the row is staged in the warp's shared-memory scratch)."""

    def __init__(self, dim, a=5.0, beta=0.05, **build_options):
        from . import plugin
        if dim < 2:
            raise ValueError("Rosenbrock needs dim >= 2")
        super().__init__(dim, plugin.read_example("rosenbrock"), np.asarray([a, beta], np.float32), name="rosenbrock",
                         **build_options)
