"""Engine: one libbjx handle per (device, stream, n_chains, dim, target, depth).  Thin, typed calls
into the C ABI; all arrays are torch CUDA tensors used purely as device memory."""
import ctypes as C

import numpy as np
import torch

from . import _lib
from ._lib import check, lib, ptr

import collections

# Engines own device workspaces (NUTS: (9 + 2*depth) rows of [C,D]; dense path: 4 rows + operand planes), so the cache is a
# small LRU: the least recently used engine leaves the cache when a new shape/target comes in and is destroyed (handle
# and workspaces freed) as soon as nobody else holds it.
_ENGINES = collections.OrderedDict()
_MAX_ENGINES = 8


def _f32(t, shape=None, name="array"):
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise TypeError(f"{name} must be a CUDA tensor (blackjax_b200 has no CPU path)")
    if t.dtype != torch.float32:
        raise TypeError(f"{name} must be float32, got {t.dtype}")
    if not t.is_contiguous():
        raise ValueError(f"{name} must be contiguous")
    if shape is not None and tuple(t.shape) != tuple(shape):
        raise ValueError(f"{name} has shape {tuple(t.shape)}, expected {tuple(shape)}")
    return t


def as_keys(keys, n, device):
    """uint32 [n,2] per-chain keys, or ONE key uint32 [2] (per-chain keys are then derived in-kernel), on ``device``."""
    if not isinstance(keys, torch.Tensor):
        raise TypeError("rng_key must be a torch tensor of raw uint32 key data")
    if keys.dtype not in (torch.uint32, torch.int32):
        raise TypeError(f"rng_key must be uint32 (or int32 bit patterns), got {keys.dtype}")
    keys = keys.to(device).contiguous()
    if tuple(keys.shape) not in ((n, 2), (2,)):
        raise ValueError(f"rng_key has shape {tuple(keys.shape)}, expected ({n}, 2) or (2,)")
    return keys


class Engine:
    def __init__(self, device, n_chains, dim, target, max_tree_depth=10, divergence_threshold=1000.0, stream=None):
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise _lib.BjxError("blackjax_b200 runs on CUDA devices only (no CPU fallback)")
        self.index = self.device.index if self.device.index is not None else torch.cuda.current_device()
        self.device = torch.device("cuda", self.index)
        self.C, self.D = int(n_chains), int(dim)
        self.target = target
        self.max_tree_depth = int(max_tree_depth)
        self.stream = torch.cuda.current_stream(self.device) if stream is None else stream
        cfg = _lib.Config()
        cfg.device = self.index
        cfg.n_chains, cfg.dim = self.C, self.D
        cfg.max_tree_depth = self.max_tree_depth
        cfg.divergence_threshold = float(divergence_threshold)
        cfg.stream = self.stream.cuda_stream
        cfg.target = target.desc(self.device)
        h = C.c_void_p()
        check(lib().bjx_create(C.byref(cfg), C.byref(h)))
        self.h = h
        self._imm = None      # keeps the caller's inverse mass matrix alive
        self._imm_key = None

    def close(self):
        """Destroy the libbjx handle (synchronises its stream and frees its workspaces)."""
        if getattr(self, "h", None):
            lib().bjx_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- metric ---------------------------------------------------------------------------------
    def set_metric(self, inverse_mass_matrix, diagonal_only=False):
        """1-D => diagonal, 2-D [D,D] => dense, 2-D [C,D] => per-chain diagonal, 3-D [C,D,D] => per-chain dense
        (blackjax/mcmc/metrics.py:701-729 semantics incl. the ValueError; the per-chain layouts are what jax.vmap
        over chains gives the reference).  ``diagonal_only`` (MCLMC, whose metric is always diagonal): a 2-D array is
        per-chain diagonal [C,D] whatever C and D are."""
        imm = inverse_mass_matrix
        from .mcmc.metrics import LowRankMetric
        if isinstance(imm, LowRankMetric):  # metrics.gaussian_euclidean_low_rank (metrics.py:349-467)
            sg, U, lam = (t.to(self.device, torch.float32).contiguous() for t in imm)
            if sg.shape[0] != self.D:
                raise ValueError(f"low-rank metric has {sg.shape[0]} dimensions, expected {self.D}")
            check(lib().bjx_set_metric_low_rank(self.h, ptr(sg), ptr(U), ptr(lam), int(lam.shape[0])), self.h)
            self._imm = (sg, U, lam)
            return imm
        if not isinstance(imm, torch.Tensor):
            imm = torch.as_tensor(imm, dtype=torch.float32)
        imm = imm.to(self.device, torch.float32).contiguous()
        if imm.ndim == 1:
            if imm.shape[0] != self.D:
                raise ValueError(f"inverse_mass_matrix has {imm.shape[0]} entries, expected {self.D}")
            kind = _lib.METRIC_DIAG
        elif diagonal_only and imm.ndim == 2:
            if tuple(imm.shape) != (self.C, self.D):
                raise ValueError(f"per-chain diagonal inverse_mass_matrix has shape {tuple(imm.shape)}, "
                                 f"expected ({self.C}, {self.D})")
            kind = _lib.METRIC_DIAG_PER_CHAIN
        elif imm.ndim == 2 and tuple(imm.shape) == (self.D, self.D):
            kind = _lib.METRIC_DENSE
        elif imm.ndim == 2 and tuple(imm.shape) == (self.C, self.D):
            kind = _lib.METRIC_DIAG_PER_CHAIN
        elif imm.ndim == 3 and tuple(imm.shape) == (self.C, self.D, self.D):
            kind = _lib.METRIC_DENSE_PER_CHAIN   # one dense matrix per chain (vmapped dense adaptation), dim <= 64
        else:
            raise ValueError(
                "The mass matrix has the wrong number of dimensions:"
                f" expected 1 or 2, got {imm.ndim}.")
        self._imm = imm
        check(lib().bjx_set_metric(self.h, kind, ptr(imm)), self.h)
        return imm

    def ensure_metric(self, inverse_mass_matrix, diagonal_only=False):
        """Install the metric unless this exact tensor CONTENT is already installed: the cache key is (storage pointer,
        shape, torch's in-place version counter), so an in-place update of the caller's tensor re-derives
        mass_matrix_sqrt and the dense operand planes instead of silently keeping stale ones."""
        imm = inverse_mass_matrix
        from .mcmc.metrics import LowRankMetric
        if isinstance(imm, LowRankMetric):
            key = tuple((t.data_ptr(), tuple(t.shape), t._version, str(t.device)) for t in imm)
        else:
            key = ((imm.data_ptr(), tuple(imm.shape), imm._version, str(imm.device), diagonal_only)
                   if isinstance(imm, torch.Tensor) else None)
        if key is None or key != self._imm_key:
            installed = self.set_metric(imm, diagonal_only)
            # a converted copy (dtype / device / layout) is owned by the engine: key on the caller's tensor all the same
            self._imm_key = key
            return installed
        return self._imm

    def _key_mode(self, keys, chain_offset=0):
        """Select per-chain keys [C,2] or a shared step key [2] (+ global chain offset) for the next transition."""
        mode = (1 if keys.ndim == 1 else 0, int(chain_offset))
        if getattr(self, "_keymode", None) != mode:
            check(lib().bjx_set_key_mode(self.h, mode[0], mode[1]), self.h)
            self._keymode = mode

    def set_integrator(self, coefficients):
        """integrators.py:62-152 coefficient table (tuple of floats); cached per engine."""
        coef = tuple(float(c) for c in coefficients)
        if getattr(self, "_coef", (0.5, 1.0, 0.5)) != coef:
            arr = (C.c_float * len(coef))(*coef)
            check(lib().bjx_set_integrator(self.h, arr, len(coef)), self.h)
            self._coef = coef

    def mass_matrix_sqrt(self):
        out = C.c_void_p()
        check(lib().bjx_get_mass_matrix_sqrt(self.h, C.byref(out)), self.h)
        return out.value

    # -- building blocks ----------------------------------------------------------------------------
    def init_state(self, q):
        q = _f32(q, (self.C, self.D), "position")
        logp = torch.empty(self.C, dtype=torch.float32, device=self.device)
        g = torch.empty_like(q)
        check(lib().bjx_init_state(self.h, ptr(q), ptr(logp), ptr(g)), self.h)
        return logp, g

    def sample_momentum(self, keys, chain_offset=0):
        keys = as_keys(keys, self.C, self.device)
        self._key_mode(keys, chain_offset)
        p = torch.empty(self.C, self.D, dtype=torch.float32, device=self.device)
        check(lib().bjx_sample_momentum(self.h, ptr(keys), ptr(p)), self.h)
        return p

    def leapfrog_(self, q, p, logp, g, step_size, n_steps):
        """n_steps velocity-Verlet steps IN PLACE on (q, p, logp, g)."""
        eps, eps_dev = self._eps(step_size)
        check(lib().bjx_leapfrog(self.h, ptr(_f32(q, (self.C, self.D))), ptr(_f32(p, (self.C, self.D))),
                                 ptr(_f32(logp, (self.C,))), ptr(_f32(g, (self.C, self.D))), eps, ptr(eps_dev),
                                 int(n_steps)), self.h)

    def velocity(self, p):
        """linear_map(M^-1, p) for every chain (dim > 128)."""
        v = torch.empty(self.C, self.D, dtype=torch.float32, device=self.device)
        check(lib().bjx_metric_velocity(self.h, ptr(_f32(p, (self.C, self.D))), ptr(v)), self.h)
        return v

    def energy(self, p, logp):
        e = torch.empty(self.C, dtype=torch.float32, device=self.device)
        check(lib().bjx_energy(self.h, ptr(_f32(p, (self.C, self.D))), ptr(_f32(logp, (self.C,))), ptr(e)), self.h)
        return e

    def is_turning(self, pl, pr, ps):
        out = torch.empty(self.C, dtype=torch.uint8, device=self.device)
        check(lib().bjx_is_turning(self.h, ptr(_f32(pl, (self.C, self.D))), ptr(_f32(pr, (self.C, self.D))),
                                   ptr(_f32(ps, (self.C, self.D))), ptr(out)), self.h)
        return out.bool()

    def _eps(self, step_size, name="step_size"):
        """A per-chain parameter (step size, MCLMC's L): scalar -> (value, None); [C] tensor -> (0, device array)."""
        if isinstance(step_size, torch.Tensor) and step_size.ndim >= 1:
            return 0.0, _f32(step_size.to(self.device), (self.C,), name)
        return float(step_size), None

    def _info(self, fields, struct=_lib.Info):
        info = struct()
        for k, v in fields.items():
            setattr(info, k, ptr(v))
        return info

    # -- transitions -----------------------------------------------------------------------------------
    def hmc_step(self, keys, q, logp, g, step_size, num_integration_steps, out=None, info_fields=None,
                 multinomial=False, chain_offset=0):
        keys = as_keys(keys, self.C, self.device)
        self._key_mode(keys, chain_offset)
        q = _f32(q, (self.C, self.D), "position")
        g = _f32(g, (self.C, self.D), "logdensity_grad")
        logp = _f32(logp, (self.C,), "logdensity")
        qo, lo, go = out if out is not None else (torch.empty_like(q), torch.empty_like(logp), torch.empty_like(g))
        eps, eps_dev = self._eps(step_size)
        info = self._info(info_fields or {})
        fn = lib().bjx_mhmc_step if multinomial else lib().bjx_hmc_step
        steps_dev = None
        if isinstance(num_integration_steps, torch.Tensor):  # dynamic HMC: one trajectory length per chain
            steps_dev = num_integration_steps.to(device=self.device, dtype=torch.int32).contiguous()
            if steps_dev.shape != (self.C,):
                raise ValueError(f"per-chain num_integration_steps must have shape ({self.C},)")
            num_integration_steps = 1
        check(lib().bjx_set_integration_steps(self.h, ptr(steps_dev)), self.h)
        try:
            check(fn(self.h, ptr(keys), ptr(q), ptr(logp), ptr(g), ptr(qo), ptr(lo), ptr(go), eps,
                     ptr(eps_dev), int(num_integration_steps), C.byref(info)), self.h)
        finally:
            if steps_dev is not None:
                check(lib().bjx_set_integration_steps(self.h, None), self.h)
                self._steps_keepalive = steps_dev  # the launch is asynchronous: keep the array until the next call
        return qo, lo, go

    def nuts_step(self, keys, q, logp, g, step_size, max_num_doublings, out=None, info_fields=None,
                  momentum=None, key_integrator=None, chain_offset=0):
        if max_num_doublings > self.max_tree_depth:
            raise ValueError("max_num_doublings exceeds the engine's max_tree_depth")
        q = _f32(q, (self.C, self.D), "position")
        g = _f32(g, (self.C, self.D), "logdensity_grad")
        logp = _f32(logp, (self.C,), "logdensity")
        if key_integrator is not None:
            key_integrator = as_keys(key_integrator, self.C, self.device)
            momentum = _f32(momentum, (self.C, self.D), "momentum")
            keys = None
        else:
            keys = as_keys(keys, self.C, self.device)
            self._key_mode(keys, chain_offset)
        qo, lo, go = out if out is not None else (torch.empty_like(q), torch.empty_like(logp), torch.empty_like(g))
        eps, eps_dev = self._eps(step_size)
        info = self._info(info_fields or {})
        check(lib().bjx_nuts_step(self.h, ptr(keys), ptr(q), ptr(logp), ptr(g), ptr(qo), ptr(lo), ptr(go), eps,
                                  ptr(eps_dev), int(max_num_doublings), C.byref(info), ptr(momentum),
                                  ptr(key_integrator)), self.h)
        if key_integrator is not None:
            self._keymode = None  # per-call override: re-establish the key mode on the next ordinary call
        return qo, lo, go

    def mclmc_init(self, keys, q, chain_offset=0):
        """mclmc.init: (logp, grad, unit momentum)."""
        keys = as_keys(keys, self.C, self.device)
        self._key_mode(keys, chain_offset)
        q = _f32(q, (self.C, self.D), "position")
        logp = torch.empty(self.C, dtype=torch.float32, device=self.device)
        g, p = torch.empty_like(q), torch.empty_like(q)
        check(lib().bjx_mclmc_init(self.h, ptr(keys), ptr(q), ptr(logp), ptr(g), ptr(p)), self.h)
        return logp, g, p

    def mclmc_step_(self, keys, q, p, logp, g, step_size, L, energy_cutoff, info_fields=None, chain_offset=0):
        """One MCLMC transition IN PLACE on (q, p, logp, g)."""
        keys = as_keys(keys, self.C, self.device)
        self._key_mode(keys, chain_offset)
        eps, eps_dev = self._eps(step_size)
        L, L_dev = self._eps(L, "L")
        info = self._info(info_fields or {}, _lib.MclmcInfo)
        check(lib().bjx_mclmc_step(self.h, ptr(keys), ptr(_f32(q, (self.C, self.D), "position")),
                                   ptr(_f32(p, (self.C, self.D), "momentum")), ptr(_f32(logp, (self.C,), "logdensity")),
                                   ptr(_f32(g, (self.C, self.D), "logdensity_grad")), eps, ptr(eps_dev), L, ptr(L_dev),
                                   float(energy_cutoff), C.byref(info)), self.h)
        self._mclmc_keepalive = (eps_dev, L_dev)  # the launch is asynchronous

    def adjusted_mclmc_step(self, keys, q, logp, g, step_size, num_integration_steps, L_proposal_factor, out=None,
                            info_fields=None, chain_offset=0):
        """One adjusted MCLMC transition; ``num_integration_steps`` is an int or an int32 tensor [C] (one per chain)."""
        keys = as_keys(keys, self.C, self.device)
        self._key_mode(keys, chain_offset)
        q = _f32(q, (self.C, self.D), "position")
        g = _f32(g, (self.C, self.D), "logdensity_grad")
        logp = _f32(logp, (self.C,), "logdensity")
        qo, lo, go = out if out is not None else (torch.empty_like(q), torch.empty_like(logp), torch.empty_like(g))
        eps, eps_dev = self._eps(step_size)
        info = self._info(info_fields or {})
        steps_dev = avg_dev = None
        if isinstance(num_integration_steps, torch.Tensor) and num_integration_steps.is_floating_point():
            avg_dev = _f32(num_integration_steps.to(self.device, torch.float32).contiguous(), (self.C,),
                           "num_integration_steps")  # ceil per chain
            num_integration_steps = 0
        elif isinstance(num_integration_steps, torch.Tensor):  # adjusted_mclmc_dynamic: one step count per chain
            steps_dev = num_integration_steps.to(device=self.device, dtype=torch.int32).contiguous()
            if steps_dev.shape != (self.C,):
                raise ValueError(f"per-chain num_integration_steps must have shape ({self.C},)")
            num_integration_steps = 0
        check(lib().bjx_set_integration_steps(self.h, ptr(steps_dev)), self.h)
        check(lib().bjx_set_integration_steps_avg(self.h, ptr(avg_dev)), self.h)
        try:
            check(lib().bjx_adjusted_mclmc_step(self.h, ptr(keys), ptr(q), ptr(logp), ptr(g), ptr(qo), ptr(lo), ptr(go),
                                                eps, ptr(eps_dev), int(num_integration_steps), float(L_proposal_factor),
                                                C.byref(info)), self.h)
        finally:
            if steps_dev is not None:
                check(lib().bjx_set_integration_steps(self.h, None), self.h)
            if avg_dev is not None:
                check(lib().bjx_set_integration_steps_avg(self.h, None), self.h)
        self._amclmc_keepalive = (steps_dev, eps_dev, avg_dev)  # the launch is asynchronous: keep the arrays
        return qo, lo, go

    def gist_step(self, keys, q, logp, g, params, step_size, out=None, info_fields=None, chain_offset=0):
        """One GIST transition (libbjx ``bjx_gist_step``); ``params`` is a ``_lib.GistParams``."""
        keys = as_keys(keys, self.C, self.device)
        self._key_mode(keys, chain_offset)
        q = _f32(q, (self.C, self.D), "position")
        g = _f32(g, (self.C, self.D), "logdensity_grad")
        logp = _f32(logp, (self.C,), "logdensity")
        qo, lo, go = out if out is not None else (torch.empty_like(q), torch.empty_like(logp), torch.empty_like(g))
        eps, eps_dev = self._eps(step_size)
        info = self._info(info_fields or {}, _lib.GistInfo)
        check(lib().bjx_gist_step(self.h, C.byref(params), ptr(keys), ptr(q), ptr(logp), ptr(g), ptr(qo), ptr(lo),
                                  ptr(go), eps, ptr(eps_dev), C.byref(info)), self.h)
        return qo, lo, go

    def langevin_step(self, sampler, keys, q, logp, g, step_size, out=None, info_fields=None, chain_offset=0):
        """One MALA (``sampler="mala"``, libbjx ``bjx_mala_step``) or Barker (``"barker"``, ``bjx_barker_step``)
        transition; Barker uses the installed metric."""
        keys = as_keys(keys, self.C, self.device)
        self._key_mode(keys, chain_offset)
        q = _f32(q, (self.C, self.D), "position")
        g = _f32(g, (self.C, self.D), "logdensity_grad")
        logp = _f32(logp, (self.C,), "logdensity")
        qo, lo, go = out if out is not None else (torch.empty_like(q), torch.empty_like(logp), torch.empty_like(g))
        eps, eps_dev = self._eps(step_size)
        info = self._info(info_fields or {}, _lib.LangevinInfo)
        fn = lib().bjx_mala_step if sampler == "mala" else lib().bjx_barker_step
        check(fn(self.h, ptr(keys), ptr(q), ptr(logp), ptr(g), ptr(qo), ptr(lo), ptr(go), eps, ptr(eps_dev),
                 C.byref(info)), self.h)
        return qo, lo, go

    def mala_step(self, keys, q, logp, g, step_size, out=None, info_fields=None, chain_offset=0):
        return self.langevin_step("mala", keys, q, logp, g, step_size, out, info_fields, chain_offset)

    def barker_step(self, keys, q, logp, g, step_size, out=None, info_fields=None, chain_offset=0):
        return self.langevin_step("barker", keys, q, logp, g, step_size, out, info_fields, chain_offset)

    def ensure_elliptical_prior(self, mean, cov):
        """Install the elliptical slice prior N(mean, cov) (libbjx ``bjx_set_elliptical_prior``) unless this exact
        content is installed: tensors are keyed as in ``ensure_metric``, a Python scalar mean by its value.  mean:
        scalar or [D]; cov: [D] variances or [D, D]."""
        def content_key(t):
            if isinstance(t, torch.Tensor):
                return (t.data_ptr(), tuple(t.shape), t._version, str(t.device))
            return ("scalar", float(t)) if np.ndim(t) == 0 else None
        key = (content_key(mean), content_key(cov))
        given = (mean, cov)
        if None not in key and key == getattr(self, "_prior_key", None):
            return
        mean = torch.as_tensor(mean, dtype=torch.float32, device=self.device)
        cov = torch.as_tensor(cov, dtype=torch.float32, device=self.device)
        if cov.ndim == 1 and cov.shape[0] == self.D:
            kind = _lib.METRIC_DIAG
        elif cov.ndim == 2 and tuple(cov.shape) == (self.D, self.D):
            kind = _lib.METRIC_DENSE
        else:
            raise ValueError(f"cov has shape {tuple(cov.shape)}, expected ({self.D},) or ({self.D}, {self.D})")
        m = torch.broadcast_to(mean, (self.D,)).contiguous()
        cov = cov.contiguous()
        check(lib().bjx_set_elliptical_prior(self.h, kind, ptr(m), ptr(cov)), self.h)
        self._prior = given  # the key's tensors stay alive, so their addresses are not reused
        self._prior_key = key if None not in key else None

    def elliptical_slice_step(self, keys, q, logl, max_subiter, out=None, info_fields=None, chain_offset=0):
        """One elliptical slice transition (libbjx ``bjx_elliptical_slice_step``) under the installed prior."""
        keys = as_keys(keys, self.C, self.device)
        self._key_mode(keys, chain_offset)
        q = _f32(q, (self.C, self.D), "position")
        logl = _f32(logl, (self.C,), "logdensity")
        qo, lo = out if out is not None else (torch.empty_like(q), torch.empty_like(logl))
        info = self._info(info_fields or {}, _lib.EllipticalSliceInfo)
        check(lib().bjx_elliptical_slice_step(self.h, ptr(keys), ptr(q), ptr(logl), ptr(qo), ptr(lo), int(max_subiter),
                                              C.byref(info)), self.h)
        return qo, lo

    def ensure_slice_scale(self, scale):
        """Install slice sampling's direction scale (libbjx ``bjx_set_slice_direction_scale``) unless this exact content
        is installed, keyed as ``ensure_elliptical_prior``: a scalar (expanded to [D]), [D] or [D, D]."""
        if isinstance(scale, torch.Tensor):
            key = (scale.data_ptr(), tuple(scale.shape), scale._version, str(scale.device))
        else:
            key = ("scalar", float(scale)) if np.ndim(scale) == 0 else None
        given = scale
        if key is not None and key == getattr(self, "_slice_scale_key", None):
            return
        s = torch.as_tensor(scale, dtype=torch.float32, device=self.device)
        if s.ndim == 0:
            s = s.expand(self.D)
        if s.ndim == 1 and s.shape[0] == self.D:
            kind = _lib.METRIC_DIAG
        elif s.ndim == 2 and tuple(s.shape) == (self.D, self.D):
            kind = _lib.METRIC_DENSE
        else:
            raise ValueError(f"scale has shape {tuple(s.shape)}, expected (), ({self.D},) or ({self.D}, {self.D})")
        s = s.contiguous()
        check(lib().bjx_set_slice_direction_scale(self.h, kind, ptr(s)), self.h)
        self._slice_scale = (given, s)  # the key's tensor stays alive, so its address is not reused
        self._slice_scale_key = key

    def slice_step(self, keys, q, logp, width, interval, max_expansions, max_shrinkage, out=None, info_fields=None,
                   chain_offset=0):
        """One slice sampling transition (libbjx ``bjx_slice_step``) along a direction of the installed scale."""
        keys = as_keys(keys, self.C, self.device)
        self._key_mode(keys, chain_offset)
        q = _f32(q, (self.C, self.D), "position")
        logp = _f32(logp, (self.C,), "logdensity")
        qo, lo = out if out is not None else (torch.empty_like(q), torch.empty_like(logp))
        w, w_dev = self._eps(width, "width")
        info = self._info(info_fields or {}, _lib.SliceInfo)
        check(lib().bjx_slice_step(self.h, ptr(keys), ptr(q), ptr(logp), ptr(qo), ptr(lo), w, ptr(w_dev), int(interval),
                                   int(max_expansions), int(max_shrinkage), C.byref(info)), self.h)
        self._width_keepalive = w_dev  # the launch is asynchronous
        return qo, lo

    def ensure_rw_proposal(self, kind, sigma, mean=None):
        """Install random-walk Metropolis's Gaussian proposal (libbjx ``bjx_set_rw_proposal``) unless this exact content
        is installed, keyed as ``ensure_slice_scale``: ``kind`` ``RW_ADDITIVE`` (y = x + lin) or ``RW_INDEPENDENT``
        (y = mean + lin, ``mean`` a scalar or [D]); ``sigma`` a scalar (expanded to [D]), [D] or [D, D]."""
        def content_key(t):
            if t is None:
                return ("none",)
            if isinstance(t, torch.Tensor):
                return (t.data_ptr(), tuple(t.shape), t._version, str(t.device))
            return ("scalar", float(t)) if np.ndim(t) == 0 else None
        key = (int(kind), content_key(sigma), content_key(mean))
        given = (sigma, mean)
        if None not in key and key == getattr(self, "_rw_key", None):
            return
        s = torch.as_tensor(sigma, dtype=torch.float32, device=self.device)
        if s.ndim == 0:
            s = s.expand(self.D)
        if s.ndim == 1 and s.shape[0] == self.D:
            sigma_kind = _lib.METRIC_DIAG
        elif s.ndim == 2 and tuple(s.shape) == (self.D, self.D):
            sigma_kind = _lib.METRIC_DENSE
        else:
            raise ValueError(f"sigma has shape {tuple(s.shape)}, expected (), ({self.D},) or ({self.D}, {self.D})")
        s = s.contiguous()
        m = None
        if kind == _lib.RW_INDEPENDENT:
            m = torch.broadcast_to(torch.as_tensor(mean, dtype=torch.float32, device=self.device), (self.D,)).contiguous()
        check(lib().bjx_set_rw_proposal(self.h, int(kind), ptr(m), sigma_kind, ptr(s)), self.h)
        self._rw = (given, s, m)  # the key's tensors stay alive, so their addresses are not reused
        self._rw_key = key if None not in key else None

    def rw_step(self, keys, q, logp, correct=False, out=None, info_fields=None, chain_offset=0):
        """One random-walk Metropolis transition (libbjx ``bjx_rw_step``) with the installed proposal."""
        keys = as_keys(keys, self.C, self.device)
        self._key_mode(keys, chain_offset)
        q = _f32(q, (self.C, self.D), "position")
        logp = _f32(logp, (self.C,), "logdensity")
        qo, lo = out if out is not None else (torch.empty_like(q), torch.empty_like(logp))
        info = self._info(info_fields or {}, _lib.RwInfo)
        check(lib().bjx_rw_step(self.h, ptr(keys), ptr(q), ptr(logp), ptr(qo), ptr(lo), int(bool(correct)),
                                C.byref(info)), self.h)
        return qo, lo

    def adjusted_mclmc_num_steps(self, device_rule, avg, random_generator_arg):
        """The step counts int32 [C] of a dynamic rule ``device_rule = (rule, min_steps)`` at a per-chain ``avg`` [C]
        (libbjx ``bjx_adjusted_mclmc_num_steps``); random_generator_arg [C, 2] is read, not advanced.  The fixed rule
        clips at 1, as make_random_trajectory_length_fn(False) does."""
        rule, min_steps = device_rule
        if rule == _lib.AMCLMC_STEPS_FIXED:
            min_steps = max(int(min_steps), 1)
        avg = _f32(avg.to(self.device, torch.float32).contiguous(), (self.C,), "avg_num_integration_steps")
        rga = random_generator_arg.to(self.device).contiguous()
        out = torch.empty(self.C, dtype=torch.int32, device=self.device)
        check(lib().bjx_adjusted_mclmc_num_steps(self.h, int(rule), ptr(avg), int(min_steps), ptr(rga), ptr(out)), self.h)
        self._num_steps_keepalive = (avg, rga)
        return out

    def nuts_last_stats(self):
        a, b = C.c_int64(), C.c_int64()
        check(lib().bjx_nuts_last_stats(self.h, C.byref(a), C.byref(b)), self.h)
        return a.value, b.value

    def synchronize(self):
        check(lib().bjx_synchronize(self.h), self.h)


def get_engine(position, target, max_tree_depth=10, divergence_threshold=1000.0):
    """Engine cache keyed by (device, stream, shape, target identity, depth, threshold)."""
    if not isinstance(position, torch.Tensor) or not position.is_cuda:
        raise TypeError("position must be a CUDA tensor of shape [n_chains, dim]")
    if position.ndim != 2:
        raise ValueError("position must have shape [n_chains, dim] (the chain axis is explicit in blackjax_b200)")
    dev = position.device
    stream = torch.cuda.current_stream(dev)
    key = (dev.index, stream.cuda_stream, position.shape[0], position.shape[1], id(target), int(max_tree_depth),
           float(divergence_threshold))
    eng = _ENGINES.get(key)
    if eng is None:
        if position.shape[1] != target.dim:
            raise ValueError(f"position has dim {position.shape[1]} but the target has dim {target.dim}")
        eng = Engine(dev, position.shape[0], position.shape[1], target, max_tree_depth, divergence_threshold, stream)
        _ENGINES[key] = eng
        while len(_ENGINES) > _MAX_ENGINES:
            # drop the least recently used engine from the cache only: callers may still hold it (its handle and
            # workspaces are freed by Engine.__del__ once the last reference goes)
            _ENGINES.popitem(last=False)
    else:
        _ENGINES.move_to_end(key)
    return eng
