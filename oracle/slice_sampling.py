"""The multivariate slice sampler (blackjax/mcmc/slice.py: build_kernel, direction_proposal, doubling, stepping_out,
_best_interval, _doubling_accept, _shrink; util.py generate_gaussian_noise) restated in float32 NumPy, chain by chain,
in the reference's own eager order: every doubling level's two ends are evaluated, both ends in every pass of the
acceptance test, and the test for every shrinkage candidate.  The acceptance test's bisection is capped at
max_expansions + 1 passes, as the device kernels cap it.  For every chain it also returns the smallest decision margin
|logp(x + t d) - level| over all its in-slice tests, so that a test can tell a disagreement from a tie."""
import numpy as np

from . import prng

F = np.float32


def best_interval(x):
    """_best_interval: the index of the first True, else the last."""
    x = np.asarray(x, np.int64)
    k = x.shape[0]
    return int(np.argmax(np.arange(2 * k, k, -1) * x + np.arange(k)))


def direction(keys, D, scale=1.0):
    """sample_direction for every chain: n = 0 + scale z ([D] or scalar scale) or scale @ z (dense), z =
    normal(prop_key, (D,)) with prop_key = split(key)[0]; d = n / |n|."""
    z = prng.normal(prng.split(keys)[:, 0], (D,))
    scale = np.asarray(scale, F)
    if scale.ndim == 2:
        n = (z.astype(np.float64) @ scale.astype(np.float64).T).astype(F)
    else:
        n = (scale * z).astype(F)
    n = (F(0) + n).astype(F)
    nrm = np.sqrt(np.sum(n.astype(np.float64) ** 2, axis=1)).astype(F)
    return (n / nrm[:, None]).astype(F)


def doubling_accept(in_slice, t, left, right, width, max_passes):
    """_doubling_accept with at most max_passes bisections; returns (ok, passes)."""
    left, right, t = F(left), F(right), F(t)
    thr = F(F(1.1) * F(width))
    d, ok, passes = False, True, 0
    with np.errstate(invalid="ignore", over="ignore"):
        while F(right - left) > thr and ok and passes < max_passes:
            mid = F(F(0.5) * F(left + right))
            d = d or (F(0) < mid and t >= mid) or (F(0) >= mid and t < mid)
            if t < mid:
                right = mid
            if t >= mid:
                left = mid
            both_out = (not in_slice(left)) and (not in_slice(right))
            ok = not (d and both_out)
            passes += 1
    return ok, passes


def chain_step(key, x, logp, fn, d, width=1.0, interval="doubling", max_expansions=10, max_shrinkage=100):
    """One transition of one chain: key [2], x [D], logp, fn maps [n, D] to ([n], grad), d [D] the direction.
    Returns (x, logp, info) with info is_accepted, num_expansions, num_shrink, bracket_left, bracket_right and margin."""
    width = F(width)
    slice_key = prng.split(key)[1]
    level_key, interval_key, shrink_key = prng.split(slice_key, 3)
    with np.errstate(divide="ignore"):
        level = F(F(logp) + np.log(prng.uniform(level_key)))
    margin = [np.inf]

    def point(t):
        with np.errstate(invalid="ignore", over="ignore"):
            return (x + (F(t) * d).astype(F)).astype(F)

    def evaluate(t):
        with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
            lp = F(np.asarray(fn(point(t)[None])[0], F)[0])
            m = abs(float(lp) - float(level))
        if not np.isnan(m):
            margin[0] = min(margin[0], m)
        return lp, bool(lp >= level)

    def in_slice(t):
        return evaluate(t)[1]

    k = max_expansions + 1
    if interval == "doubling":
        key1, key2 = prng.split(interval_key)
        l0 = F(F(-width) * prng.uniform(key1))
        r0 = F(l0 + width)
        left_expands = prng.uniform(key2, (k,)) < F(0.5)
        with np.errstate(over="ignore", invalid="ignore"):
            sw = (width * np.ldexp(F(1), np.arange(k)).astype(F)).astype(F)
            lacc, racc = F(0), F(0)
            lefts, rights = np.empty(k, F), np.empty(k, F)
            for j in range(k):  # exclusive cumulative sums, in index order
                lefts[j], rights[j] = F(l0 - lacc), F(r0 + racc)
                lacc = F(lacc + F(sw[j] * F(left_expands[j])))
                racc = F(racc + F(sw[j] * F(1 - int(left_expands[j]))))
        both_out = [not in_slice(a) and not in_slice(b) for a, b in zip(lefts, rights)]
        idx = best_interval(both_out)
        left, right, n_exp = lefts[idx], rights[idx], idx

        def accept(t):
            return doubling_accept(in_slice, t, left, right, width, k)[0]
    elif interval == "stepping_out":
        u_key, jk_key = prng.split(interval_key)
        left = F(F(-width) * prng.uniform(u_key))
        right = F(left + width)
        j = int(np.floor(F(F(max_expansions) * prng.uniform(jk_key))))
        kk = max_expansions - 1 - j
        jl, kr = j, kk
        while in_slice(left) and jl > 0:
            left, jl = F(left - width), jl - 1
        while in_slice(right) and kr > 0:
            right, kr = F(right + width), kr - 1
        n_exp = (j - jl) + (kk - kr)

        def accept(t):
            return True
    else:
        raise ValueError(interval)

    skey = shrink_key
    l, r = left, right
    n, found = 0, False
    x_new, lp_new = x, F(logp)
    while not found and n < max_shrinkage:
        skey, sub = prng.split(skey)
        with np.errstate(invalid="ignore", over="ignore"):
            t = F(l + F(prng.uniform(sub) * F(r - l)))
        lp, ins = evaluate(t)
        ok = accept(t)  # eager: the test runs for every candidate
        found = ins and ok
        if found:
            x_new, lp_new = point(t), lp
        if t < 0:
            l = t
        if t >= 0:
            r = t
        n += 1
    info = dict(is_accepted=found, num_expansions=n_exp, num_shrink=n, bracket_left=F(left), bracket_right=F(right),
                margin=margin[0])
    return x_new, F(lp_new), info


def step(keys, x, logp, fn, scale=1.0, width=1.0, interval="doubling", max_expansions=10, max_shrinkage=100):
    """One transition of every chain: keys [C, 2]; x [C, D]; logp [C]; width a scalar or [C].  Returns ((x, logp),
    info) with info's fields stacked over chains, plus the directions."""
    x, logp = np.asarray(x, F), np.asarray(logp, F)
    C, D = x.shape
    d = direction(keys, D, scale)
    w = np.broadcast_to(np.asarray(width, F), (C,))
    out_x, out_l, infos = np.empty_like(x), np.empty(C, F), []
    for c in range(C):
        out_x[c], out_l[c], info = chain_step(keys[c], x[c], logp[c], fn, d[c], w[c], interval, max_expansions,
                                              max_shrinkage)
        infos.append(info)
    info = {k: np.array([i[k] for i in infos]) for k in infos[0]}
    info["is_accepted"] = info["is_accepted"].astype(bool)
    info["num_expansions"] = info["num_expansions"].astype(np.int32)
    info["num_shrink"] = info["num_shrink"].astype(np.int32)
    info["direction"] = d
    return (out_x, out_l), info
