"""The NUTS oracle with per-chain metrics and step sizes: a batch of chains must equal the chains run one at a time.
This is what ``jax.vmap`` over chains computes, and the per-chain warm-up tests compare the device against it.  CPU only."""
import numpy as np
import pytest

from oracle import adaptation, hmc, nuts, prng, targets

F = np.float32


@pytest.mark.parametrize("per_chain_eps", [False, True])
def test_batched_nuts_equals_single_chain_runs_with_per_chain_metric(per_chain_eps):
    C, D, depth = 64, 8, 8
    otgt = targets.DiagGaussian(np.logspace(-0.5, 0.5, D))
    rs = np.random.default_rng(3)
    q = (rs.standard_normal((C, D)) * otgt.scale).astype(F)
    imm = np.exp(rs.uniform(-1.5, 1.5, (C, D))).astype(F)
    eps = (0.3 * np.exp(rs.uniform(-0.3, 0.3, C))).astype(F) if per_chain_eps else F(0.3)
    keys = prng.split(prng.key(11), C)
    margins = np.full(C, np.inf)
    new, info = nuts.nuts_kernel(keys, hmc.init(q, otgt), otgt, eps, adaptation._PerChainDiag(imm), depth,
                                 margins=margins)
    assert len(np.unique(info.num_integration_steps)) >= 4     # the trees really differ between chains
    for c in range(C):
        m1 = np.full(1, np.inf)
        e1 = eps[c:c + 1] if per_chain_eps else eps
        n1, i1 = nuts.nuts_kernel(keys[c:c + 1], hmc.init(q[c:c + 1], otgt), otgt, e1, hmc.Metric(imm[c]), depth,
                                  margins=m1)
        for name in ("num_integration_steps", "num_trajectory_expansions", "is_turning", "is_divergent", "energy",
                     "acceptance_rate"):
            np.testing.assert_array_equal(getattr(info, name)[c], getattr(i1, name)[0], err_msg=f"chain {c}: {name}")
        for a, b in zip(new, n1):
            np.testing.assert_array_equal(a[c], b[0], err_msg=f"chain {c}: state")
        for k in range(4):
            np.testing.assert_array_equal(info.trajectory_leftmost_state[k][c], i1.trajectory_leftmost_state[k][0])
            np.testing.assert_array_equal(info.trajectory_rightmost_state[k][c], i1.trajectory_rightmost_state[k][0])
        assert margins[c] == m1[0], f"chain {c}: margin"


def test_chain_view_of_shared_and_per_chain_metrics():
    m = hmc.Metric(np.array([1.0, 2.0], F))
    assert m.chain(5) is m
    imm = np.arange(1, 7, dtype=F).reshape(3, 2)
    v = adaptation._PerChainDiag(imm).chain(1)
    assert v.imm.shape == (2,) and (v.imm == imm[1]).all() and (v.mass_sqrt == F(1.0) / np.sqrt(imm[1])).all()
