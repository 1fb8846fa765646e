"""CPU restatements ("oracles") of the BlackJAX samplers and warm-ups that ``blackjax_b200`` runs on the GPU.

TEST INFRASTRUCTURE ONLY.  Nothing under ``oracle/`` is imported by the product
package ``blackjax_b200``; only ``tests/``, ``__graft_entry__.smoke()`` and the
``cpu_baseline`` / ``--impl reference`` legs of ``bench.py`` may use it, and
there only as the checker / the CPU timing stand-in.

Modules (each names the reference files and lines it follows):

* building blocks   ``prng`` (threefry2x32 and the JAX samplers), ``targets``
                    (analytic ``value_and_grad`` of the named targets),
                    ``diagnostics`` (R-hat, ESS), ``cport`` (ctypes wrapper of the
                    C twin of the HMC path in ``oracle/c/``)
* samplers          ``hmc``, ``nuts``, ``ghmc``, ``mclmc`` (the isokinetic
                    integrators), ``adjusted_mclmc`` (MAMS, static and dynamic
                    trajectory lengths)
* warm-ups          ``adaptation`` (Stan window adaptation: dual averaging, Welford
                    and Chan-Golub-LeVeque moments), ``low_rank_window``
                    (``window_adaptation_low_rank``), ``chees``, ``meads``,
                    ``meads_lrd`` (MEADS with a low-rank metric), ``mclmc_tuning``
                    (``mclmc_find_L_and_step_size``), ``adjusted_mclmc_tuning``
                    (``adjusted_mclmc_find_L_and_step_size``), ``laps``

Why a restatement: the reference (blackjax-devs/blackjax @ 63912a4) is pure
Python on top of ``jax 0.10.0`` (uv.lock:1309-1310), which is NOT installed in
this image (no wheel, no network), so the reference cannot be imported or run
here.  The arithmetic that fixes sample values (threefry2x32 PRNG, the
bits->uniform->normal transforms, ``expit``/``logaddexp``) lives in that absent
dependency; ``oracle/prng.py`` restates its published algorithm.

Pinning status
--------------
* Building blocks are pinned against every known-answer test the reference's
  own test-suite holds for this path (see ``tests/test_oracle_kat.py``):
  velocity-Verlet golden end state (tests/mcmc/test_integrators.py:74-103),
  momentum-draw identity (tests/mcmc/test_metrics.py:124-179), NUTS discrete
  outcomes (tests/mcmc/test_trajectory.py:193-260), sub-tree divergence
  (:20-74), iterative U-turn truth table (tests/mcmc/test_uturn.py:13-43),
  progressive == recursive (test_trajectory.py:76-191), warm-up schedule
  (tests/adaptation/test_adaptation.py:27-49), and the JAX PRNG known answers
  recorded in SURVEY.md section 8c.  The later oracles are checked against the
  reference's own tests of their algorithms in ``tests/test_*_oracle.py``.
* SAMPLE-LEVEL PARITY (same seed -> same draw as live JAX) IS **UNPINNED**:
  the reference stores no sample-level golden vectors and JAX cannot be run
  here.  "parity unpinned" at that level; see DESIGN.md.

The arithmetic is float32 (JAX default, x64 disabled), vectorised over chains
with masks, i.e. what ``jax.vmap`` of the reference kernels computes.  The
exceptions say so in their docstrings: ``low_rank_window`` is float64, and
``laps`` forms its ensemble averages as float64 sums.
"""
