"""Palindromic two-stage integrators of ``blackjax/mcmc/integrators.py:321-369`` as coefficient tables.

The kernels run ``generalized_two_stage_integrator`` (integrators.py:62-152) for any palindromic table:
even entries kick the momentum, odd entries drift the position and re-evaluate the gradient.  The numbers
below are the published constants of the schemes (velocity Verlet; McLachlan 1995 two-stage "minimal norm";
the three-stage scheme the reference calls yoshida; Omelyan et al. 2003 eleven-stage), as used by the
reference."""

velocity_verlet = (0.5, 1.0, 0.5)                                                   # integrators.py:321-322

_b1 = 0.1931833275037836
mclachlan = (_b1, 0.5, 1.0 - 2.0 * _b1, 0.5, _b1)                                   # integrators.py:335-340

_b1y, _a1y = 0.11888010966548, 0.29619504261126
yoshida = (_b1y, _a1y, 0.5 - _b1y, 1.0 - 2.0 * _a1y, 0.5 - _b1y, _a1y, _b1y)        # integrators.py:351-357

_b1o, _a1o, _b2o, _a2o = 0.08398315262876693, 0.2539785108410595, 0.6822365335719091, -0.03230286765269967
_b3o, _a3o = 0.5 - _b1o - _b2o, 1.0 - 2.0 * (_a1o + _a2o)
omelyan = (_b1o, _a1o, _b2o, _a2o, _b3o, _a3o, _b3o, _a2o, _b2o, _a1o, _b1o)        # integrators.py:363-369

# The isokinetic integrators of MCLMC (integrators.py:533-539) run the same tables: mclmc's kernel interprets even entries as
# the ESH momentum update and odd entries as the position update.
isokinetic_velocity_verlet = velocity_verlet
isokinetic_mclachlan = mclachlan
isokinetic_yoshida = yoshida
isokinetic_omelyan = omelyan


def as_coefficients(integrator):
    """Accepts one of the tables above (or any odd-length palindromic sequence of 3..11 floats)."""
    if isinstance(integrator, str):
        try:
            integrator = {"velocity_verlet": velocity_verlet, "mclachlan": mclachlan, "yoshida": yoshida,
                          "omelyan": omelyan, "isokinetic_velocity_verlet": velocity_verlet,
                          "isokinetic_mclachlan": mclachlan, "isokinetic_yoshida": yoshida,
                          "isokinetic_omelyan": omelyan}[integrator]
        except KeyError:
            raise ValueError(f"unknown integrator {integrator!r}") from None
    coef = tuple(float(c) for c in integrator)
    if len(coef) % 2 == 0 or not 3 <= len(coef) <= 11 or any(a != b for a, b in zip(coef, coef[::-1])):
        raise ValueError("integrator must be an odd-length (3..11) palindromic coefficient table")
    return coef
