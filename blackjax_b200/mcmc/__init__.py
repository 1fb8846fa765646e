from . import dynamic_hmc, ghmc, hmc, integrators, nuts  # noqa: F401
from . import metrics  # noqa: F401,E402
from . import composed  # noqa: F401,E402
from . import barker, mala  # noqa: F401,E402
from . import elliptical_slice  # noqa: F401,E402
from . import slice  # noqa: F401,E402
from . import random_walk  # noqa: F401,E402
