"""Homotopy -- mirror of src/utils/homotopy.jl: the continuation parameter of a smooth approximation (e.g. the sharpness
kappa of a sigmoid) as a function of a progress variable x in [0, 1]."""
from __future__ import annotations

import math


class Homotopy:
    """Homotopy(delta_min; delta_max = 1, eps = 1e-2) (homotopy.jl:45-56): h(x) = log(1/eps - 1) / (rho^x delta_max)
    with rho = delta_min / delta_max, so that the sigmoid reaches 1 - eps at a transition half-width delta_max for x = 0
    and delta_min for x = 1 (homotopy.jl:70-73)."""

    def __init__(self, delta_min: float, delta_max: float = 1.0, eps: float = 1e-2):
        self.eps, self.delta_min, self.delta_max = float(eps), float(delta_min), float(delta_max)
        self.rho = self.delta_min / self.delta_max

    def __call__(self, x: float) -> float:
        return math.log(1 / self.eps - 1) / (self.rho ** x * self.delta_max)
