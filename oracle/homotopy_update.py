"""Oracle of the in-loop homotopy schedule: the callback of test/examples/rendezvous_3d/definition.jl:96-151 as PTR.solve
calls it (src/solvers/ptr.jl:484-512), restated independently of the product code.

  HomotopyUpdate      the callback's rule on one seed: grid index, last_update, iter_max
  scripted_loop       the PTR loop's control flow (unsafe exit, stopping rule, callback, iter_max) driven by scripted
                      improv_rel / stop sequences, for tests of the rule alone
  CallbackPTR         the oracle IMPULSE PTR loop (oracle/rendezvous.py) with the callback: kappa = grid[index] whenever a
                      subproblem is built; records improv_rel, grid index, iter_max and J_aug per iteration

The reference mutates the shared pars.iter_max and mdl.traj.hom, so both carry over to the next PTR.create on the same
parameters; here every solve starts from grid[0], last_update = 1 and the configured iter_max, as the device does.
"""
from __future__ import annotations

import math

import numpy as np

from . import rendezvous as rz


class HomotopyUpdate:
    """One seed's state of the callback.  last_update starts at 1: the reference reads ref.bay[:last_update] and falls
    back to 1 while the reference solution carries none (definition.jl:117)."""

    def __init__(self, grid, beta, worsen_tol=-1e-3, iter_max=30):
        self.grid = [float(g) for g in grid]
        self.beta, self.worsen_tol = float(beta), float(worsen_tol)
        self.index, self.last_update, self.iter_max = 0, 1, int(iter_max)

    @property
    def kappa(self):
        return self.grid[self.index]

    def __call__(self, it, improv_rel):
        """the callback after the stopping rule of iteration `it`; returns whether it acted (definition.jl:111-134).
        A NaN improv_rel compares false both ways, so nothing acts on it."""
        increase = improv_rel <= self.beta and improv_rel >= self.worsen_tol
        if increase and self.index < len(self.grid) - 1:
            self.index += 1
            self.iter_max += it - self.last_update
            self.last_update = it
            return True
        return False


def scripted_loop(rule: HomotopyUpdate, improv_rel, stop, unsafe_at=None):
    """ptr.jl:465-526 with scripted iteration outcomes: improv_rel[k-1] and stop[k-1] are iteration k's; the sequences
    must cover every iteration the loop runs.  Returns (iterations, status, index history, iter_max history) with status
    0 = stopped on the rule, 1 = iter_max reached, 2 = unsafe subproblem (the callback does not run, ptr.jl:488-491)."""
    k, hist_idx, hist_itmax = 1, [], []
    while True:
        hist_idx.append(rule.index)
        if unsafe_at is not None and k == unsafe_at:
            hist_itmax.append(rule.iter_max)
            return k, 2, hist_idx, hist_itmax
        acted = rule(k, improv_rel[k - 1])
        hist_itmax.append(rule.iter_max)
        if stop[k - 1] and not acted:
            return k, 0, hist_idx, hist_itmax
        k += 1
        if k > rule.iter_max:
            return k - 1, 1, hist_idx, hist_itmax


class CallbackPTR(rz.ImpulsePTR):
    """The oracle IMPULSE PTR loop of oracle/rendezvous.py with the homotopy callback."""

    def solve_with_schedule(self, guess, grid, beta, worsen_tol=-1e-3, prefer="ipm", verbose=False):
        rule = HomotopyUpdate(grid, beta, worsen_tol, self.pars.iter_max)
        xd, ud, p = guess
        ref = self.make_solution(xd, ud, p)
        hist = dict(improv_rel=[], index=[], iter_max=[], J_aug=[], acted=[])
        k, status, last, on_rule = 1, "SCP_FAILED", None, False
        while True:
            self.set_kappa(rule.kappa)
            hist["index"].append(rule.index)
            sol = self.solve_subproblem(ref, prefer=prefer)[0]
            last = sol
            if sol.status not in ("OPTIMAL", "ALMOST_OPTIMAL"):
                status = f"SCP_FAILED ({sol.status})"
                for key in ("improv_rel", "J_aug"):
                    hist[key].append(math.nan)
                hist["iter_max"].append(rule.iter_max)
                hist["acted"].append(False)
                break
            stop = self.check_stop(k, ref, sol)
            acted = rule(k, sol.improv_rel)
            hist["improv_rel"].append(sol.improv_rel)
            hist["J_aug"].append(sol.J_aug)
            hist["iter_max"].append(rule.iter_max)
            hist["acted"].append(acted)
            if verbose:
                print(f"{k:3d} J {sol.J_aug:+.9e} improv {sol.improv_rel:+.3e} hom {rule.index} itmax {rule.iter_max}"
                      f"{' *' if acted else ''}{' stop' if stop else ''}", flush=True)
            status = "SCP_SOLVED"
            if stop and not acted:
                on_rule = True
                break
            ref = sol
            k += 1
            if k > rule.iter_max:
                k -= 1
                break
        out = {key: np.array(v) for key, v in hist.items()}
        return dict(status=status, iterations=k, sol=last, history=out, index=rule.index, iter_max=rule.iter_max,
                    stopped_on_rule=on_rule)
