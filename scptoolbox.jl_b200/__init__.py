"""scptoolbox.jl_b200 -- CUDA SCP inner loop for the H100 (discretize! + subproblem solve) behind a C ABI.

The directory name carries a dot, so the package is imported under the alias
`scptoolbox_jl_b200` (see __graft_entry__.load_package()).
"""
from . import gusto, homotopy, lib, ordering, parser, problem, ptr, scvx, sharded  # noqa: F401
from . import examples  # noqa: F401
from .examples import starship as _starship  # noqa: F401
from .examples import rocket_landing as _rocket_landing  # noqa: F401
from .examples import double_integrator as _double_integrator  # noqa: F401
from .examples import freeflyer as _freeflyer  # noqa: F401
from .examples import quadrotor as _quadrotor  # noqa: F401
from .examples import rendezvous_planar as _rendezvous_planar  # noqa: F401
from .examples import oscillator as _oscillator  # noqa: F401
from .lib import Handle, ScpbError  # noqa: F401
