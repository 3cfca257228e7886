"""neurodiffeq_b200 -- an H100-native PINN residual-evaluation engine behind the neurodiffeq API.

Import root swap for the hot path of NeuroDiffGym/neurodiffeq: ``diff``/operators, ``FCNN``, the conditions and the
``Solver1D / Solver2D / SolverSpherical / BundleSolver1D`` ``.fit()`` loop, with the per-batch closure
(reference solvers.py:369-395) replaced by hand-written sm_90a CUDA kernels (``csrc/``) reached through the C ABI in
``include/pinnjet.h``.
"""
from .neurodiffeq import diff, safe_diff, unsafe_diff  # noqa: F401

__version__ = "0.1.0"
