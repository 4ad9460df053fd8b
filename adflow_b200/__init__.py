"""adflow_b200 -- H100-native (sm_90a CUDA) drop-in for ADflow's per-block
residual / smoother / matrix-free Jacobian-vector hot path.

Only what the path needs lives here: ``csrc/`` (CUDA kernels + the C ABI of
``include/adflow_b200.h``), ``_lib`` (ctypes loader, fails loudly without the CUDA
library), ``solver`` (host-side mirror of the pyADflow calls on the path),
``params``/``layout``/``synthetic`` (options, array extents, synthetic workload).
"""
from .layout import BlockDims, HostBlock  # noqa: F401
from .params import AdfbParams, make_params  # noqa: F401

__version__ = "0.1.0"
