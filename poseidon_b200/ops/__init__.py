"""Op namespaces.  ``get(ctx)`` returns the engine a layer should call into:

* ``torch``  – :mod:`.torch_engine` (CPU, or cuDNN/cuBLAS through PyTorch: the baseline)
* ``sm100``  – :mod:`.sm100` (hand-written sm_90a CUDA kernels; requires an H100)
"""
from __future__ import annotations

from . import reference, torch_engine


def get(ctx):
    if ctx.engine == "sm100":
        from . import sm100
        return sm100
    return torch_engine
