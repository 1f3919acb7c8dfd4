"""k4nerf -- H100 (sm_90a) drop-in for the 4K-NeRF rendering hot path.

Host-side mirror of the reference's model API (frozoul/4K-NeRF ``lib/dvgo.py``, ``lib/dmpigo.py``,
``lib/grid.py``, ``lib/sr_esrnet.py`` and ``render_viewpoints`` of ``run.py`` / ``run_sr.py``)
over the C-ABI CUDA library ``libk4nerf.so`` (``include/k4nerf.h``).  PyTorch is used for device
memory, streams and ``torch.distributed`` only; every hot op is a hand-written sm_90a kernel.
There is NO CPU fallback: a missing library or CPU tensors raise.
"""
from . import _lib  # noqa: F401  (fails loudly if libk4nerf.so is missing)
from . import act, grid, dvgo, dmpigo, dcvgo, utils, render, sr_esrnet, masked_adam  # noqa: F401
from .masked_adam import MaskedAdam  # noqa: F401
from .dvgo import DirectVoxGO, get_rays_of_a_view  # noqa: F401
from .dmpigo import DirectMPIGO  # noqa: F401
from .dcvgo import DirectContractedVoxGO  # noqa: F401
from .sr_esrnet import SFTNet  # noqa: F401

__all__ = ['DirectVoxGO', 'DirectMPIGO', 'DirectContractedVoxGO', 'SFTNet', 'get_rays_of_a_view', 'grid', 'dvgo', 'dmpigo', 'utils', 'render',
           'sr_esrnet', 'act']
