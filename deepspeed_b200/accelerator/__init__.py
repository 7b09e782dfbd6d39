"""Device abstraction for deepspeed_b200.

Parity target: reference ``accelerator/abstract_accelerator.py`` (the 69-method ABC) and
``accelerator/real_accelerator.py:51 get_accelerator``.  The reference dispatches over eight
vendors; this framework is H100-only, so there are exactly two concrete devices:

* :class:`B200Accelerator` -- CUDA sm_90a, NCCL over NVLink 5.
* :class:`HostAccelerator` -- CPU + gloo, used by the no-GPU test tier and by the
  GPT-2/gloo plumbing config in BASELINE.json.

The method names follow the reference ABC so user code written against
``deepspeed.accelerator.get_accelerator()`` keeps working.
"""
from .real_accelerator import get_accelerator, set_accelerator, is_current_accelerator_supported  # noqa: F401
from .b200_accelerator import B200Accelerator  # noqa: F401
from .host_accelerator import HostAccelerator  # noqa: F401
from .base import AcceleratorBase as DeepSpeedAccelerator  # noqa: F401,E402  (reference ABC name)
