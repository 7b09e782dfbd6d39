"""Accelerator selection (reference: ``accelerator/real_accelerator.py:51``).

``DS_ACCELERATOR`` (reference env name) or ``DSB200_ACCELERATOR`` may force ``cuda`` / ``cpu``;
otherwise CUDA is chosen whenever a device is visible.
"""
import os

_accel = None
SUPPORTED = ("cuda", "cpu")


def is_current_accelerator_supported():
    return get_accelerator().device_name() in SUPPORTED


def get_accelerator():
    global _accel
    if _accel is not None:
        return _accel
    import torch
    forced = os.environ.get("DSB200_ACCELERATOR", os.environ.get("DS_ACCELERATOR"))
    if forced is not None and forced not in SUPPORTED:
        raise ValueError(f"accelerator {forced!r} is not supported; this framework targets H100 (cuda) "
                         f"with a cpu/gloo tier for tests. Choose from {SUPPORTED}.")
    name = forced or ("cuda" if torch.cuda.is_available() else "cpu")
    if name == "cuda":
        from .b200_accelerator import B200Accelerator
        _accel = B200Accelerator()
    else:
        from .host_accelerator import HostAccelerator
        _accel = HostAccelerator()
    return _accel


def set_accelerator(accel_obj):
    global _accel
    _accel = accel_obj
