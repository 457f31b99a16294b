"""Loading of the native runtime and kernel-path selection.

On a GPU box the sm_90a extension is mandatory: ops fail loudly instead of silently falling back to eager PyTorch
(set ``TUTEL_B200_ALLOW_FALLBACK=1`` to permit a fallback, e.g. when debugging on another architecture).
"""
from __future__ import annotations

import logging
import os

import torch

_C = None
_ERR = None


def _load():
    global _C, _ERR
    if _C is not None or _ERR is not None:
        return
    try:
        from .. import _C as ext  # in-tree build: tutel_b200/_C*.so
        _C = ext
    except Exception as first:  # noqa
        if int(os.environ.get('TUTEL_B200_AUTO_BUILD', '1')):
            try:
                from .. import _build
                _build.build()
                import importlib
                _C = importlib.import_module('tutel_b200._C')
                return
            except Exception as ex:  # noqa
                _ERR = ex
        else:
            _ERR = first
        logging.warning('tutel_b200: native extension unavailable (%s)', _ERR)


def ext():
    """The native module, or None when it could not be built/loaded."""
    _load()
    return _C


def require_ext():
    _load()
    if _C is None:
        raise RuntimeError('tutel_b200: the native sm_90a extension (tutel_b200/_C*.so) is missing: %r. '
                           'Run `python -m tutel_b200._build`.' % (_ERR,))
    return _C


def has_ext() -> bool:
    return ext() is not None


def allow_fallback() -> bool:
    return bool(int(os.environ.get('TUTEL_B200_ALLOW_FALLBACK', '0')))


_SM90 = {}


def is_sm90(device=None) -> bool:
    if not torch.cuda.is_available():
        return False
    idx = torch.cuda.current_device() if device is None or getattr(device, 'index', None) is None else device.index
    if idx not in _SM90:
        _SM90[idx] = torch.cuda.get_device_capability(idx) == (9, 0)
    return _SM90[idx]


def has_cuda_ext() -> bool:
    """True when CUDA tensors should take the native kernel path."""
    if not torch.cuda.is_available():
        return False
    if ext() is None:
        if allow_fallback():
            return False
        require_ext()
    return True


def use_wgmma(t: torch.Tensor) -> bool:
    """Expert GEMMs go to the hand-written wgmma kernel for fp16/bf16 CUDA tensors on sm_90."""
    if not (t.is_cuda and t.dtype in (torch.bfloat16, torch.float16)):
        return False
    if os.environ.get('TUTEL_B200_GEMM', 'wgmma').lower() in ('cublas', 'torch'):
        return False
    return has_cuda_ext() and is_sm90(t.device)


# ---- native launch accounting (bench.py reports it as `gpu_launches`) ----------------------------------------------
_LAUNCHES = [0]


def count_launch(n: int = 1) -> None:
    _LAUNCHES[0] += n


def launch_count() -> int:
    return _LAUNCHES[0]
