"""The C-ABI library: loads without a GPU, exports every symbol include/pyflyt_b200.h declares,
agrees with Python on struct layouts, and refuses to compute without a device (no CPU fallback)."""
import ctypes
import os
import re

import pytest

from pyflyt_b200 import _lib
from pyflyt_b200.models import PfbEnvConfig, PfbModel, build_model

HEADER = os.path.join(os.path.dirname(__file__), "..", "include", "pyflyt_b200.h")


@pytest.fixture(scope="module")
def L():
    if not os.path.exists(_lib.LIB_PATH):
        _lib.build()
    return _lib.lib()


def test_header_symbols_are_exported(L):
    text = open(HEADER).read()
    declared = set(re.findall(r"\b(pfb_[a-z_]+)\s*\(", text))
    assert declared == set(_lib.EXPORTS), declared ^ set(_lib.EXPORTS)
    for name in declared:
        assert hasattr(L, name), name


def test_struct_layouts_agree(L):
    assert L.pfb_abi_version() == 1
    assert L.pfb_sizeof_model() == ctypes.sizeof(PfbModel)
    assert L.pfb_sizeof_env_config() == ctypes.sizeof(PfbEnvConfig)
    assert L.pfb_sizeof_buffers() == ctypes.sizeof(_lib.PfbBuffers)


def test_no_cpu_fallback(L):
    import torch

    if torch.cuda.is_available():
        pytest.skip("a device is present")
    m = build_model("quadx")
    h = ctypes.c_void_p()
    rc = L.pfb_create(ctypes.byref(m), None, 8, 0, 0, ctypes.byref(h))
    assert rc != 0 and not h.value
    assert b"no CPU fallback" in L.pfb_last_error()
    from pyflyt_b200.core.aviary import BatchedAviary
    import numpy as np

    with pytest.raises(_lib.PfbError):
        BatchedAviary(np.zeros((2, 3)), np.zeros((2, 3)))


@pytest.mark.parametrize("value", [2, -1])
def test_create_refuses_inline_reset_other_than_0_or_1(L, value):
    """``inline_reset`` is a flag; the check comes before the device lookup, so it is the same with and without a GPU."""
    from engines import hover_config

    env = hover_config(autoreset=True)
    env.inline_reset = value
    h = ctypes.c_void_p()
    assert L.pfb_create(ctypes.byref(build_model("quadx")), ctypes.byref(env), 8, 0, 0, ctypes.byref(h)) != 0 and not h.value
    assert L.pfb_last_error() == f"inline_reset must be 0 or 1, got {value}".encode()


def test_aviary_argument_checks_match_reference_messages():
    import numpy as np

    from pyflyt_b200.core.aviary import AviaryInitException, BatchedAviary

    with pytest.raises(AviaryInitException, match="start_pos must be shape"):
        BatchedAviary(np.zeros(3), np.zeros(3))
    with pytest.raises(AviaryInitException, match="start_orn must be same shape"):
        BatchedAviary(np.zeros((2, 3)), np.zeros((3, 3)))
    with pytest.raises(AviaryInitException, match="Can't find `drone_type`"):
        BatchedAviary(np.zeros((2, 3)), np.zeros((2, 3)), drone_type="blimp")
