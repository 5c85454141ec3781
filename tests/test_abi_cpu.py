"""CPU: the C-ABI library loads and exports every symbol include/openmatch_b200.h declares; no compute
entry point works without a GPU (no silent CPU fallback)."""
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    text = open(os.path.join(ROOT, "include", "openmatch_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(om_[a-z0-9_]+)\s*\(", text)))


def test_abi_v2_exports_and_binds_every_header_symbol():
    from openmatch_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        from openmatch_b200.build import build
        build()
    lib = _lib.load()
    declared = _declared_symbols()
    assert len(declared) >= 20
    for name in declared:
        assert hasattr(lib, name), "library does not export %s" % name
        assert name in _lib.SIGNATURES, "ctypes binding lacks %s" % name
    assert lib.om_abi_version() == 2


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_no_cpu_fallback():
    import ctypes

    from openmatch_b200 import _lib
    lib = _lib.load()
    assert lib.om_device_sm_count() < 0
    h = ctypes.c_void_p()
    rc = lib.om_index_create(64, ctypes.byref(h))
    assert rc < 0 and b"no CPU path" in lib.om_last_error()
    with pytest.raises(RuntimeError):
        _lib.check(rc)
