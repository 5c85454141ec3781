"""CPU: argument rules of the fp16 index storage that hold without a GPU."""
import ctypes
import types

import pytest
import torch


def test_storage_argument_rules():
    from openmatch_b200 import _lib
    from openmatch_b200.index import FlatIPIndex
    lib = _lib.load()
    h = ctypes.c_void_p()
    # bf16 storage is refused before any device is needed; the scan operand must stay fp16
    assert lib.om_index_create_typed(16, _lib.OM_BF16, ctypes.byref(h)) == -1
    assert lib.om_index_create_typed(16, 7, ctypes.byref(h)) == -1 and b"OM_F16" in lib.om_last_error()
    with pytest.raises(ValueError, match="float16"):
        FlatIPIndex(16, dtype=torch.bfloat16)


def test_index_dtype_argument():
    from openmatch_b200.arguments import InferenceArguments
    from openmatch_b200.retriever.dense_retriever import _index_dtype
    assert InferenceArguments.__dataclass_fields__["index_dtype"].default == "float32"
    assert _index_dtype(types.SimpleNamespace(index_dtype="float16")) == torch.float16
    assert _index_dtype(types.SimpleNamespace(index_dtype="float32")) == torch.float32
    with pytest.raises(ValueError, match="index_dtype"):
        _index_dtype(types.SimpleNamespace(index_dtype="bfloat16"))
