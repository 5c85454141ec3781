"""CPU: the rules of the host-resident index that hold without a GPU: ``--index_memory`` parsing, the paths that refuse
it before any GPU work, and the window argument of ``om_index_create_host``."""
import ctypes
import types

import pytest
import torch


def test_create_host_argument_rules():
    from openmatch_b200 import _lib
    from openmatch_b200.index import FlatIPIndex
    lib = _lib.load()
    h = ctypes.c_void_p()
    for window in (-256, 1, 300, 1000):
        assert lib.om_index_create_host(16, _lib.OM_F32, window, ctypes.byref(h)) == -1 and not h.value
        assert b"multiple of 256" in lib.om_last_error()
    assert lib.om_index_create_host(16, _lib.OM_BF16, 256, ctypes.byref(h)) == -1 and not h.value
    assert lib.om_index_create_host(0, _lib.OM_F32, 256, ctypes.byref(h)) == -1
    with pytest.raises(ValueError, match="memory"):
        FlatIPIndex(16, memory="disk")


def test_index_memory_argument():
    from transformers import HfArgumentParser
    from openmatch_b200.arguments import InferenceArguments
    from openmatch_b200.retriever.dense_retriever import _index_memory
    assert InferenceArguments.__dataclass_fields__["index_memory"].default == "device"
    (args,) = HfArgumentParser(InferenceArguments).parse_args_into_dataclasses(
        ["--output_dir", "unused", "--index_memory", "host"])
    assert args.index_memory == "host"
    one = dict(world_size=1)
    assert _index_memory(types.SimpleNamespace(**one)) == "device"
    assert _index_memory(types.SimpleNamespace(index_memory="device", world_size=4), writes_rows=True) == "device"
    assert _index_memory(types.SimpleNamespace(index_memory="host", **one)) == "host"
    with pytest.raises(ValueError, match="index_memory"):
        _index_memory(types.SimpleNamespace(index_memory="disk", **one))
    with pytest.raises(ValueError, match="world_size is 2"):
        _index_memory(types.SimpleNamespace(index_memory="host", world_size=2))
    with pytest.raises(ValueError, match="in place"):
        _index_memory(types.SimpleNamespace(index_memory="host", **one), writes_rows=True)


class _Model(torch.nn.Module):
    def to(self, *a, **kw):  # would be the first GPU work of a Retriever
        raise AssertionError("GPU work before the --index_memory check")


def _args(tmp, **kw):
    base = dict(device=torch.device("cpu"), output_dir=str(tmp), process_index=0, local_process_index=0, world_size=1,
                index_memory="host")
    base.update(kw)
    return types.SimpleNamespace(**base)


def test_retriever_refuses_host_index_before_gpu_work(tmp_path):
    from openmatch_b200.retriever.dense_retriever import Retriever
    with pytest.raises(ValueError, match="world_size is 2"):
        Retriever.from_embeddings(_Model(), _args(tmp_path, world_size=2, process_index=0))
    for build in (Retriever.build_all, Retriever.build_embeddings):
        with pytest.raises(ValueError, match="in place"):
            build(_Model(), [object()], _args(tmp_path))
    r = Retriever.__new__(Retriever)  # a retriever built elsewhere: doc_embedding_inference checks before encoding
    r.args, r.corpus_dataset, r.index = _args(tmp_path), [object()], None
    with pytest.raises(ValueError, match="in place"):
        r.doc_embedding_inference()
