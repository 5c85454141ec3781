"""CPU: the Python side of filtered search, without a GPU: the allowed-row bit packing, the exclusion CSR, the doc-id
mapping of ``Retriever.search(allowed_docs=, exclude=)`` and the argument errors raised before the library is called."""
import numpy as np
import pytest
import torch

from openmatch_b200.index import exclusion_csr, local_allow, pack_allow, unpack_allow
from openmatch_b200.retriever.dense_retriever import doc_filter


@pytest.mark.parametrize("n", [0, 1, 31, 32, 33, 64, 1000])
def test_pack_allow_bit_layout(n):
    rng = np.random.default_rng(n)
    mask = rng.random(n) < 0.5
    words = pack_allow(mask, n)
    assert words.dtype == torch.int32 and words.numel() == (n + 31) // 32
    u = words.numpy().view(np.uint32)
    for r in range(n):  # bit r & 31 of word r >> 5
        assert bool((u[r >> 5] >> (r & 31)) & 1) == mask[r]
    if n % 32:
        assert (u[-1] >> (n % 32)) == 0, "bits past n are zero"
    assert torch.equal(unpack_allow(words, n), torch.from_numpy(mask))


def test_pack_allow_sign_bit_and_packed_input():
    mask = np.zeros(64, bool)
    mask[31] = mask[63] = True
    w = pack_allow(torch.from_numpy(mask), 64)
    assert w.numpy().view(np.uint32).tolist() == [1 << 31, 1 << 31]
    assert pack_allow(w, 64) is not None and torch.equal(pack_allow(w, 64), w)
    assert torch.equal(pack_allow(w.numpy().view(np.uint32), 64), w), "uint32 ndarray words"


def test_pack_allow_errors():
    with pytest.raises(ValueError, match="entries"):
        pack_allow(np.ones(10, bool), 11)
    with pytest.raises(ValueError, match="packed words"):
        pack_allow(torch.zeros(1, dtype=torch.int32), 33)
    with pytest.raises(ValueError, match="bool"):
        pack_allow(np.ones(10, np.float32), 10)
    with pytest.raises(ValueError, match="one-dimensional"):
        pack_allow(np.ones((2, 5), bool), 10)
    with pytest.raises(TypeError):
        pack_allow([True, False], 2)


def test_local_allow_slices_global_ids():
    rng = np.random.default_rng(1)
    g = rng.random(200) < 0.5
    assert torch.equal(local_allow(g, 70, 50), torch.from_numpy(g[70:120]))
    assert torch.equal(local_allow(pack_allow(g, 200), 70, 50), torch.from_numpy(g[70:120]))
    assert local_allow(None, 0, 10) is None
    with pytest.raises(ValueError, match="covers"):
        local_allow(g, 190, 20)


def test_exclusion_csr_from_lists_and_pairs():
    off, ids = exclusion_csr([[5, 3], [], [7, 7, 1 << 40]], 3)
    assert off.tolist() == [0, 2, 2, 5] and ids.tolist() == [5, 3, 7, 7, 1 << 40]
    assert off.dtype == ids.dtype == torch.int64
    off2, ids2 = exclusion_csr((np.array([0, 1, 1], np.int32), torch.tensor([9])), 2)
    assert off2.tolist() == [0, 1, 1] and ids2.tolist() == [9] and off2.dtype == torch.int64
    off3, ids3 = exclusion_csr([[], []], 2)
    assert off3.tolist() == [0, 0, 0] and ids3.numel() == 0


def test_exclusion_csr_errors():
    with pytest.raises(ValueError, match="2 id lists for 3 queries"):
        exclusion_csr([[1], [2]], 3)
    with pytest.raises(ValueError, match=r"\[nq \+ 1\]"):
        exclusion_csr((torch.tensor([0, 1]), torch.tensor([1])), 2)
    with pytest.raises(ValueError, match="integer"):
        exclusion_csr((torch.tensor([0.0, 1.0]), torch.tensor([1])), 1)
    with pytest.raises(ValueError, match=r"\(offsets, ids\)"):
        exclusion_csr((torch.tensor([0, 1]),), 1)


def test_doc_filter_maps_doc_ids():
    lookup = ["d0", "d1", "d2", "d3", "d4"]
    allow, excl = doc_filter(lookup, ["q1", "q2", "q3"], allowed_docs=["d1", "d4", "unknown"],
                             exclude={"q1": ["d0", "nope", "d3"], "q3": ["d2"]})
    assert allow.tolist() == [False, True, False, False, True]
    assert excl == [[0, 3], [], [2]]
    assert doc_filter(lookup, ["q1"]) == (None, None)
    allow, excl = doc_filter(lookup, ["q1"], exclude={"q1": ["d4"]}, id_offset=100)
    assert allow is None and excl == [[104]]
    allow, excl = doc_filter(lookup, ["q1"], allowed_docs=[])
    assert allow.tolist() == [False] * 5 and excl is None


def test_doc_filter_per_shard():
    """Every rank of a sharded retriever maps the same arguments on its own lookup: its slice of the bitmap and the
    global ids of its own excluded documents."""
    shards = [["a", "b"], ["c", "d", "e"]]
    offsets = [0, 2]
    args = dict(allowed_docs=["b", "e"], exclude={"q": ["a", "d"]})
    got = [doc_filter(s, ["q"], id_offset=o, **args) for s, o in zip(shards, offsets)]
    assert got[0][0].tolist() == [False, True] and got[0][1] == [[0]]
    assert got[1][0].tolist() == [False, False, True] and got[1][1] == [[3]]
