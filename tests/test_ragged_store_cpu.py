"""CPU: the ragged pretokenised store (write_ragged_store + PretokenizedDataset) against the padded ``.npy`` store of the
same rows: round trip, truncation to max_len, and the rank interleaving and ids of iter_batches / __iter__."""
import numpy as np
import pytest

from openmatch_b200.arguments import DataArguments
from openmatch_b200.dataset import InferenceDataset, write_ragged_store


def _rows(seed, n, L):
    rng = np.random.default_rng(seed)
    ids = rng.integers(5, 1000, (n, L)).astype(np.int32)
    for r in range(n):
        ids[r, rng.integers(1, L + 1):] = 0
    return ids


def _stores(tmp_path, ids, names=True):
    np.save(tmp_path / "pad.npy", ids)
    ids_txt = ["doc%d" % i for i in range(ids.shape[0])]
    if names:
        (tmp_path / "pad.ids.txt").write_text("\n".join(ids_txt))
    ragged = write_ragged_store(str(tmp_path / "rag"), ids, ids_txt if names else None)
    return str(tmp_path / "pad.npy"), ragged


def test_round_trip(tmp_path):
    ids = _rows(1, 37, 50)
    _, ragged = _stores(tmp_path, ids)
    assert ragged == str(tmp_path / "rag.tokens.npy")
    tokens, offsets = np.load(tmp_path / "rag.tokens.npy"), np.load(tmp_path / "rag.offsets.npy")
    assert tokens.dtype == np.int32 and offsets.dtype == np.int64 and offsets.shape == (38,) and offsets[0] == 0
    for i in range(37):
        row = ids[i][ids[i] != 0]
        np.testing.assert_array_equal(tokens[offsets[i]:offsets[i + 1]], row)
    ds = InferenceDataset.load(None, DataArguments(corpus_path=ragged, p_max_len=64), batch_size=8)
    assert ds.is_ragged and ds.num_local_rows() == 37
    (names, toks, lens), = [b for b in ds.iter_batches()][:1]
    assert names == ["doc%d" % i for i in range(8)]
    np.testing.assert_array_equal(lens, (ids[:8] != 0).sum(1))
    np.testing.assert_array_equal(toks, ids[:8][ids[:8] != 0])
    with pytest.raises(ValueError, match="no token"):
        write_ragged_store(str(tmp_path / "bad"), np.zeros((2, 4), dtype=np.int32))


@pytest.mark.parametrize("max_len", [16, 50, 64])
def test_truncation_like_padded_store(tmp_path, max_len):
    ids = _rows(2, 29, 50)
    padded, ragged = _stores(tmp_path, ids)
    pad = InferenceDataset.load(None, DataArguments(corpus_path=padded, p_max_len=max_len), batch_size=7)
    rag = InferenceDataset.load(None, DataArguments(corpus_path=ragged, p_max_len=max_len), batch_size=7)
    assert not pad.is_ragged
    for (pn, block), (rn, toks, lens) in zip(pad.iter_batches(), rag.iter_batches()):
        assert pn == rn and lens.dtype == np.int32
        keep = block != 0
        np.testing.assert_array_equal(lens, keep.sum(1))
        np.testing.assert_array_equal(toks, block[keep])
    # the per-example path (DataLoader + collator) yields the same padded examples from both stores
    assert list(pad) == list(rag)


@pytest.mark.parametrize("world,names", [(1, True), (3, True), (4, False)])
def test_rank_interleaving(tmp_path, world, names):
    ids = _rows(3, 50, 20)
    padded, ragged = _stores(tmp_path, ids, names)
    for r in range(world):
        kw = dict(batch_size=6, num_processes=world, process_index=r)
        pad = InferenceDataset.load(None, DataArguments(corpus_path=padded, p_max_len=20), **kw)
        rag = InferenceDataset.load(None, DataArguments(corpus_path=ragged, p_max_len=20), **kw)
        assert pad.num_local_rows() == rag.num_local_rows()
        pb, rb = list(pad.iter_batches()), list(rag.iter_batches())
        assert [b[0] for b in pb] == [b[0] for b in rb]
        assert sum(len(b[2]) for b in rb) == rag.num_local_rows()
        assert [e["text_id"] for e in pad] == [e["text_id"] for e in rag]
