"""CPU: the constructions of tests/attention_stress.py on the float64 oracle.  For each one, the premise it claims (a
magnet's margin, a tile gap, a median row-max probability) holds, and the kernel mistakes it targets move a sequence's
hidden rows by at least NEED = 8x the bound tests/test_attention_stress_gpu.py holds that sequence to (C_SEQ *
err_autocast + FLOOR, err_autocast from the oracle with bf16 autocast emulated), which is >= 12x the whole-call bound
C * err_autocast + FLOOR.  The ratio of every other applicable fault model is
printed ("[stress]" lines, run with -s)."""
import pytest
import torch

import attention_stress as st
from test_encoder_gpu import _rand_bert_sd

H = 128
NEED = 8.0


def _model(dh, seed, layers=1):
    gen = torch.Generator().manual_seed(seed)
    heads = H // dh
    return gen, st.bert_spec(layers, H, heads), _rand_bert_sd(gen, layers, H, 256, 1000, 8192), heads


def _ratios(monkeypatch, what, sd, spec, ids, clean, faults, n_judged, targeted):
    """hidden rows [0, n_judged) of row 0 under each fault against the clean run: rel-L2 / (C_SEQ err_autocast + FLOOR);
    asserts >= NEED for the targeted faults"""
    h0 = st.oracle_hidden(monkeypatch, sd, spec, ids, clean)[0, :n_judged]
    ha = st.oracle_hidden(monkeypatch, sd, spec, ids, clean, emulate_bf16=True)[0, :n_judged]
    bound = st.C_SEQ * st.rel(ha, h0) + st.FLOOR
    out = {}
    for name, (allowed, swap) in faults.items():
        hf = st.oracle_hidden(monkeypatch, sd, spec, ids, allowed, swap_pairs=swap)[0, :n_judged]
        out[name] = st.rel(hf, h0) / bound
        print("[stress] %-34s fault %-18s error / bound %8.1f%s" % (what, name, out[name],
                                                                   "  (targeted)" if name in targeted else ""))
    for name in targeted:
        assert out[name] >= NEED, "%s: fault %s moves the output by only %.1fx the bound" % (what, name, out[name])
    return out


@pytest.mark.parametrize("dh", [64, 32])
def test_magnet_premise(dh):
    gen, spec, sd, heads = _model(dh, 100 + dh)
    st.magnet_model(sd, heads, dh)
    ids, mask, _ = st.magnet_padded_batch(gen, 33, 8)
    probe = st.Logits()
    import oracle
    oracle.encode_reps(sd, st.ospec(spec), ids, mask, dtype=st.F64, probe=probe)
    allowed = mask.bool()[:, None, :].expand(-1, 33, -1)
    m_even, m_odd, p_even = st.magnet_margins(probe.by_layer[0], ids, allowed)
    print("[stress] dh=%d magnet margins: even heads %.1f nats, odd heads %.1f nats, even P(magnet) >= %.6f"
          % (dh, m_even, m_odd, p_even))
    assert m_even >= 30 and m_odd >= 30 and p_even >= 0.999


@pytest.mark.parametrize("L", [17, 129, 513])
@pytest.mark.parametrize("dh", [64, 32])
def test_magnet_neighbour_leak(monkeypatch, dh, L):
    # a sequence without a magnet, followed by its neighbour's boundary token, a magnet (the next sequence's first
    # token at c_hi, or the previous one's last token at c_lo - 1: the same key content, placed after the sequence so
    # that its positions stay those it has alone)
    gen, spec, sd, heads = _model(dh, 200 + dh + L)
    st.magnet_model(sd, heads, dh)
    ids = torch.cat([st.with_magnets(gen, L, "none"), torch.tensor([st.MAGNET])])[None]
    clean = st.seq_allowed(L + 1, 0, L)
    faults = {"neighbour_key_leaked": (st.seq_allowed(L + 1, 0, L + 1), False),
              "heads_swapped": (clean, True)}
    _ratios(monkeypatch, "dh=%d L=%d no magnet" % (dh, L), sd, spec, ids, clean, faults, L, ["neighbour_key_leaked"])


@pytest.mark.parametrize("dh", [64, 32])
def test_magnet_masked_key_and_head_swap(monkeypatch, dh):
    gen, spec, sd, heads = _model(dh, 300 + dh)
    st.magnet_model(sd, heads, dh)
    ids, mask, kinds = st.magnet_padded_batch(gen, 33, 4)
    # a row whose masked keys are magnets: one of them kept
    b = kinds.index(2)
    valid = mask[b].bool()
    kept = valid.clone()
    kept[int((~valid).nonzero()[0])] = True
    clean = valid[None, None, :].expand(1, 33, 33)
    faults = {"masked_key_kept": (kept[None, None, :].expand(1, 33, 33), False), "heads_swapped": (clean, True)}
    _ratios(monkeypatch, "dh=%d L=33 masked magnets" % dh, sd, spec, ids[b:b + 1], clean, faults, 33,
                  ["masked_key_kept"])
    # a row with magnets at both ends: the heads of a unit swapped (at dh = 64 the pair spans two units: printed)
    b = kinds.index(1)
    full = st.seq_allowed(33, 0, 33)
    _ratios(monkeypatch, "dh=%d L=33 magnets at the ends" % dh, sd, spec, ids[b:b + 1], full,
            {"heads_swapped": (full, True)}, 33, ["heads_swapped"] if dh == 32 else [])


@pytest.mark.parametrize("dh", [64, 32])
def test_padding_keys_of_the_last_tile(monkeypatch, dh):
    # a 2049-token sequence without a magnet (attn_stream_kernel), followed by the 127 padding rows of its last tile at
    # the level of the packed layout's zeroed padding rows: keeping them is what the key bits of the previous ring slot
    # (all valid) do to the last tile
    gen, spec, sd, heads = _model(dh, 400 + dh)
    st.magnet_model(sd, heads, dh)
    L = 2049
    ids = torch.cat([st.with_magnets(gen, L, "none"), torch.full((127,), st.NEUTRAL)])[None]
    clean = st.seq_allowed(L + 127, 0, L)
    faults = {"ring_prev_key_bits": (st.seq_allowed(L + 127, 0, L + 127), False),
              "last_tile_dropped": (st.seq_allowed(L + 127, 0, 2048), False)}
    _ratios(monkeypatch, "dh=%d L=2049 padding keys" % dh, sd, spec, ids, clean, faults, L, ["ring_prev_key_bits"])


@pytest.mark.parametrize("where,L", [("tile0", 512), ("last_tile", 512), ("last_key", 2049)])
@pytest.mark.parametrize("dh", [64, 32])
def test_tile_maxima(monkeypatch, dh, where, L):
    gen, spec, sd, heads = _model(dh, 500 + dh + L)
    early = where == "tile0"
    st.tile_level_model(sd, heads, dh, st.tile_level(L, where), early)
    n = L + (127 if L % 128 else 0)  # with the padding rows of a partial last tile (level 0)
    ids = torch.cat([st.plain(gen, L), torch.full((n - L,), st.NEUTRAL)])[None]
    clean = st.seq_allowed(n, 0, L)
    probe = st.Logits()
    st.oracle_hidden(monkeypatch, sd, spec, ids[:, :L], st.seq_allowed(L, 0, L), probe=probe)
    g_even, g_odd = st.tile_gaps(probe.by_layer[0], L, early)
    need = 30.0 if early else 20.0
    print("[stress] dh=%d L=%d %s: tile gap even heads %.1f, odd heads %.1f nats (>= %.0f)" % (dh, L, where, g_even,
                                                                                            g_odd, need))
    assert g_even >= need and g_odd >= need
    faults = {"heads_swapped": (clean, True)}
    targeted = ["heads_swapped"] if dh == 32 else []
    if L % 128:
        faults["last_tile_dropped"] = (st.seq_allowed(n, 0, L // 128 * 128), False)
        faults["ring_prev_key_bits"] = (st.seq_allowed(n, 0, n), False)
        targeted.append("last_tile_dropped")
    _ratios(monkeypatch, "dh=%d L=%d max %s" % (dh, L, where), sd, spec, ids, clean, faults, L, targeted)


@pytest.mark.parametrize("L", [17, 128, 512, 1000, 3000])
@pytest.mark.parametrize("dh", [64, 32])
def test_peaked_premise(dh, L):
    # hidden 768 as the suite's peaked cases; the logit statistics do not depend on the head width (q.k over dh dims,
    # scaled by dh^-1/2), so the same query scales give the same levels at dh = 32
    import oracle
    gen = torch.Generator().manual_seed(600 + L)
    sd = _rand_bert_sd(gen, 1, 768, 256, 1000, 8192)
    spec = st.bert_spec(1, 768, 768 // dh)
    ids = st.plain(gen, L)[None]
    for level in ("flat", "half", "sharp"):
        alpha, lo, hi = st.PEAK[level][L]
        probe = st.Logits()
        oracle.encode_reps(st.scale_query(sd, 1, alpha), st.ospec(spec), ids, torch.ones_like(ids), dtype=st.F64,
                           probe=probe)
        med = st.row_pmax_median(probe.by_layer[0])
        print("[stress] dh=%d L=%d %s: median row-max probability %.3f in [%.2f, %.2f]" % (dh, L, level, med, lo, hi))
        assert lo <= med <= hi


@pytest.mark.parametrize("dh", [64, 32])
def test_isolated_premise_and_head_swap(monkeypatch, dh):
    gen = torch.Generator().manual_seed(700 + dh)
    heads = 768 // dh
    sd = st.isolate_layer(st.scale_query(_rand_bert_sd(gen, 1, 768, 256, 1000, 8192), 1, 30), 768)
    spec = st.bert_spec(1, 768, heads)
    for L in (64, 1025):
        ids = st.plain(gen, L)[None]
        probe = st.Logits()
        full = st.seq_allowed(L, 0, L)
        st.oracle_hidden(monkeypatch, sd, spec, ids, full, probe=probe)
        med = st.row_pmax_median(probe.by_layer[0])
        print("[stress] dh=%d isolated L=%d: median row-max probability %.3f >= 0.5" % (dh, L, med))
        assert med >= 0.5
        _ratios(monkeypatch, "dh=%d isolated L=%d" % (dh, L), sd, spec, ids, full, {"heads_swapped": (full, True)}, L,
                ["heads_swapped"] if dh == 32 else [])
