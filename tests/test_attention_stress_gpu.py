"""GPU: every attention kernel (attn_kernel and attn_stream_kernel, each at head width 64 and 32) at the
adversarial attention statistics of tests/attention_stress.py, judged sequence by sequence against the float64 oracle.

Each sequence's reps and attended hidden rows, and the aggregate over the call, are held to the rule of _judge in
tests/test_encoder_numerics_gpu.py (rel-L2 <= 1e-2 and cosine >= 0.9999 where autocast itself stays within 5.3e-3, and
err_kernel <= 2 err_autocast + 2e-4 for the call, 3 err_autocast + 2e-4 for one sequence).  Judged per sequence, one wrong short sequence is not diluted by the others of
its batch.  tests/test_attention_stress_cpu.py shows on the oracle that the mistakes each case targets (a neighbour's
key leaked across a sequence boundary, a masked or padding key kept, the partial last key tile dropped, the two heads
of a 32-wide unit swapped) move the judged sequence by >= 8x its bound.  Each case prints one "[numerics]" line with
its worst per-output err_kernel / err_autocast, and the premise it relies on."""
import numpy as np
import pytest
import torch

import attention_stress as st
import oracle
import roberta_oracle as ro
from test_encoder_gpu import _rand_bert_sd, _rand_t5_sd
from test_encoder_numerics_gpu import _t5_rel_pattern, _t5_spec

pytestmark = pytest.mark.gpu

H = 128  # the magnet and tile-level cases: 2 heads of 64 or 4 heads of 32


@pytest.fixture(scope="module")
def enc_mod():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from openmatch_b200 import encoder
    return encoder


def _oracle(arch, sd, spec, ids, mask, pooling, emulate, probe=None):
    if arch == "roberta":
        return ro.encode_reps(sd, st.ospec(spec, pooling), ids, mask, dtype=st.F64, emulate_bf16=emulate)
    return oracle.encode_reps(sd, st.ospec(spec, pooling), ids, mask, dtype=st.F64, emulate_bf16=emulate, probe=probe)


def _packed(enc_mod, what, spec, sd, seqs, pooling="first", max_batch_tokens=16384, premise=None):
    """encode_packed the sequences and judge each one (one oracle call per sequence); premise(i, seq, logits) is
    called with the float64 oracle's layer-0 logits of every sequence (BERT / T5)"""
    enc = enc_mod.CudaEncoder(spec, sd, pooling=pooling, max_batch_tokens=max_batch_tokens)
    lens = np.array([len(s) for s in seqs], dtype=np.int32)
    got_h, got = enc.encode_packed(torch.cat(seqs).cuda(), lens, return_hidden=True)
    got_h, got = got_h.cpu().numpy(), got.cpu().numpy()
    offs = np.cumsum([0] + list(lens))
    items, want, auto, wh, ah = [], [], [], [], []
    for i, s in enumerate(seqs):
        probe = st.Logits() if premise is not None else None
        ones = torch.ones(1, len(s), dtype=torch.long)
        h0, r0 = _oracle(spec["arch"], sd, spec, s[None], ones, pooling, False, probe)
        h1, r1 = _oracle(spec["arch"], sd, spec, s[None], ones, pooling, True)
        if premise is not None:
            premise(i, s, probe.by_layer[0])
        want.append(r0[0].numpy())
        auto.append(r1[0].numpy())
        wh.append(h0[0].numpy())
        ah.append(h1[0].numpy())
        items.append(("#%d L=%d reps" % (i, len(s)), got[i:i + 1], want[-1][None], auto[-1][None]))
        items.append(("#%d L=%d hidden" % (i, len(s)), got_h[offs[i]:offs[i + 1]], wh[-1], ah[-1]))
    items.append(("all reps", got, np.stack(want), np.stack(auto)))
    items.append(("all hidden", got_h, np.concatenate(wh), np.concatenate(ah)))
    st.judge_each(what, items)
    return got_h, (wh, ah)


def _padded(enc_mod, what, spec, sd, ids, mask, pooling="first", probe=None):
    """om_encode of a padded batch, every sequence judged on its attended rows"""
    enc = enc_mod.CudaEncoder(spec, sd, pooling=pooling, max_batch_tokens=ids.numel())
    hidden, reps = enc.encode(ids.cuda(), mask.cuda(), return_hidden=True)
    hidden, reps = hidden.cpu().numpy(), reps.cpu().numpy()
    oh, orp = _oracle(spec["arch"], sd, spec, ids, mask, pooling, False, probe)
    ah, arp = _oracle(spec["arch"], sd, spec, ids, mask, pooling, True)
    oh, orp, ah, arp = oh.numpy(), orp.numpy(), ah.numpy(), arp.numpy()
    m = mask.numpy().astype(bool)
    items = []
    for b in range(ids.shape[0]):
        items.append(("#%d reps" % b, reps[b:b + 1], orp[b:b + 1], arp[b:b + 1]))
        items.append(("#%d hidden" % b, hidden[b][m[b]], oh[b][m[b]], ah[b][m[b]]))
    items.append(("all reps", reps, orp, arp))
    items.append(("all hidden", hidden[m], oh[m], ah[m]))
    st.judge_each(what, items)
    return hidden, (oh, ah)


def _magnet_premise(what, s, ids, allowed=None):
    m_even, m_odd, p_even = st.magnet_margins(s, ids, allowed)
    print("[numerics] premise %s: magnet margin even heads %.1f, odd heads %.1f nats (>= 30), P(magnet) >= %.4f"
          % (what, m_even, m_odd, p_even))
    assert m_even >= 30 and m_odd >= 30 and p_even >= 0.999, "premise: magnet margins"


def _magnet_model(dh, seed, arch="bert", layers=1):
    gen = torch.Generator().manual_seed(seed)
    heads = H // dh
    max_pos = 8194 if arch == "roberta" else 8192
    sd = st.magnet_model(_rand_bert_sd(gen, layers, H, 256, 1000, max_pos), heads, dh)
    if arch == "roberta":
        sd["embeddings.token_type_embeddings.weight"] = sd["embeddings.token_type_embeddings.weight"][:1]
    return gen, st.bert_spec(layers, H, heads, max_pos=max_pos, arch=arch), sd


# ------------------------------------------------------------------------------------------------------------------
# token magnets
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("L", [17, 32, 33, 64, 256, 512])
@pytest.mark.parametrize("dh", [64, 32])
def test_magnets_padded(enc_mod, dh, L):
    # multi-sequence tiles (L <= 64): sequences without a magnet sit between neighbours whose first and last tokens are
    # magnets; other rows hide magnets behind the mask (holes and a masked tail; at L >= 256 all of key tile 0)
    gen, spec, sd = _magnet_model(dh, 3000 + dh + L)
    ids, mask, _ = st.magnet_padded_batch(gen, L, max(8, 2 * (128 // L)))
    probe = st.Logits()
    _padded(enc_mod, "magnets padded dh=%d L=%d" % (dh, L), spec, sd, ids, mask, pooling="mean", probe=probe)
    allowed = mask.bool()[:, None, :].expand(-1, L, -1)
    _magnet_premise("L=%d" % L, probe.by_layer[0], ids, allowed)


# (length, magnets) of one packed call: a 4097-token sequence without a magnet (its last tile holds one key and 127
# padding rows) and a 513-token one with magnets at its ends; 129 - 512-token sequences (all attn_stream_kernel); bins whose sequences alternate with and without boundary magnets: [127 ends, 1 none],
# [60 ends, 40 none, 23 ends, 5 none], [2 none, 1 ends] (first-fit decreasing), [128 none] first after the long units
PACKED = [(4097, "none"), (513, "ends"), (511, "none"), (129, "ends"), (512, "none"), (60, "ends"), (128, "none"),
          (40, "none"), (127, "ends"), (23, "ends"), (1, "none"), (5, "none"), (2, "none"), (1, "ends"),
          (300, "inside")]


@pytest.mark.parametrize("layout", ["one_group", "cut"])
@pytest.mark.parametrize("dh", [64, 32])
def test_magnets_packed(enc_mod, dh, layout):
    # "cut": without the 4097-token sequence and max_batch_tokens 700, so the call is cut into row groups between the
    # the long units and the bins
    gen, spec, sd = _magnet_model(dh, 3100 + dh)
    cases = PACKED if layout == "one_group" else PACKED[1:]
    seqs = [st.with_magnets(gen, n, where) for n, where in cases]

    def premise(i, s, logits):
        if (s == st.MAGNET).any() and len(s) > 1:
            _magnet_premise("#%d L=%d" % (i, len(s)), logits, s[None])

    _packed(enc_mod, "magnets packed dh=%d %s" % (dh, layout), spec, sd, seqs,
            max_batch_tokens=16384 if layout == "one_group" else 700, premise=premise)


@pytest.mark.parametrize("dh", [64, 32])
def test_magnets_roberta_packed(enc_mod, dh):
    # RoBERTa's position ids skip its pad id 1: a few of them inside the content; <s> (id 0) is an ordinary token here
    gen, spec, sd = _magnet_model(dh, 3200 + dh, arch="roberta")
    sd["embeddings.word_embeddings.weight"][0, 0] = -st.A
    seqs = []
    for n, where in PACKED[1:]:
        s = st.with_magnets(gen, n, where)
        if n > 4:
            s[torch.randint(1, n - 1, (max(1, n // 50),), generator=gen)] = 1
        seqs.append(s)
    _packed(enc_mod, "magnets roberta packed dh=%d" % dh, spec, sd, seqs)


# ------------------------------------------------------------------------------------------------------------------
# online softmax across key tiles: the favoured key tile by position, polarity alternating by head
# ------------------------------------------------------------------------------------------------------------------
def _tile_model(dh, seed, level, early):
    gen = torch.Generator().manual_seed(seed)
    heads = H // dh
    sd = st.tile_level_model(_rand_bert_sd(gen, 1, H, 256, 1000, 8192), heads, dh, level, early)
    return gen, st.bert_spec(1, H, heads), sd


def _gap_premise(what, s, L, early, rows=None):
    g_even, g_odd = st.tile_gaps(s, L, early, rows)
    need = 30.0 if early else 20.0
    print("[numerics] premise %s: tile gap even heads %.1f, odd heads %.1f nats (>= %.0f)" % (what, g_even, g_odd,
                                                                                          need))
    assert g_even >= need and g_odd >= need, "premise: tile gap"


@pytest.mark.parametrize("layout", ["padded", "packed"])
@pytest.mark.parametrize("where", ["tile0", "last_tile"])
@pytest.mark.parametrize("L", [256, 512])
@pytest.mark.parametrize("dh", [64, 32])
def test_tile_maxima_long(enc_mod, dh, L, where, layout):
    early = where == "tile0"
    gen, spec, sd = _tile_model(dh, 3300 + dh + L + early, st.tile_level(L, where), early)
    what = "tile maxima %s dh=%d L=%d %s" % (layout, dh, L, where)
    if layout == "padded":
        ids = st.plain(gen, 3 * L).view(3, L)
        mask = torch.ones(3, L, dtype=torch.long)
        mask[1, 3:40] = 0  # holes inside key tile 0
        probe = st.Logits()
        _padded(enc_mod, what, spec, sd, ids, mask, pooling="mean", probe=probe)
        s = probe.by_layer[0][[0, 2]]
    else:
        seqs = [st.plain(gen, n) for n in (L, 77, L, 5)]
        gaps = []
        _packed(enc_mod, what, spec, sd, seqs, premise=lambda i, q, lg: gaps.append(lg) if len(q) == L else None)
        s = torch.cat(gaps)
    _gap_premise("L=%d" % L, s, L, early)


@pytest.mark.parametrize("dh,L,where", [(64, 2049, "last_key"), (64, 4097, "last_key"), (32, 2049, "last_key"),
                                        (32, 4097, "last_key"), (32, 8192, "tile0"), (32, 8192, "last_tile"),
                                        (32, 8192, "moving")])
def test_tile_maxima_stream(enc_mod, dh, L, where):
    # last_key: at L = 128 k + 1 the partial last key tile holds one key (the favoured one) and 127 padding rows
    early = where == "tile0"
    gen, spec, sd = _tile_model(dh, 3400 + dh + L + len(where), st.tile_level(L, where), early)
    seqs = [st.plain(gen, n) for n in (L, 300, 40)]
    got = []
    _packed(enc_mod, "tile maxima stream dh=%d L=%d %s" % (dh, L, where), spec, sd, seqs,
            premise=lambda i, q, lg: got.append(lg) if i == 0 else None)
    s = got[0]
    if where != "moving":
        _gap_premise("L=%d" % L, s, L, early)
        return
    tmax = s[:, 0::2].reshape(1, -1, L, L // 128, 128).amax(-1)  # even heads: the maximum rises tile by tile
    raised = (tmax[..., 1:] > torch.cummax(tmax, -1).values[..., :-1]).double().mean(-1)
    spread = float((tmax[..., -1] - tmax[..., 0]).min())
    print("[numerics] premise: running maximum raised at >= %.3f of the tile steps, last - first tile maximum "
          ">= %.1f nats" % (float(raised.min()), spread))
    assert float(raised.min()) >= 0.4 and spread >= 25.0


# ------------------------------------------------------------------------------------------------------------------
# peaked rows, isolated tokens, non-prefix masks (hidden 768: 12 heads of 64 or 24 of 32)
# ------------------------------------------------------------------------------------------------------------------
def _peak_premise(what, s, L, level, rows=None):
    _, lo, hi = st.PEAK[level][L]
    med = st.row_pmax_median(s, rows)
    print("[numerics] premise %s: median row-max probability %.3f in [%.2f, %.2f]" % (what, med, lo, hi))
    assert lo <= med <= hi, "premise: median row-max probability"


@pytest.mark.parametrize("level", ["flat", "half", "sharp"])
@pytest.mark.parametrize("L,B", [(17, 40), (128, 6), (512, 2)])
def test_peaked_padded_hd32(enc_mod, L, B, level):
    gen = torch.Generator().manual_seed(3500 + L)
    spec = st.bert_spec(2, 768, 24, F=1536, vocab=2000, max_pos=512)
    sd = st.scale_query(_rand_bert_sd(gen, 2, 768, 1536, 2000, 512), 2, st.PEAK[level][L][0])
    ids = torch.randint(10, 2000, (B, L), generator=gen)
    mask = torch.ones(B, L, dtype=torch.long)
    mask[-1, L // 2:] = 0
    probe = st.Logits()
    _padded(enc_mod, "peaked dh=32 %s L=%d" % (level, L), spec, sd, ids, mask, probe=probe)
    _peak_premise("L=%d" % L, probe.by_layer[0], L, level, mask.bool() & mask.bool().all(1, keepdim=True))


@pytest.mark.parametrize("level", ["flat", "half", "sharp"])
@pytest.mark.parametrize("dh", [64, 32])
def test_peaked_packed(enc_mod, dh, level):
    # ~1000 and ~3000 tokens (attn_stream_kernel) next to a bin; one query scale per call, that of 1000 tokens
    gen = torch.Generator().manual_seed(3600 + dh)
    spec = st.bert_spec(2, 768, 768 // dh, F=1536, vocab=2000)
    sd = st.scale_query(_rand_bert_sd(gen, 2, 768, 1536, 2000, 8192), 2, st.PEAK[level][1000][0])
    seqs = [st.plain(gen, n, 2000) for n in (1000, 77, 3000)]

    def premise(i, s, logits):
        if len(s) == 1000:
            _peak_premise("L=1000", logits, 1000, level)

    _packed(enc_mod, "peaked packed dh=%d %s" % (dh, level), spec, sd, seqs, premise=premise)


def _per_token(what, got, ref, auto):
    ek = np.linalg.norm(got - ref, axis=1) / np.linalg.norm(ref, axis=1)
    ea = np.linalg.norm(auto - ref, axis=1) / np.linalg.norm(ref, axis=1)
    worst = int(np.argmax(ek - st.C * ea))
    print("[numerics] %s per token: max err_kernel %.3e  max err_autocast %.3e  worst token %.3e vs %.3e"
          % (what, ek.max(), ea.max(), ek[worst], ea[worst]))
    assert ek.max() <= st.C * ea.max() + st.FLOOR
    assert (ek <= st.C * ea + 5 * st.FLOOR + 2 ** -8).all(), "token %d: %.3e vs %.3e" % (worst, ek[worst], ea[worst])


def _isolated_model(dh, seed):
    gen = torch.Generator().manual_seed(seed)
    sd = st.isolate_layer(st.scale_query(_rand_bert_sd(gen, 1, 768, 256, 2000, 8192), 1, 30), 768)
    return gen, st.bert_spec(1, 768, 768 // dh, vocab=2000), sd


@pytest.mark.parametrize("L,B", [(64, 8), (128, 6), (512, 2)])
def test_isolated_per_token_padded_hd32(enc_mod, L, B):
    gen, spec, sd = _isolated_model(32, 3700 + L)
    ids = torch.randint(10, 2000, (B, L), generator=gen)
    mask = torch.ones(B, L, dtype=torch.long)
    for b in range(1, B):
        mask[b, int(torch.randint(1, L + 1, (1,), generator=gen)):] = 0
    probe = st.Logits()
    hidden, (oh, ah) = _padded(enc_mod, "isolated dh=32 L=%d" % L, spec, sd, ids, mask, probe=probe)
    med = st.row_pmax_median(probe.by_layer[0], mask.bool())
    print("[numerics] premise: median row-max probability %.3f >= 0.5" % med)
    assert med >= 0.5
    m = mask.numpy().astype(bool)
    _per_token("isolated dh=32 L=%d" % L, hidden[m], oh[m], ah[m])


@pytest.mark.parametrize("dh", [64, 32])
def test_isolated_per_token_packed(enc_mod, dh):
    gen, spec, sd = _isolated_model(dh, 3800 + dh)
    seqs = [st.plain(gen, n, 2000) for n in (1025, 64, 300, 17)]
    meds = []
    got_h, (wh, ah) = _packed(enc_mod, "isolated packed dh=%d" % dh, spec, sd, seqs,
                              premise=lambda i, s, lg: meds.append(st.row_pmax_median(lg)))
    print("[numerics] premise: median row-max probability >= %.3f (>= 0.5)" % min(meds))
    assert min(meds) >= 0.5
    _per_token("isolated packed dh=%d" % dh, got_h, np.concatenate(wh), np.concatenate(ah))


@pytest.mark.parametrize("case", ["left_pad_100", "holes_17", "holes_32", "single_token", "tile0_masked_256",
                                  "tile0_masked_512"])
def test_non_prefix_masks_hd32(enc_mod, case):
    gen = torch.Generator().manual_seed(3900 + len(case))
    L, B = {"left_pad_100": (100, 4), "holes_17": (17, 16), "holes_32": (32, 12), "single_token": (32, 6),
            "tile0_masked_256": (256, 2), "tile0_masked_512": (512, 2)}[case]
    spec = st.bert_spec(2, 768, 24, F=1536, vocab=2000, max_pos=512)
    sd = st.scale_query(_rand_bert_sd(gen, 2, 768, 1536, 2000, 512), 2, 15)
    ids = torch.randint(10, 2000, (B, L), generator=gen)
    mask = torch.ones(B, L, dtype=torch.long)
    if case == "left_pad_100":
        for b in range(1, B):
            mask[b, :7 * b] = 0
    elif case.startswith("holes"):
        for b in range(B):
            mask[b, torch.randperm(L, generator=gen)[:L // 3]] = 0
            mask[b, b % L] = 1
    elif case == "single_token":
        mask[:] = 0
        for b in range(B):
            mask[b, (5 * b) % L] = 1
    else:
        mask[:, :128] = 0
        mask[0, 128:150] = 0
    _padded(enc_mod, "mask dh=32 %s" % case, spec, sd, ids, mask, pooling="mean")


# ------------------------------------------------------------------------------------------------------------------
# T5 relative bias in the packed layout (indexed tile-locally), sequences in bins and behind other units
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pattern", ["far", "local"])
def test_t5_relative_bias_packed(enc_mod, pattern):
    gen = torch.Generator().manual_seed(4000 + len(pattern))
    spec = _t5_spec(2, 768, 12, 1536)
    sd = _t5_rel_pattern(_rand_t5_sd(gen, 2, 768, 12, 1536, 2000), 12, pattern)
    seqs = [st.plain(gen, n, 2000) for n in (300, 40, 512, 129, 17, 128, 3, 200, 70)]
    spreads = []

    def premise(i, s, logits):
        # local: every row of 17+ tokens spans >= 20 nats; far: the rows with a key >= 91 positions ahead do
        L = len(s)
        if pattern == "local" and L >= 17:
            spreads.append(float((logits.amax(-1) - logits.amin(-1)).min()))
        elif pattern == "far" and L >= 129:
            spreads.append(float((logits.amax(-1) - logits.amin(-1))[..., :L - 91].min()))

    _packed(enc_mod, "t5 packed %s" % pattern, spec, sd, seqs, pooling="mean", premise=premise)
    print("[numerics] premise: min logit spread of a row %.1f nats (>= 20)" % min(spreads))
    assert min(spreads) >= 20


# ------------------------------------------------------------------------------------------------------------------
# 32-wide heads: bitwise determinism and batch invariance
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("L", [128, 256])
def test_bitwise_determinism_and_batch_invariance_hd32(enc_mod, L):
    gen = torch.Generator().manual_seed(4100 + L)
    spec = st.bert_spec(2, 768, 24, F=1536, vocab=2000, max_pos=512)
    sd = st.scale_query(_rand_bert_sd(gen, 2, 768, 1536, 2000, 512), 2, 15)
    enc = enc_mod.CudaEncoder(spec, sd, pooling="mean", max_batch_tokens=40 * L)
    ids = torch.randint(10, 2000, (40, L), generator=gen)
    mask = torch.ones(40, L, dtype=torch.long)
    for b in range(1, 40):
        mask[b, int(torch.randint(2, L + 1, (1,), generator=gen)):] = 0
    ids, mask = ids.cuda(), mask.cuda()
    h1, r1 = enc.encode(ids, mask, return_hidden=True)
    h1, r1 = h1.clone(), r1.clone()
    h2, r2 = enc.encode(ids, mask, return_hidden=True)
    assert torch.equal(h1, h2) and torch.equal(r1, r2), "run-to-run difference"
    for b in (0, 1, 17, 39):
        ha, ra = enc.encode(ids[b:b + 1], mask[b:b + 1], return_hidden=True)
        assert torch.equal(ra[0], r1[b]), "sequence %d alone differs from its row in the batch" % b
        assert torch.equal(ha[0], h1[b])
