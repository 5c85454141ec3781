"""GPU numerics of the CUDA encoder against a float64 oracle, at the activation statistics where bf16 kernels go wrong:
peaked and saturated attention rows, online-softmax rescales across key tiles, large residual offsets, odd shapes and
non-prefix masks, plus bitwise determinism and batch invariance.

Every case compares the kernel's reps and attended last_hidden_state with ``oracle.encode_reps(dtype=float64)`` and
asserts two bounds:
  * the fixed bound of tests/test_encoder_gpu.py (SURVEY 8c): rel-L2 <= 1e-2 and per-row cosine >= 0.9999;
  * the error model  err_kernel <= C * err_autocast + FLOOR,  where err_autocast is the rel-L2 of the same oracle with
    bf16 autocast emulated (``emulate_bf16=True``: bf16 matmul operands, Linear outputs and P).
C and FLOOR come from counting rounding sites, not from fitting.  The kernel rounds to bf16 where autocast does (matmul
operands, Linear outputs, P) and in a few more places: the folded weights W diag(gamma) (one more rounding of W), the
un-normalised residual s instead of LN(s), the QKV / FFN1 outputs after the fused bias + activation.  That is at most
twice as many independent relative-2^-9 roundings per layer, and independent errors add in quadrature: sqrt(2) ~ 1.4,
so C = 2 leaves headroom for the correlated part.  The kernel's own approximations (ex2.approx, the rational erf with
|err| 2e-5, fp32 accumulation in another order) stay near 1e-5 relative; FLOOR = 2e-4 covers them.
A probe on the oracle's attention logits asserts, for each stress case, that the stress is really present.
Each case prints one "[numerics]" line (err_kernel, err_autocast, their ratio); run with -s to see them."""
import numpy as np
import pytest
import torch

import oracle
from oracle.encoder import EncoderSpec
from test_encoder_gpu import _check, _ids, _rand_bert_sd, _rand_t5_sd

pytestmark = pytest.mark.gpu

C, FLOOR = 2.0, 2e-4
AUTOCAST_ANCHOR = 5.3e-3
F64 = torch.float64


@pytest.fixture(scope="module")
def enc_mod():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from openmatch_b200 import encoder
    return encoder


def _rel(got, want):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    return float(np.linalg.norm(got - want) / max(np.linalg.norm(want), 1e-30))


def _judge(what, got, ref, auto, fixed=True):
    """Fixed bound and the error model for one output; returns (err_kernel, err_autocast).  The fixed bound is anchored
    on the reference's own autocast drift (5.3e-3, SURVEY 8c); where autocast itself drifts further from float64
    (saturated attention rows: logits of +-50 carry bf16 errors of 0.1 nats) only the error model applies."""
    got, ref, auto = (np.asarray(x, np.float64).reshape(-1, np.shape(x)[-1]) for x in (got, ref, auto))
    assert np.isfinite(got).all(), what + ": non-finite output"
    ek, ea = _rel(got, ref), _rel(auto, ref)
    print("[numerics] %-44s err_kernel %.3e  err_autocast %.3e  ratio %.2f" % (what, ek, ea, ek / max(ea, 1e-30)))
    if fixed and ea <= AUTOCAST_ANCHOR:
        _check(got, ref, what)
    assert ek <= C * ea + FLOOR, "%s: err_kernel %.3e > %.1f * err_autocast %.3e + %.0e" % (what, ek, C, ea, FLOOR)
    return ek, ea


def _bert_spec(layers, H, heads, F, vocab=2000, max_pos=512):
    return dict(arch="bert", layers=layers, hidden=H, heads=heads, ffn=F, vocab=vocab, max_pos=max_pos, type_vocab=2,
                ln_eps=1e-12)


def _t5_spec(layers, H, heads, F, vocab=2000):
    return dict(arch="t5", layers=layers, hidden=H, heads=heads, ffn=F, vocab=vocab, ln_eps=1e-6, rel_buckets=32,
                rel_max_distance=128)


def _ospec(spec, pooling="first", normalize=False):
    return EncoderSpec(spec["arch"], spec["layers"], spec["hidden"], spec["heads"], spec["ffn"], spec["ln_eps"],
                       pooling=pooling, normalize=normalize)


def _compare(enc_mod, what, spec, sd, ids, mask, tt=None, head=None, pooling="first", normalize=False, probe=None,
             fixed=True, enc=None, shift=None):
    """Encode on the GPU and judge reps and attended hidden rows against the float64 oracle.  shift [H] (no head,
    no normalisation) is subtracted from every output first, so that a constant offset does not mask the errors."""
    if enc is None:
        enc = enc_mod.CudaEncoder(spec, sd, head_weight=head, pooling=pooling, normalize=normalize,
                                  max_batch_tokens=ids.numel())
    hidden, reps = enc.encode(ids.cuda(), mask.cuda(), tt.cuda() if tt is not None else None, return_hidden=True)
    ospec = _ospec(spec, pooling, normalize)
    oh, oreps = oracle.encode_reps(sd, ospec, ids, mask, tt, head, dtype=F64, probe=probe)
    ah, areps = oracle.encode_reps(sd, ospec, ids, mask, tt, head, dtype=F64, emulate_bf16=True)
    if shift is not None:
        hidden, reps, oh, oreps, ah, areps = (x - shift.to(x) for x in (hidden, reps, oh, oreps, ah, areps))
    m = mask.numpy().astype(bool)
    out = {"reps": _judge(what + " reps", reps.cpu().numpy(), oreps.numpy(), areps.numpy(), fixed),
           "hidden": _judge(what + " hidden", hidden.cpu().numpy()[m], oh.numpy()[m], ah.numpy()[m], fixed)}
    return out, (hidden.cpu().numpy(), reps.cpu().numpy()), (oh.numpy(), ah.numpy())


class _Logits:
    """Probe: keeps each layer's masked attention logits (float64, natural-log units)."""

    def __init__(self):
        self.by_layer = {}

    def __call__(self, layer, s):
        self.by_layer[layer] = s

    def row_pmax(self, layer, rows):
        """largest softmax probability of every (sequence, head, query) row selected by the bool mask rows [B, L]"""
        p = torch.softmax(self.by_layer[layer], -1).amax(-1)  # [B, heads, L]
        return p[rows[:, None, :].expand_as(p)]


def _scale_query(sd, layers, alpha):
    sd = dict(sd)
    for i in range(layers):
        for n in ("weight", "bias"):
            k = f"encoder.layer.{i}.attention.self.query.{n}"
            sd[k] = sd[k] * alpha
    return sd


# ------------------------------------------------------------------------------------------------------------------
# peaked attention: the query weights scaled so the typical row-max probability is flat / ~0.5 / >= 0.95
# ------------------------------------------------------------------------------------------------------------------
# (alpha, lo, hi) of the median row-max probability; the flat level is the suite's usual weights (std 0.02)
_PEAK = {"flat": {17: (1, 0, 0.15), 128: (1, 0, 0.05), 512: (1, 0, 0.02)},
         "half": {17: (9, 0.3, 0.7), 128: (15, 0.3, 0.7), 512: (20, 0.3, 0.7)},
         "sharp": {17: (40, 0.95, 1), 128: (64, 0.95, 1), 512: (80, 0.95, 1)}}


@pytest.mark.parametrize("level", ["flat", "half", "sharp"])
@pytest.mark.parametrize("L,B", [(17, 40), (128, 6), (512, 2)])
def test_peaked_attention(enc_mod, L, B, level):
    alpha, lo, hi = _PEAK[level][L]
    gen = torch.Generator().manual_seed(1000 + L)
    layers, H, F = 2, 768, 1536
    spec = _bert_spec(layers, H, 12, F)
    sd = _scale_query(_rand_bert_sd(gen, layers, H, F, 2000, 512), layers, alpha)
    ids, mask = _ids(gen, B, L, 2000, ragged=False)
    mask[-1, L // 2:] = 0  # one padded sequence (its rows are not part of the premise)
    full = mask.bool() & mask.bool().all(1, keepdim=True)
    probe = _Logits()
    _compare(enc_mod, "peaked %s L=%d" % (level, L), spec, sd, ids, mask, probe=probe)
    med = float(probe.row_pmax(0, full).median())
    print("[numerics] premise: median row-max probability %.3f in [%.2f, %.2f]" % (med, lo, hi))
    assert lo <= med <= hi, "premise: median row-max probability %.3f not in [%.2f, %.2f]" % (med, lo, hi)


@pytest.mark.parametrize("L,B", [(64, 8), (128, 6), (512, 2)])
def test_attention_isolated_per_token(enc_mod, L, B):
    # one layer whose FFN is zero and whose O-proj is the identity: the output is LN2(LN1(s0 + ctx)), so an attention
    # error reaches every token undiluted; checked token by token
    gen = torch.Generator().manual_seed(1100 + L)
    H, F = 768, 256
    spec = _bert_spec(1, H, 12, F)
    sd = _scale_query(_rand_bert_sd(gen, 1, H, F, 2000, 512), 1, 30)
    p = "encoder.layer.0."
    for n in ("intermediate.dense", "output.dense"):
        sd[p + n + ".weight"].zero_()
        sd[p + n + ".bias"].zero_()
    sd[p + "attention.output.dense.weight"] = torch.eye(H)
    sd[p + "attention.output.dense.bias"].zero_()
    sd[p + "output.LayerNorm.weight"].fill_(1.0)
    sd[p + "output.LayerNorm.bias"].zero_()
    ids, mask = _ids(gen, B, L, 2000)
    probe = _Logits()
    _, (hidden, _), (oh, ah) = _compare(enc_mod, "isolated L=%d" % L, spec, sd, ids, mask, probe=probe)
    assert float(probe.row_pmax(0, mask.bool()).median()) >= 0.5  # premise: attention is peaked
    m = mask.numpy().astype(bool)
    g, o, a = hidden[m], oh[m], ah[m]
    ek = np.linalg.norm(g - o, axis=1) / np.linalg.norm(o, axis=1)
    ea = np.linalg.norm(a - o, axis=1) / np.linalg.norm(o, axis=1)
    worst = int(np.argmax(ek - C * ea))
    print("[numerics] isolated L=%d per token: max err_kernel %.3e  max err_autocast %.3e  worst token %.3e vs %.3e"
          % (L, ek.max(), ea.max(), ek[worst], ea[worst]))
    assert ek.max() <= C * ea.max() + FLOOR
    assert (ek <= C * ea + 5 * FLOOR + 2 ** -8).all(), "token %d: %.3e vs autocast %.3e" % (worst, ek[worst], ea[worst])


# ------------------------------------------------------------------------------------------------------------------
# online softmax across key tiles (attn_stream_kernel) and saturated exponents (both attention kernels)
# ------------------------------------------------------------------------------------------------------------------
def _tile_gap(s, rows, q_tiles, early):
    """for every selected query row: (max logit of key tile 0 - max of later tiles) if early, else
    (max of the last key tile - max of the earlier tiles); s [B, heads, L, L], rows [B, L] bool"""
    first, rest = s[..., :128].amax(-1), s[..., 128:].amax(-1)
    last, before = s[..., -128:].amax(-1), s[..., :-128].amax(-1)
    gap = (first - rest) if early else (last - before)
    sel = rows.clone()
    sel[:, q_tiles * 128:] = False
    return gap[sel[:, None, :].expand_as(gap)]


@pytest.mark.parametrize("early", [False, True], ids=["max_in_last_tile", "max_in_tile0"])
@pytest.mark.parametrize("L,B", [(256, 3), (512, 2)])
def test_online_softmax_tile_maxima_bert(enc_mod, L, B, early):
    # hidden dim 0 of the position embedding marks the key tile (+a in the favoured tile, -a elsewhere); the key
    # projection turns it into +-beta in dimension 0 of every head's key and the query bias puts gamma there, so the
    # favoured tile's logits exceed every other tile's by 2 * gamma * beta / 8 nats (BERT scales logits by 1/8)
    gen = torch.Generator().manual_seed(1200 + L + early)
    H, F = 768, 1536
    spec = _bert_spec(1, H, 12, F)
    sd = _rand_bert_sd(gen, 1, H, F, 2000, 512)
    fav = torch.zeros(512, dtype=torch.bool)
    fav[:128] = early
    fav[L - 128:L] = not early
    a = 0.18  # LN-normalised value of dimension 0: about +-5
    sd["embeddings.position_embeddings.weight"][:, 0] = torch.where(fav, a, -a)
    sd["embeddings.LayerNorm.weight"][0], sd["embeddings.LayerNorm.bias"][0] = 1.0, 0.0
    gamma, beta = (12.0, 16.0) if early else (10.0, 14.0)
    p = "encoder.layer.0.attention.self."
    wk, bq = sd[p + "key.weight"], sd[p + "query.bias"]
    for h in range(12):
        wk[64 * h] = 0.0
        wk[64 * h, 0] = beta / 5.0
        bq[64 * h] = gamma
    ids, mask = _ids(gen, B, L, 2000, ragged=False)
    mask[1, 3:40] = 0  # holes inside tile 0
    probe = _Logits()
    _compare(enc_mod, "bert %s L=%d" % ("tile0-max" if early else "last-tile-max", L), spec, sd, ids, mask, probe=probe)
    gap = _tile_gap(probe.by_layer[0], mask.bool(), L // 128, early)
    need = 30.0 if early else 20.0
    print("[numerics] premise: min tile gap %.1f nats >= %.0f" % (float(gap.min()), need))
    assert float(gap.min()) >= need, "premise: tile gap %.1f < %.0f nats" % (float(gap.min()), need)


def _t5_rel_pattern(sd, heads, pattern):
    """relative-position bias table [32 buckets, heads]: 'far' = +15 for keys >= 91 positions ahead (the saturated
    bucket), -15 elsewhere: a query's maximum sits in a later key tile; 'local' = +10 for |rel| < 8, -20 elsewhere:
    every row's exponents beyond its neighbourhood underflow"""
    from oracle.encoder import t5_relative_position_bucket
    rel = torch.arange(-600, 601)
    b = t5_relative_position_bucket(rel, 32, 128)
    if pattern == "far":
        table = torch.full((32, heads), -15.0)
        table[b[rel >= 91].unique()] = 15.0
    else:
        table = torch.full((32, heads), -20.0)
        table[b[rel.abs() < 8].unique()] = 10.0
    sd["encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight"] = table
    return sd


@pytest.mark.parametrize("pattern,L,B", [("far", 128, 4), ("far", 256, 2), ("far", 512, 1), ("local", 32, 12),
                                         ("local", 256, 2), ("local", 512, 1)])
def test_t5_extreme_relative_bias(enc_mod, pattern, L, B):
    gen = torch.Generator().manual_seed(1300 + L)
    H, heads, F = 768, 12, 1536
    spec = _t5_spec(2, H, heads, F)
    sd = _t5_rel_pattern(_rand_t5_sd(gen, 2, H, heads, F, 2000), heads, pattern)
    head_w = torch.randn(H, H, generator=gen) * H ** -0.5
    ids, mask = _ids(gen, B, L, 2000, ragged=False)
    probe = _Logits()
    _compare(enc_mod, "t5 %s L=%d" % (pattern, L), spec, sd, ids, mask, head=head_w, pooling="mean", normalize=True,
             probe=probe)
    s = probe.by_layer[0]
    q = torch.arange(L)
    if pattern == "far" and L > 128:
        # queries 37..127: every favoured key lies in a later tile, so the running maximum jumps after key tile 0
        gap = (s[..., 128:].amax(-1) - s[..., :128].amax(-1))[..., 37:128]
        need, what = 20.0, "later-tile max - tile-0 max"
    elif pattern == "local" and L > 128:
        # queries 0..119: the neighbourhood lies in key tile 0, every later tile is >= 30 nats lower
        gap = (s[..., :128].amax(-1) - s[..., 128:].amax(-1))[..., :120]
        need, what = 25.0, "tile-0 max - later-tile max"
    else:  # one attention tile (attn_kernel): rows that span >= 20 nats, most of their exponents underflow
        spread = s.amax(-1) - s.masked_fill(torch.isinf(s), float("inf")).amin(-1)
        gap = spread[..., q < 37] if pattern == "far" else spread
        need, what = 20.0, "logit spread"
    print("[numerics] premise: min %s %.1f nats >= %.0f" % (what, float(gap.min()), need))
    assert float(gap.min()) >= need, "premise: %s %.1f < %.0f nats" % (what, float(gap.min()), need)


# ------------------------------------------------------------------------------------------------------------------
# residual offsets: the folded LayerNorm sees |mean(s)| >> std(s)
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("b0,massive", [(0, False), (1, False), (4, False), (16, False), (1, True)])
def test_bert_residual_offset(enc_mod, b0, massive):
    # every LayerNorm beta gets a common offset b0 and the embedding sum gets one too (through the word embeddings):
    # the un-normalised residual rows that the QKV / FFN1 GEMMs read then have |mean| / std >> 1
    gen = torch.Generator().manual_seed(1400 + b0)
    layers, H, F = 2, 768, 1536
    spec = _bert_spec(layers, H, 12, F)
    sd = _rand_bert_sd(gen, layers, H, F, 2000, 512)
    sd["embeddings.word_embeddings.weight"] += b0
    for k in list(sd):
        if k.endswith("LayerNorm.bias"):
            sd[k] = sd[k] + b0
        if massive and k.endswith("LayerNorm.weight"):
            sd[k][[17, 301]] = 20.0
    ids, mask = _ids(gen, 6, 64, 2000)
    tt = torch.randint(0, 2, ids.shape, generator=gen)
    emb = (sd["embeddings.word_embeddings.weight"][ids] + sd["embeddings.token_type_embeddings.weight"][tt]
           + sd["embeddings.position_embeddings.weight"][:64][None]).double()
    ratio = float((emb.mean(-1).abs() / emb.std(-1)).median())
    print("[numerics] premise: embedding |mean| / std = %.1f" % ratio)
    assert (ratio > 10 * b0) if b0 else (ratio < 0.5)
    # the outputs carry the last LayerNorm's beta (~b0 in every column): judged without it
    out, _, _ = _compare(enc_mod, "bert offset b0=%d%s" % (b0, " massive" if massive else ""), spec, sd, ids, mask, tt,
                         fixed=b0 <= 4, shift=sd["encoder.layer.%d.output.LayerNorm.bias" % (layers - 1)])
    ek, ea = out["hidden"]
    print("[numerics] offset b0=%d%s: hidden err_kernel / err_autocast = %.2f" % (b0, " massive" if massive else "",
                                                                              ek / ea))


def test_t5_massive_embedding_dims(enc_mod):
    # RMSNorm has no centring: two embedding dimensions x100 dominate the row norm of the residual stream
    gen = torch.Generator().manual_seed(1500)
    H, heads, F = 768, 12, 1536
    spec = _t5_spec(2, H, heads, F)
    sd = _rand_t5_sd(gen, 2, H, heads, F, 2000)
    sd["shared.weight"][:, [5, 600]] *= 100.0
    ids, mask = _ids(gen, 6, 64, 2000)
    _compare(enc_mod, "t5 massive dims", spec, sd, ids, mask)


# ------------------------------------------------------------------------------------------------------------------
# shapes no other test runs
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("arch,H,heads,F", [("bert", 256, 4, 832), ("t5", 768, 12, 1088), ("t5", 512, 16, 2048),
                                            ("t5", 1024, 8, 2048), ("t5", 1024, 16, 1024)])
def test_shape_edges(enc_mod, arch, H, heads, F):
    # ffn % 128 == 64 (half-width last tile of FFN1, K = ffn for FFN2), heads * 64 != hidden (T5), hidden 1024 (all 16
    # row-statistics slots)
    gen = torch.Generator().manual_seed(1600 + H + heads + F)
    if arch == "bert":
        spec = _bert_spec(2, H, heads, F)
        sd = _rand_bert_sd(gen, 2, H, F, 2000, 512)
    else:
        spec = _t5_spec(2, H, heads, F)
        sd = _rand_t5_sd(gen, 2, H, heads, F, 2000)
    ids, mask = _ids(gen, 5, 100, 2000)
    _compare(enc_mod, "%s H=%d heads=%d F=%d" % (arch, H, heads, F), spec, sd, ids, mask, pooling="mean")


@pytest.mark.parametrize("head_out", [8, 100, 768])
def test_bert_linear_head(enc_mod, head_out):
    gen = torch.Generator().manual_seed(1700 + head_out)
    H, F = 256, 512
    spec = _bert_spec(2, H, 4, F)
    sd = _rand_bert_sd(gen, 2, H, F, 2000, 512)
    head_w = torch.randn(head_out, H, generator=gen) * H ** -0.5
    ids, mask = _ids(gen, 9, 48, 2000)
    for pooling in ("first", "mean"):
        for normalize in (False, True):
            enc = enc_mod.CudaEncoder(spec, sd, head_weight=head_w, pooling=pooling, normalize=normalize,
                                      max_batch_tokens=ids.numel())
            assert enc.rep_dim == head_out
            _, (_, reps), _ = _compare(enc_mod, "head %d %s%s" % (head_out, pooling, " norm" if normalize else ""), spec,
                                       sd, ids, mask, head=head_w, pooling=pooling, normalize=normalize, enc=enc)
            # bf16 output into a strided buffer: the same values rounded once, neighbours untouched
            buf = torch.full((9, head_out + 24), 7.0, dtype=torch.bfloat16, device="cuda")
            enc.encode(ids.cuda(), mask.cuda(), out=buf[:, 8:8 + head_out])
            assert torch.equal(buf[:, 8:8 + head_out].cpu(), torch.from_numpy(reps).to(torch.bfloat16))
            assert (buf[:, :8] == 7).all() and (buf[:, 8 + head_out:] == 7).all()


@pytest.mark.parametrize("case", ["left_pad_100", "holes_17", "holes_32", "single_token", "tile0_masked_256",
                                  "tile0_masked_512"])
def test_non_prefix_masks(enc_mod, case):
    gen = torch.Generator().manual_seed(1800 + len(case))
    L, B = {"left_pad_100": (100, 4), "holes_17": (17, 16), "holes_32": (32, 12), "single_token": (32, 6),
            "tile0_masked_256": (256, 2), "tile0_masked_512": (512, 2)}[case]
    H, F = 768, 1536
    spec = _bert_spec(2, H, 12, F)
    sd = _scale_query(_rand_bert_sd(gen, 2, H, F, 2000, 512), 2, 15)  # peaked rows: a wrongly kept key shows
    ids, mask = _ids(gen, B, L, 2000, ragged=False)
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
        mask[:, :128] = 0  # the first key tile of every sequence is fully masked
        mask[0, 128:150] = 0
    _compare(enc_mod, "mask %s" % case, spec, sd, ids, mask, pooling="mean")


# ------------------------------------------------------------------------------------------------------------------
# determinism and batch invariance
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("L", [128, 256])
def test_bitwise_determinism_and_batch_invariance(enc_mod, L):
    # L > 64: one sequence per attention tile, every row's arithmetic is independent of the others -> bitwise.
    # 40 sequences x 12 heads exceed the persistent attn_kernel grid at L = 128, so CTAs loop over items.
    gen = torch.Generator().manual_seed(1900 + L)
    H, F = 768, 1536
    spec = _bert_spec(2, H, 12, F)
    sd = _scale_query(_rand_bert_sd(gen, 2, H, F, 2000, 512), 2, 15)
    enc = enc_mod.CudaEncoder(spec, sd, pooling="mean", max_batch_tokens=40 * L)
    ids, mask = _ids(gen, 40, L, 2000)
    ids, mask = ids.cuda(), mask.cuda()
    h1, r1 = enc.encode(ids, mask, return_hidden=True)
    h1, r1 = h1.clone(), r1.clone()
    h2, r2 = enc.encode(ids, mask, return_hidden=True)
    assert torch.equal(h1, h2) and torch.equal(r1, r2), "run-to-run difference"
    for b in (0, 1, 17, 39):
        ha, ra = enc.encode(ids[b:b + 1], mask[b:b + 1], return_hidden=True)
        assert torch.equal(ra[0], r1[b]), "sequence %d alone differs from its row in the batch" % b
        assert torch.equal(ha[0], h1[b])


def test_packed_slot_invariance(enc_mod):
    # L = 32 packs 4 sequences per attention tile: the same sequence at slot 0 and slot 3 uses another key grouping of
    # the P V k-steps, so the two agree within the error model, not bitwise
    gen = torch.Generator().manual_seed(2000)
    H, F = 768, 1536
    spec = _bert_spec(2, H, 12, F)
    sd = _scale_query(_rand_bert_sd(gen, 2, H, F, 2000, 512), 2, 15)
    ids, mask = _ids(gen, 8, 32, 2000)
    ids[3], mask[3] = ids[0], mask[0]
    ids[6], mask[6] = ids[0], mask[0]  # slot 2 of the second tile
    enc = enc_mod.CudaEncoder(spec, sd, pooling="mean", max_batch_tokens=ids.numel())
    reps = enc.encode(ids.cuda(), mask.cuda()).cpu().numpy()
    ospec = _ospec(spec, "mean")
    _, o = oracle.encode_reps(sd, ospec, ids[:1], mask[:1], dtype=F64)
    _, a = oracle.encode_reps(sd, ospec, ids[:1], mask[:1], dtype=F64, emulate_bf16=True)
    ea = _rel(a.numpy(), o.numpy())
    for slot in (3, 6):
        d = _rel(reps[slot:slot + 1], reps[:1])
        print("[numerics] packed slot 0 vs %d: rel diff %.3e (err_autocast %.3e)" % (slot, d, ea))
        assert d <= 2 * C * ea + FLOOR
