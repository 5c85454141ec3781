"""Adversarial attention statistics for the encoder's attention kernels, and fault models of those kernels on the float64
oracle; shared by tests/test_attention_stress_cpu.py and tests/test_attention_stress_gpu.py.

Every construction is generic in the head width dh = hidden // heads, so the same case drives the 64-wide kernels and
the 32-wide ones, where two heads share one 64-column unit:
  * token magnets: word-embedding dimension 0 is +A for the magnet id MAGNET, 0 for NEUTRAL and -A for every other id
    (the embedding LayerNorm keeps dimension 0: gamma_0 = 1, beta_0 = 0, so it stays about +-5 after it).  Each head's
    key row dh * h reads that dimension (BETA / 5 per unit) and its query bias puts +-GAMMA there: even heads put all
    their probability on a visible magnet, odd heads none, with a margin of 2 GAMMA BETA / sqrt(dh) >= 30 nats.  A
    sequence without a magnet attends almost uniformly, so one magnet key that leaks into it moves its output by O(1).
    NEUTRAL sits at the level of the packed layout's zeroed padding rows, 17 - 25 nats above ordinary tokens in the
    even heads: a padding key that is wrongly kept takes over those heads too.
  * tile levels: the same key / query planting, read from dimension 0 of the position embedding, so that the favoured
    key tile (or key) is chosen by position; polarity alternates by head here too.
  * peaked levels (``scale_query``) and isolated-per-token layers (``isolate_layer``).

Fault models run the oracle with ``oracle.encoder._softmax_rows`` replaced (through pytest's monkeypatch; the oracle
files are not touched): ``oracle_hidden`` runs it with an all-ones attention mask and applies the keys a query may see
as an explicit [B, 1 | heads, L, L] mask, so a fault is a changed mask (a neighbour's key leaked, a masked key kept, the
valid keys of the partial last tile dropped, the padding keys of the last tile kept) or a changed P (the two heads of a
unit swapped)."""
import contextlib
import io

import numpy as np
import torch

import oracle
import oracle.encoder as oe
from oracle.encoder import EncoderSpec

F64 = torch.float64
A, GAMMA, BETA = 0.18, 12.0, 16.0  # the scale of the suite's tile-maxima tests (key tile 0 favoured)
MAGNET, NEUTRAL = 7, 0
C, FLOOR = 2.0, 2e-4  # the error model of tests/test_encoder_numerics_gpu.py, applied to a whole call
# one sequence: the constructions put a 25 - 50 nat constant into every logit of a row, whose bf16 rounding the kernel's
# extra rounding sites (folded weights, un-normalised residual) carry per key; a single sequence then measures up to
# 2.8x its autocast error on an H100 (a tail of the per-sequence ratio that the aggregate averages out)
C_SEQ = 3.0


def bert_spec(layers, H, heads, F=256, vocab=1000, max_pos=8192, arch="bert"):
    return dict(arch=arch, layers=layers, hidden=H, heads=heads, ffn=F, vocab=vocab, max_pos=max_pos,
                type_vocab=2 if arch == "bert" else 1, ln_eps=1e-12)


def ospec(spec, pooling="first", normalize=False):
    arch = "t5" if spec["arch"] == "t5" else "bert"  # RoBERTa: the BERT oracle with RoBERTa's position ids
    return EncoderSpec(arch, spec["layers"], spec["hidden"], spec["heads"], spec["ffn"], spec["ln_eps"],
                       pooling=pooling, normalize=normalize)


def plant_dim0(sd, heads, dh, gamma=GAMMA, beta=BETA, layer=0):
    """key row dh * h of every head reads hidden dimension 0, the query bias puts +gamma (even heads) or -gamma (odd
    heads) there; the embedding LayerNorm passes dimension 0 through unscaled"""
    sd["embeddings.LayerNorm.weight"][0], sd["embeddings.LayerNorm.bias"][0] = 1.0, 0.0
    p = f"encoder.layer.{layer}.attention.self."
    wk, bq = sd[p + "key.weight"], sd[p + "query.bias"]
    for h in range(heads):
        wk[dh * h] = 0.0
        wk[dh * h, 0] = beta / 5.0
        bq[dh * h] = gamma if h % 2 == 0 else -gamma
    return sd


def magnet_model(sd, heads, dh):
    w = sd["embeddings.word_embeddings.weight"]
    w[:, 0] = -A
    w[MAGNET, 0] = A
    w[NEUTRAL, 0] = 0.0
    return plant_dim0(sd, heads, dh)


def tile_level_model(sd, heads, dh, level, early):
    """level [n <= max_pos]: dimension 0 of the first n position-embedding rows (later rows 0, the padding level);
    (gamma, beta) as the suite's tile-maxima tests: a wider margin when the maximum sits in key tile 0"""
    pe = sd["embeddings.position_embeddings.weight"]
    pe[:, 0] = 0.0
    pe[:len(level), 0] = level
    gamma, beta = (12.0, 16.0) if early else (10.0, 14.0)
    return plant_dim0(sd, heads, dh, gamma, beta)


def tile_level(L, where):
    """dimension-0 level of positions [0, L): +A in the favoured keys, -A elsewhere; 'tile0' / 'last_tile' favour a
    128-key tile, 'last_key' only position L - 1 (at L = 128 k + 1 the whole partial last tile), 'moving' rises
    linearly from -A to +A"""
    pos = torch.arange(L)
    if where == "moving":
        return A * (2.0 * pos / (L - 1) - 1.0)
    fav = {"tile0": pos < 128, "last_tile": pos >= (L - 1) // 128 * 128, "last_key": pos == L - 1}[where]
    return torch.where(fav, A, -A)


def scale_query(sd, layers, alpha):
    sd = dict(sd)
    for i in range(layers):
        for n in ("weight", "bias"):
            k = f"encoder.layer.{i}.attention.self.query.{n}"
            sd[k] = sd[k] * alpha
    return sd


def isolate_layer(sd, H):
    """layer 0 with a zero FFN and the identity as O-projection: its output is LN2(LN1(s0 + ctx)), so an attention
    error reaches every token undiluted"""
    p = "encoder.layer.0."
    for n in ("intermediate.dense", "output.dense"):
        sd[p + n + ".weight"].zero_()
        sd[p + n + ".bias"].zero_()
    sd[p + "attention.output.dense.weight"] = torch.eye(H)
    sd[p + "attention.output.dense.bias"].zero_()
    sd[p + "output.LayerNorm.weight"].fill_(1.0)
    sd[p + "output.LayerNorm.bias"].zero_()
    return sd


# peaked levels: (query scale alpha, lo, hi) of the median row-max probability at each length, hidden 768
PEAK = {"flat": {17: (1, 0, 0.15), 128: (1, 0, 0.05), 512: (1, 0, 0.02), 1000: (1, 0, 0.01), 3000: (1, 0, 0.005)},
        "half": {17: (9, 0.3, 0.7), 128: (15, 0.3, 0.7), 512: (20, 0.3, 0.7), 1000: (22, 0.25, 0.7),
                 3000: (25, 0.2, 0.7)},
        "sharp": {17: (40, 0.95, 1), 128: (64, 0.95, 1), 512: (80, 0.95, 1), 1000: (90, 0.9, 1),
                  3000: (100, 0.9, 1)}}


# ------------------------------------------------------------------------------------------------------------------
# sequences
# ------------------------------------------------------------------------------------------------------------------
def plain(gen, n, vocab=1000):
    """ids in [10, vocab): neither MAGNET nor NEUTRAL, nor a special id"""
    return torch.randint(10, vocab, (n,), generator=gen)


def with_magnets(gen, n, where, vocab=1000):
    """'none': no magnet; 'ends': magnets at the first and the last token (every bin neighbour sees one across a
    boundary); 'inside': one magnet at a random position"""
    s = plain(gen, n, vocab)
    if where == "ends":
        s[0] = MAGNET
        s[-1] = MAGNET
    elif where == "inside":
        s[int(torch.randint(0, n, (1,), generator=gen))] = MAGNET
    return s


def magnet_padded_batch(gen, L, B):
    """[B, L] ids and mask: sequences without a magnet between sequences with magnets at both ends (neighbour slots of
    a multi-sequence tile), and sequences whose masked keys are magnets (a masked tail, holes; at L >= 256 key tile 0
    fully masked).  Returns ids, mask and the kind of every row."""
    kinds = ([1, 0, 1, 2, 0, 1, 2, 1] * B)[:B]
    ids = torch.empty(B, L, dtype=torch.long)
    mask = torch.ones(B, L, dtype=torch.long)
    for b, k in enumerate(kinds):
        ids[b] = with_magnets(gen, L, ["none", "ends", "none"][k])
        if k == 2:
            cut = max(1, L - L // 3)
            if L >= 256:
                mask[b, :128] = 0
                ids[b, torch.randint(0, 128, (12,), generator=gen)] = MAGNET
            elif L > 2:
                hole = torch.randint(1, cut, (max(1, L // 8),), generator=gen)
                mask[b, hole] = 0
                ids[b, hole] = MAGNET
            mask[b, cut:] = 0
            ids[b, cut:] = MAGNET
            if L == 1:
                mask[b] = 1
    return ids, mask, kinds


# ------------------------------------------------------------------------------------------------------------------
# premises on the float64 oracle's logits
# ------------------------------------------------------------------------------------------------------------------
class Logits:
    """probe: each layer's masked attention logits (float64, natural-log units)"""

    def __init__(self):
        self.by_layer = {}

    def __call__(self, layer, s):
        self.by_layer[layer] = s


def magnet_margins(s, ids, allowed):
    """(even-head margin, odd-head margin, even-head min P(magnets)) over the query rows that see a magnet: even heads
    min(magnet logit) - max(other logit), odd heads min(other logit) - max(magnet logit); s [B, heads, L, L], ids
    [B, L], allowed [B, L, L] bool (query, key) or None for every key allowed"""
    B, nh, L, _ = s.shape
    if allowed is None:
        allowed = torch.ones(B, L, L, dtype=torch.bool)
    allowed = allowed & torch.isfinite(s).all(1)
    mag = (ids == MAGNET)[:, None, :] & allowed  # [B, q, k]
    oth = (ids != MAGNET)[:, None, :] & allowed
    rows = mag.any(-1) & oth.any(-1)
    inf = float("inf")
    big, small = s.masked_fill(~mag[:, None], inf).amin(-1), s.masked_fill(~oth[:, None], -inf).amax(-1)
    m_even = (big - small)[:, 0::2][rows[:, None].expand(-1, (nh + 1) // 2, -1)]
    big, small = s.masked_fill(~oth[:, None], inf).amin(-1), s.masked_fill(~mag[:, None], -inf).amax(-1)
    m_odd = (big - small)[:, 1::2][rows[:, None].expand(-1, nh // 2, -1)]
    p = torch.softmax(s.masked_fill(~allowed[:, None], -inf), -1)
    pm = (p * mag[:, None]).sum(-1)[:, 0::2][rows[:, None].expand(-1, (nh + 1) // 2, -1)]
    return float(m_even.min()), float(m_odd.min()), float(pm.min())


def tile_gaps(s, L, early, q_rows=None):
    """(even-head gap, odd-head gap) of one sequence's logits s [1, heads, L, L]: even heads (max of the favoured key
    tile - max of the others), odd heads (max of the others - max of the favoured tile); the favoured tile is key tile
    0 if early, else the last (possibly partial) one"""
    t = 128 if early else (L - 1) // 128 * 128
    fav, rest = (s[..., :t], s[..., t:]) if early else (s[..., t:], s[..., :t])
    gap = fav.amax(-1) - rest.amax(-1)
    if q_rows is not None:
        gap = gap[..., q_rows]
    return float(gap[:, 0::2].min()), float(-gap[:, 1::2].max())


def row_pmax_median(s, rows=None):
    p = torch.softmax(s, -1).amax(-1)  # [B, heads, L]
    if rows is not None:
        p = p[rows[:, None, :].expand_as(p)]
    return float(p.median())


# ------------------------------------------------------------------------------------------------------------------
# the oracle under a fault model
# ------------------------------------------------------------------------------------------------------------------
def keyed_softmax(orig, allowed, swap_pairs=False):
    """a _softmax_rows that forbids the keys ``allowed`` [B, 1 | heads, L, L] excludes and, with swap_pairs, hands head
    2u the probabilities of head 2u + 1 and back (the two 32-wide heads of a unit swapped)"""

    def softmax_rows(s):
        p = orig(s.masked_fill(~allowed, float("-inf")))
        if swap_pairs:
            B, nh, L, K = p.shape
            p = p.reshape(B, nh // 2, 2, L, K).flip(2).reshape(B, nh, L, K)
        return p

    return softmax_rows


def oracle_hidden(monkeypatch, sd, spec, ids, allowed, swap_pairs=False, emulate_bf16=False, probe=None):
    """hidden rows [B, L, H] of the oracle (float64; bf16 autocast emulated if asked) where query q of row b may see
    key k iff allowed[b, q, k] ([B, L, L] bool)"""
    orig = oe._softmax_rows
    with monkeypatch.context() as mp:
        mp.setattr(oe, "_softmax_rows", keyed_softmax(orig, allowed[:, None], swap_pairs))
        h, _ = oracle.encode_reps(sd, ospec(spec), ids, torch.ones_like(ids), dtype=F64, emulate_bf16=emulate_bf16,
                                  probe=probe)
    return h


def seq_allowed(L_total, lo, hi, valid=None):
    """[1, L_total, L_total]: every query sees keys [lo, hi) that are valid"""
    k = torch.zeros(L_total, dtype=torch.bool)
    k[lo:hi] = True
    if valid is not None:
        k &= valid
    return k[None, None, :].expand(1, L_total, L_total).clone()


def rel(got, want):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    return float(np.linalg.norm(got - want) / max(np.linalg.norm(want), 1e-30))


def judge_each(what, items):
    """judge every (name, got, ref, auto) by the rule of tests/test_encoder_numerics_gpu.py's _judge: the fixed bound
    (rel-L2 <= 1e-2, cosine >= 0.9999) where err_autocast <= 5.3e-3, and err_kernel <= C err_autocast + FLOOR for the
    whole call ("all ..." items), C_SEQ err_autocast + FLOOR for one sequence.  A
    sequence's err_autocast is one draw of the bf16 rounding noise, over as little as one row (its reps, a 1-token
    sequence): it is taken no smaller than that of the whole call ("all reps" / "all hidden", the last items), so a
    sequence whose autocast run happens to land close to float64 is not held to a bound below the noise level.  Every
    item is judged before any failure is raised; prints one line with the worst err_kernel / err_autocast."""
    from test_encoder_gpu import _check
    from test_encoder_numerics_gpu import AUTOCAST_ANCHOR
    call = {name.split()[-1]: rel(auto, ref) for name, got, ref, auto in items if name.startswith("all ")}
    worst, worst_name, fails = -1.0, "", []
    for name, got, ref, auto in items:
        got, ref, auto = (np.asarray(x, np.float64).reshape(-1, np.shape(x)[-1]) for x in (got, ref, auto))
        ek, ea = rel(got, ref), max(rel(auto, ref), call.get(name.split()[-1], 0.0))
        if not np.isfinite(got).all():
            fails.append("%s: non-finite output" % name)
            continue
        if ek / max(ea, 1e-30) > worst:
            worst, worst_name = ek / max(ea, 1e-30), name
        c = C if name.startswith("all ") else C_SEQ
        if ek > c * ea + FLOOR:
            fails.append("%s: err_kernel %.3e > %.1f * err_autocast %.3e + %.0e" % (name, ek, c, ea, FLOOR))
        if ea <= AUTOCAST_ANCHOR:
            try:
                with contextlib.redirect_stdout(io.StringIO()):
                    _check(got, ref, name)
            except AssertionError as e:
                fails.append(str(e))
    print("[numerics] %-44s %d outputs judged, worst err_kernel / err_autocast %.2f (%s)" % (what, len(items), worst,
                                                                                          worst_name))
    assert not fails, what + ": " + "; ".join(fails)
    return worst
