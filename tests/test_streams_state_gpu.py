"""GPU: the C ABI's stream contract and handle state across calls.

The ABI (include/openmatch_b200.h) takes raw pointers plus a cudaStream_t and is asynchronous on that stream.  Every
other GPU test runs on torch's default stream, the legacy NULL stream, which orders any work the library issues
elsewhere for free.  Here the caller works on a ``torch.cuda.Stream()``: a non-blocking stream that neither waits for
the NULL stream nor is waited for by it.  ``busy`` keeps a stream occupied with a device-side sleep, so that every race
below is decided deterministically, and each test asserts that the stream really was still busy at the racing call.
  * stream ordering: reset, weight upload, and every asynchronous entry point with inputs still pending on the side
    stream, each bitwise equal to the default-stream result;
  * call sequences: one encoder handle across geometries, one index across dtype paths, reserve / commit, growth and
    reset, each step bitwise equal to a fresh handle;
  * poisoned allocations: handles whose every allocation the library fills with NaN bytes, so that any read of
    never-written workspace shows up as NaN or a mismatch instead of a silent zero.
Nothing here changes device settings or provokes a fault; every sleep is at most a quarter of a second at the card's
maximum SM clock."""
import ctypes
import os
import types

import numpy as np
import pytest
import torch

from oracle import search_bound as sb
from test_encoder_gpu import _ids, _rand_bert_sd, _rand_t5_sd
from test_search_gpu import _near_duplicate_corpus

pytestmark = pytest.mark.gpu

SLEEP = 0.25  # seconds at the maximum SM clock: at most 0.5 s even if the clock runs at half speed
STATS = ("uncertified", "uncertified_wide", "exact_queries")
BERT = dict(arch="bert", layers=2, hidden=256, heads=4, ffn=512, vocab=1000, max_pos=512, type_vocab=2, ln_eps=1e-12)
T5 = dict(arch="t5", layers=2, hidden=256, heads=4, ffn=512, vocab=1000, ln_eps=1e-6, rel_buckets=32,
          rel_max_distance=128)


@pytest.fixture(scope="module")
def om():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from openmatch_b200 import _lib, encoder, index, loss
    return types.SimpleNamespace(lib=_lib, encoder=encoder, index=index, loss=loss)


def busy(stream, seconds=SLEEP):
    """Occupies ``stream`` with a device-side spin of ``seconds`` at the maximum SM clock (clock_rate is in kHz)."""
    assert 0 < seconds <= 0.25
    cycles = int(seconds * torch.cuda.get_device_properties(torch.cuda.current_device()).clock_rate * 1e3)
    with torch.cuda.stream(stream):
        torch.cuda._sleep(cycles)


def _null():
    return torch.cuda.default_stream()


def _bits(t):
    t = t.detach().contiguous()
    return t.view({4: torch.int32, 2: torch.int16, 8: torch.int64}[t.element_size()])


def _same(a, b, what):
    """Bitwise equality (NaN payloads included), with a readable message."""
    assert a.shape == b.shape and a.dtype == b.dtype, what
    if not torch.equal(_bits(a), _bits(b)):
        diff = (_bits(a) != _bits(b)).sum().item()
        nan = torch.isnan(a.float()).sum().item() if a.is_floating_point() else 0
        raise AssertionError("%s: %d of %d elements differ bitwise (%d NaN in the first)" % (what, diff, a.numel(), nan))


def _pending_copy(stream, *srcs):
    """Copies of ``srcs`` made on ``stream`` behind a sleep: the inputs of the next call are still being written."""
    with torch.cuda.stream(stream):
        outs = [torch.empty_like(t) for t in srcs]
        busy(stream)
        for o, t in zip(outs, srcs):
            o.copy_(t)
    assert not stream.query(), "premise: the side stream must still be busy"
    return outs


def _encoder(om, spec, sd, head=None, pooling="first", normalize=False, max_batch_tokens=4096):
    return om.encoder.CudaEncoder(spec, sd, head_weight=head, pooling=pooling, normalize=normalize,
                                  max_batch_tokens=max_batch_tokens)


def _bert_batch(gen, B, L, vocab=1000):
    ids, mask = _ids(gen, B, L, vocab)
    return ids.cuda(), mask.cuda(), torch.randint(0, 2, (B, L), generator=gen).cuda()


def _hf_bert():
    from transformers import BertConfig, BertModel
    torch.manual_seed(5)
    cfg = BertConfig(vocab_size=512, hidden_size=128, num_hidden_layers=2, num_attention_heads=2, intermediate_size=512,
                     max_position_embeddings=128)
    return BertModel(cfg).cuda().eval()


def _drmodel(lm):
    from openmatch.arguments import ModelArguments
    from openmatch.modeling import DRModel
    return DRModel(lm_q=lm, lm_p=lm, tied=True, pooling="first", model_args=ModelArguments("unused")).eval()


def _search_all(idx, qd, k=10, nqs=(64, 300)):
    """D, I, the certificate statistics and the candidate-stage scores for each query count (both scan kernels)."""
    out = {}
    for nq in nqs:
        D, I = idx.search_device(qd[:nq], k)
        st = tuple(idx.stat(s) for s in STATS)
        idx.set_param("debug_stage_scores", 1)
        Ds, Is = idx.search_device(qd[:nq], k)
        idx.set_param("debug_stage_scores", 0)
        out[nq] = (D, I, st, Ds, Is)
    return out


def _same_search(got, want, what):
    for nq in want:
        D, I, st, Ds, Is = got[nq]
        D0, I0, st0, Ds0, Is0 = want[nq]
        _same(I, I0, "%s nq=%d: I" % (what, nq))
        _same(D, D0, "%s nq=%d: D" % (what, nq))
        assert st == st0, "%s nq=%d: certificate statistics %s, fresh index %s" % (what, nq, st, st0)
        _same(Is, Is0, "%s nq=%d: stage ids" % (what, nq))
        _same(Ds, Ds0, "%s nq=%d: stage scores" % (what, nq))


# ---------------------------------------------------------------------------------------------------------------------
# A. stream ordering
# ---------------------------------------------------------------------------------------------------------------------
def test_side_stream_is_non_blocking():
    # premise of every stream test below: a torch side stream does not wait for the legacy NULL stream.  This must fail,
    # not skip, when it does not hold: the tests below would then pass without testing anything.
    assert torch.cuda.is_available(), "the stream tests need a CUDA device"
    assert _null().cuda_stream == 0, "torch's default stream must be the legacy NULL stream"
    s = torch.cuda.Stream()
    x = torch.zeros(256, device="cuda")
    ev = torch.cuda.Event()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(2):  # the first pass loads the kernels (module loading may wait for the whole device)
        torch.cuda.synchronize()
        t0.record(_null())
        busy(_null())
        t1.record(_null())
        with torch.cuda.stream(s):
            x.add_(1)
            ev.record(s)
        ev.synchronize()
        null_idle = _null().query()
    assert not null_idle, "the side stream waited for the NULL stream"
    torch.cuda.synchronize()
    slept = t0.elapsed_time(t1) * 1e-3
    print("[streams] busy(%.2f s) slept %.3f s" % (SLEEP, slept))
    assert 0.5 * SLEEP <= slept <= 0.5, "busy() slept %.3f s" % slept
    assert (x == 2).all()


def test_reset_is_ordered_before_the_next_commit(om):
    # reset() while the NULL stream is busy, then a commit of the same rows on the side stream: the error-norm maxima
    # must be those of the committed rows.  Maxima zeroed after the commit certify the fp16 candidate stage of a
    # near-duplicate cluster as exact: wrong ids with 0 uncertified queries.
    rng = np.random.default_rng(2024)
    n, d, k = 40000, 128, 1000
    x, q, _ = _near_duplicate_corpus(rng, n, d, 6000, 1e-4)
    xd, qd = torch.from_numpy(x).cuda(), torch.from_numpy(q).cuda()
    nq = q.shape[0]
    fresh = om.index.FlatIPIndex(d)
    fresh.add(xd)
    fresh.search_device(qd, k)
    assert fresh.stat("uncertified") == nq, "premise: level 0 must not be able to certify the near-duplicate cluster"
    idx = om.index.FlatIPIndex(d)
    idx.reserve_rows(n)  # capacity up front: a growth synchronises the device and would hide the race
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        idx.add(xd)
        busy(_null())
        idx.reset()
        assert not _null().query(), "premise: the NULL stream must still be busy when reset returns"
        idx.add(xd)
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        D, I = idx.search_device(qd, k)
        st = {name: idx.stat(name) for name in STATS}
        idx.set_param("exact_only", 1)
        De, Ie = idx.search_device(qd, k)
        idx.set_param("exact_only", 0)
    torch.cuda.synchronize()
    print("[streams] reset race: uncertified=%d of %d, exact_queries=%d, ids equal to exact: %s" % (
        st["uncertified"], nq, st["exact_queries"], torch.equal(I, Ie)))
    assert st["uncertified"] == nq, "the certificate proved %d near-duplicate queries exact" % (nq - st["uncertified"])
    _same(I, Ie, "ids after reset + commit on a side stream")
    _same(D, De, "scores after reset + commit on a side stream")


def test_weight_upload_waits_for_pending_writes(om):
    # CudaEncoder construction from device tensors still being written on a side stream must read the final values,
    # both directly and through DRModel._cuda_encoder after an in-place parameter update on that stream
    gen = torch.Generator().manual_seed(21)
    sd = {k: v.cuda() for k, v in _rand_bert_sd(gen, 2, 256, 512, 1000, 512).items()}
    ids, mask, tt = _bert_batch(gen, 6, 64)
    ref = _encoder(om, BERT, sd).encode(ids, mask, tt, return_hidden=True)
    nan = {k: torch.full_like(v, float("nan")) for k, v in sd.items()}
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        busy(s)
        for k, v in sd.items():
            nan[k].copy_(v)
        assert not s.query(), "premise: the weights must still be pending when the encoder is built"
        enc = _encoder(om, BERT, nan)
    torch.cuda.synchronize()
    got = enc.encode(ids, mask, tt, return_hidden=True)
    _same(got[1], ref[1], "reps of an encoder built from pending weights")
    _same(got[0], ref[0], "hidden states of an encoder built from pending weights")

    lm = _hf_bert()
    model = _drmodel(lm)
    hid, hmask, _ = _bert_batch(gen, 5, 40, vocab=512)
    target = {n: p.detach() * 1.5 + 0.01 for n, p in lm.named_parameters()}
    with torch.no_grad():
        for n, p in lm.named_parameters():
            p.copy_(target[n])
    ref = model._cuda_encoder(lm, None).encode(hid, hmask)
    with torch.no_grad():
        for p in lm.parameters():
            p.fill_(float("nan"))
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        busy(s)
        with torch.no_grad():
            for n, p in lm.named_parameters():
                p.copy_(target[n])
        assert not s.query(), "premise: the parameter update must still be pending when the encoder is rebuilt"
        got = model._cuda_encoder(lm, None).encode(hid, hmask)
    torch.cuda.synchronize()
    _same(got, ref, "reps of DRModel's encoder rebuilt after a parameter update on a side stream")


def test_encode_and_ingest_on_a_side_stream(om):
    gen = torch.Generator().manual_seed(22)
    sd = _rand_bert_sd(gen, 2, 256, 512, 1000, 512)
    enc = _encoder(om, BERT, sd)
    ids, mask, tt = _bert_batch(gen, 12, 100)
    want_h, want = enc.encode(ids, mask, tt, return_hidden=True)
    want_bf = enc.encode(ids, mask, tt, out_dtype=torch.bfloat16)
    ref_idx = om.index.FlatIPIndex(enc.rep_dim)
    ref_idx.add(want)
    qd = torch.randn(64, enc.rep_dim, generator=gen).cuda()
    want_search = _search_all(ref_idx, qd, nqs=(64,))
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    ids_s, mask_s, tt_s = _pending_copy(s, ids, mask, tt)
    with torch.cuda.stream(s):
        got_h, got = enc.encode(ids_s, mask_s, tt_s, return_hidden=True)
        got_bf = enc.encode(ids_s, mask_s, tt_s, out_dtype=torch.bfloat16)
    torch.cuda.synchronize()
    _same(got, want, "reps on a side stream")
    _same(got_h, want_h, "hidden states on a side stream")
    _same(got_bf, want_bf, "bf16 reps on a side stream")

    idx = om.index.FlatIPIndex(enc.rep_dim)
    rows = idx.reserve_rows(ids.shape[0])
    ids_s, mask_s, tt_s = _pending_copy(s, ids, mask, tt)
    with torch.cuda.stream(s):
        enc.encode(ids_s, mask_s, tt_s, out=rows)
        idx.commit_rows(ids.shape[0])
        assert not s.query(), "premise: encode + commit must be queued behind the pending inputs"
    torch.cuda.synchronize()
    _same(idx.master_rows(), want, "index rows encoded in place on a side stream")
    _same_search(_search_all(idx, qd, nqs=(64,)), want_search, "search after ingest on a side stream")


def test_index_add_search_merge_on_a_side_stream(om):
    n, d, k = 6000, 256, 10
    x, q, _, _ = sb.make_regime("anisotropic", 300, n, d, k=k, seed=23)
    xd, qd = torch.from_numpy(x).cuda(), torch.from_numpy(q).cuda()
    s = torch.cuda.Stream()
    for dt in (torch.float32, torch.bfloat16, torch.float16):
        src = xd.to(dt)
        ref = om.index.FlatIPIndex(d)
        ref.add(src)
        idx = om.index.FlatIPIndex(d)
        idx.reserve_rows(n)  # capacity up front: no device synchronisation inside add
        torch.cuda.synchronize()
        (pending,) = _pending_copy(s, src)
        with torch.cuda.stream(s):
            idx.add(pending)
        torch.cuda.synchronize()
        _same(idx.master_rows(), ref.master_rows(), "rows of a %s add on a side stream" % dt)
        _same_search(_search_all(idx, qd, nqs=(64,)), _search_all(ref, qd, nqs=(64,)),
                     "search after a %s add on a side stream" % dt)

    idx = om.index.FlatIPIndex(d)
    idx.add(xd)
    for nq in (1, 129, 300):  # one query: single-CTA scan; > 128: the wide scan after the first round
        D0, I0 = idx.search_device(qd[:nq], k)
        st0 = tuple(idx.stat(name) for name in STATS)
        torch.cuda.synchronize()
        (pending,) = _pending_copy(s, qd[:nq])
        with torch.cuda.stream(s):
            D, I = idx.search_device(pending, k)
            st = tuple(idx.stat(name) for name in STATS)
        torch.cuda.synchronize()
        _same(I, I0, "search ids on a side stream, nq=%d" % nq)
        _same(D, D0, "search scores on a side stream, nq=%d" % nq)
        assert st == st0

    parts = [om.index.FlatIPIndex(d) for _ in range(3)]
    Dp, Ip = [], []
    for r, part in enumerate(parts):
        part.add(xd[r * 2000:(r + 1) * 2000])
        D, I = part.search_device(qd, 50, id_offset=r * 2000)
        Dp.append(D)
        Ip.append(I)
    Dp, Ip = torch.stack(Dp), torch.stack(Ip)
    D0, I0 = om.index.merge_topk_device(Dp, Ip, 64)
    torch.cuda.synchronize()
    Dp_s, Ip_s = _pending_copy(s, Dp, Ip)
    with torch.cuda.stream(s):
        D, I = om.index.merge_topk_device(Dp_s, Ip_s, 64)
    torch.cuda.synchronize()
    _same(I, I0, "merged ids on a side stream")
    _same(D, D0, "merged scores on a side stream")


def test_contrastive_loss_on_a_side_stream(om):
    gen = torch.Generator().manual_seed(24)
    nq, n_p, d = 64, 512, 768
    s = torch.cuda.Stream()
    for dt in (torch.bfloat16, torch.float32):
        x0 = (torch.randn(nq, d, generator=gen) * 0.05).to(dt).cuda()
        y0 = (torch.randn(n_p, d, generator=gen) * 0.05).to(dt).cuda()
        for scores in (False, True):
            def run(x_src, y_src):
                x = x_src.detach().clone().requires_grad_(True)
                y = y_src.detach().clone().requires_grad_(True)
                out = om.loss.fused_contrastive_loss(x, y, return_scores=scores)
                loss, sc = out if scores else (out, None)
                loss.backward()
                return loss.detach(), sc, x.grad, y.grad
            # default-stream reference first: this call also initialises the loss's grid barrier and sizes its
            # workspace, so the side-stream call below reuses both
            want = run(x0, y0)
            torch.cuda.synchronize()
            xs, ys = _pending_copy(s, x0, y0)
            with torch.cuda.stream(s):
                got = run(xs, ys)
            torch.cuda.synchronize()
            for name, a, b in zip(("loss", "scores", "dX", "dY"), got, want):
                if b is not None:
                    _same(a, b, "%s %s return_scores=%s on a side stream" % (dt, name, scores))


def test_retriever_ingest_on_a_side_stream(om):
    lm = _hf_bert()
    model = _drmodel(lm)
    gen = torch.Generator().manual_seed(25)
    batches = [_bert_batch(gen, B, L, vocab=512)[:2] for B, L in ((16, 32), (16, 48), (7, 128), (16, 20))]
    total = sum(b[0].shape[0] for b in batches)

    def ingest(stream, side):
        idx = om.index.FlatIPIndex(model.rep_dim())
        idx.reserve_rows(total)  # capacity up front, as Retriever does
        torch.cuda.synchronize()
        for ids, mask in batches:
            if side:
                ids, mask = _pending_copy(stream, ids, mask)
            with torch.cuda.stream(stream):
                rows = idx.reserve_rows(ids.shape[0])
                model.encode_into({"input_ids": ids, "attention_mask": mask}, rows)
                idx.commit_rows(ids.shape[0])
        torch.cuda.synchronize()
        return idx

    ref = ingest(_null(), False)
    got = ingest(torch.cuda.Stream(), True)
    _same(got.master_rows(), ref.master_rows(), "retriever rows ingested on a side stream")
    qd = torch.randn(64, model.rep_dim(), generator=gen).cuda()
    _same_search(_search_all(got, qd, nqs=(64,)), _search_all(ref, qd, nqs=(64,)),
                 "search after retriever ingest on a side stream")
    lm.cpu()


# ---------------------------------------------------------------------------------------------------------------------
# B. call sequences against fresh handles
# ---------------------------------------------------------------------------------------------------------------------
# (L, B, mask, return_hidden, out): 32 x 128 and 128 x 32 fill max_batch_tokens = 4096 exactly, 512 x 1 is one sequence
ENC_SEQ = [(32, 9, "ragged", True, None), (128, 32, "ragged", False, "f32"), (17, 11, "hole", True, None),
           (65, 5, "ragged", False, "bf16"), (100, 3, "hole", True, "f32"), (1, 7, "full", False, None),
           (256, 3, "ragged", True, "bf16"), (512, 1, "hole", False, "f32"), (32, 128, "hole", True, None)]
REFUSE_AFTER = 3  # the two refused calls go between these steps


def _enc_inputs(gen, L, B, kind, vocab):
    ids, mask = _ids(gen, B, L, vocab, ragged=kind != "full")
    if kind == "hole" and L > 4:
        lo, hi = 1 + L // 4, 1 + L // 2
        mask[::2, lo:hi] = 0  # attention holes inside the sequence (token 0 and the tail stay)
        mask[::2, 0] = 1
    return ids.cuda(), mask.cuda(), torch.randint(0, 2, (B, L), generator=gen).cuda()


def _enc_call(enc, inputs, arch, hidden, out_kind):
    ids, mask, tt = inputs
    tt = tt if arch == "bert" else None
    B = ids.shape[0]
    if out_kind is None:
        r = enc.encode(ids, mask, tt, return_hidden=hidden)
        return r if hidden else (None, r)
    dt = torch.float32 if out_kind == "f32" else torch.bfloat16
    buf = torch.full((B, enc.rep_dim + 8), -7.25, dtype=dt, device="cuda")  # row pitch wider than rep_dim
    r = enc.encode(ids, mask, tt, out=buf[:, :enc.rep_dim], return_hidden=hidden)
    assert (buf[:, enc.rep_dim:] == -7.25).all(), "om_encode wrote outside rep_dim of a pitched output"
    return (r[0] if hidden else None), buf[:, :enc.rep_dim]


@pytest.mark.parametrize("arch", ["bert", "t5"])
def test_encoder_call_sequence_matches_fresh_handles(om, arch):
    gen = torch.Generator().manual_seed(31 if arch == "bert" else 32)
    if arch == "bert":
        spec, sd, head, kw = BERT, _rand_bert_sd(gen, 2, 256, 512, 1000, 512), None, dict(pooling="first")
    else:  # relative bias, mean pooling, a linear head and normalisation
        spec, sd = T5, _rand_t5_sd(gen, 2, 256, 4, 512, 1000)
        head, kw = torch.randn(200, 256, generator=gen) * 256 ** -0.5, dict(pooling="mean", normalize=True)
    enc = _encoder(om, spec, sd, head, **kw)
    for step, (L, B, kind, hidden, out_kind) in enumerate(ENC_SEQ):
        assert B * L <= 4096
        inputs = _enc_inputs(gen, L, B, kind, spec["vocab"])
        got_h, got = _enc_call(enc, inputs, arch, hidden, out_kind)
        want_h, want = _enc_call(_encoder(om, spec, sd, head, **kw), inputs, arch, hidden, out_kind)
        what = "%s step %d (L=%d B=%d %s)" % (arch, step, L, B, kind)
        assert torch.isfinite(want.float()).all(), what + ": fresh handle gives non-finite reps"
        _same(got, want, what + ": reps of the reused handle vs a fresh one")
        if hidden:
            _same(got_h, want_h, what + ": hidden states of the reused handle vs a fresh one")
        if step == REFUSE_AFTER:
            z = torch.zeros(33, 128, dtype=torch.long, device="cuda")
            with pytest.raises(RuntimeError, match="max_batch_tokens"):
                enc.encode(z, torch.ones_like(z))
            z = torch.zeros(1, 130, dtype=torch.long, device="cuda")
            with pytest.raises(RuntimeError, match="unsupported"):
                enc.encode(z, torch.ones_like(z))


def test_index_call_sequence_matches_fresh_index(om):
    # one index through every ingest path, compared after each step with a fresh index that received the same rows as
    # one fp32 add: master rows (the dtype-path oracle: bf16 / fp16 upcast exactly), search, certificate statistics and
    # the fp16 scan copy (candidate-stage scores).  The rows before the reset are 4x longer than those after it, so
    # error-norm maxima surviving the reset would loosen the certificate and change the statistics; a slack of 2
    # candidates keeps the certificate tight enough for the statistics to see that.
    d, k, slack = 256, 10, 2
    x, q, premise, _ = sb.make_regime("anisotropic", 300, 4000, d, k=k, seed=41)
    premise()
    qd = torch.from_numpy(q).cuda()
    big = 4 * x[:2500]
    small = x[2500:]
    lib = om.lib.load()
    idx = om.index.FlatIPIndex(d)
    idx.set_param("rescore_slack", slack)
    held = []

    def host_f32(rows):
        idx.add(rows)
        return rows

    def device(rows, dt):
        t = torch.from_numpy(rows).cuda().to(dt)
        idx.add(t)
        return t.float().cpu().numpy()

    def host_half(rows, dt, code):  # FlatIPIndex.add upcasts host data: call the C ABI for its bf16 / fp16 host path
        t = torch.from_numpy(rows).to(dt).contiguous()
        om.lib.check(lib.om_index_add(idx._h, ctypes.c_void_p(t.data_ptr()), om.lib.OM_HOST, code, t.shape[0],
                                      om.lib.current_stream_ptr()))
        return t.float().numpy()

    def reserve_commit(rows):
        view = idx.reserve_rows(rows.shape[0])
        view.copy_(torch.from_numpy(rows).cuda())
        idx.commit_rows(rows.shape[0])
        return rows

    steps = [("host f32 x1", lambda: host_f32(big[0:1])),
             ("host f32 x100", lambda: host_f32(big[1:101])),
             ("device bf16 x300", lambda: device(big[101:401], torch.bfloat16)),
             ("device f16 x300", lambda: device(big[401:701], torch.float16)),
             ("host bf16 x200", lambda: host_half(big[701:901], torch.bfloat16, om.lib.OM_BF16)),
             ("host f16 x200", lambda: host_half(big[901:1101], torch.float16, om.lib.OM_F16)),
             ("reserve/commit x600 (grows)", lambda: reserve_commit(big[1101:1701])),
             ("reset", None),
             ("device f32 x700", lambda: device(small[:700], torch.float32)),
             ("reserve/commit x50", lambda: reserve_commit(small[700:750]))]
    bases = []  # device address of row 0: changes when the index grows
    for name, step in steps:
        if step is None:
            idx.reset()
            held = []
        else:
            held.append(step())
        rows = np.concatenate(held) if held else np.zeros((0, d), np.float32)
        assert idx.ntotal == rows.shape[0], name
        bases.append(idx.reserve_rows(0).data_ptr() - rows.shape[0] * d * 4)
        if rows.shape[0]:
            _same(idx.master_rows().cpu(), torch.from_numpy(rows), name + ": master rows")
        fresh = om.index.FlatIPIndex(d)
        fresh.set_param("rescore_slack", slack)
        if rows.shape[0]:
            fresh.add(rows)
        got, want = _search_all(idx, qd, k), _search_all(fresh, qd, k)
        print("[state] %-28s n=%5d stats %s" % (name, rows.shape[0], [want[nq][2] for nq in want]))
        _same_search(got, want, name)
    assert bases[6] != bases[5], "premise: the reserve / commit step must grow the index"
    assert 0 < want[300][2][0] < 300, "premise: the certificate must be tight (uncertified %d of 300)" % want[300][2][0]


# ---------------------------------------------------------------------------------------------------------------------
# poisoned allocations
# ---------------------------------------------------------------------------------------------------------------------
# Filling device memory from outside and releasing it does not work: on the H100 the driver hands every cudaMalloc
# zero-filled pages.  OPENMATCH_B200_POISON_ALLOC=1 makes the library fill its own fresh buffers with 0xFF bytes instead.
POISON_GEOMS = [(32, 11), (100, 7), (256, 3)]  # attn_kernel with 4 and 1 sequences per tile, attn_stream_kernel


@pytest.fixture(scope="module")
def poisoned(om):
    """Reference results on handles with zero-filled allocations, then the same handles created with every library
    allocation poisoned; the poison stays on for the test, which allocates the search workspace."""
    gen = torch.Generator().manual_seed(51)
    sd = _rand_bert_sd(gen, 2, 256, 512, 1000, 512)
    inputs = [_enc_inputs(gen, L, B, "hole", 1000) for L, B in POISON_GEOMS]
    x, q, _, _ = sb.make_regime("anisotropic", 300, 6000, 256, k=10, seed=52)
    xd, qd = torch.from_numpy(x).cuda(), torch.from_numpy(q).cuda()
    ref_enc = [_encoder(om, BERT, sd).encode(*i, return_hidden=True) for i in inputs]
    idx = om.index.FlatIPIndex(256)
    idx.add(xd)
    ref_search = _search_all(idx, qd)
    torch.cuda.synchronize()
    os.environ["OPENMATCH_B200_POISON_ALLOC"] = "1"
    try:
        probe = om.index.FlatIPIndex(256)
        yield dict(inputs=inputs, ref_enc=ref_enc, xd=xd, qd=qd, ref_search=ref_search, view=probe.reserve_rows(6000),
                   enc=_encoder(om, BERT, sd), idx=om.index.FlatIPIndex(256))
    finally:
        del os.environ["OPENMATCH_B200_POISON_ALLOC"]


def test_poisoned_allocations(om, poisoned):
    p = poisoned
    assert torch.isnan(p["view"]).all(), "premise: the library's fresh allocations must hold the NaN poison"
    for (L, B), i, (want_h, want) in zip(POISON_GEOMS, p["inputs"], p["ref_enc"]):
        got_h, got = p["enc"].encode(*i, return_hidden=True)
        _same(got, want, "reps on poisoned workspace (L=%d B=%d)" % (L, B))
        _same(got_h, want_h, "hidden states on poisoned workspace (L=%d B=%d)" % (L, B))
    idx = p["idx"]
    idx.add(p["xd"])  # rows beyond ntotal, up to the capacity, keep the poison
    _same_search(_search_all(idx, p["qd"]), p["ref_search"], "search on poisoned workspace")
