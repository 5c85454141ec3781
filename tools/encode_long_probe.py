"""Probe (not part of the product): sequences of 513 - 8192 tokens on the CUDA encoder at bge-m3 shape.

  python tools/encode_long_probe.py e2e [rounds] [out.json]    end to end against eager HF
  python tools/encode_long_probe.py attn [rounds] [out.json]   the attention kernel against SDPA's flash backend
  python tools/encode_long_probe.py libs ROUNDS OUT.json NAME=LIB ...   129 - 512 tokens: libraries against each other

Model: a randomly initialised XLMRobertaModel with bge-m3's shape (24 layers, hidden 1024, 16 x 64-wide heads, FFN 4096,
vocab 250 002, max_position_embeddings 8194), CLS pooling + normalise (bge-m3's dense representation).  Workloads:
  4x8192   four sequences of 8192 tokens
  docmix   document lengths uniform in [513, 8192], about 32 k tokens in all (seed 7)
e2e: om_encode_packed (CudaEncoder.encode_packed) against HF in bf16 autocast with SDPA attention on the right-padded
batch (pad id 1), in documents/s and tokens/s, and the max rel-L2 of the reps between the two; then the share of
pool_packed_kernel in a mean-pooled encode of each workload (torch.profiler).
attn: the device time of attn_stream_kernel per layer at 4x8192 (torch.profiler, one encode after a warm-up) and
scaled_dot_product_attention on [4, 16, 8192, 64] bf16 tensors with the flash backend forced (CUDA events), each as
TFLOP/s from 4 L^2 dh per head and sequence.
libs: sequences of 129 - 512 tokens on libopenmatch_b200.so builds against each other, each loaded in processes of its
own (OPENMATCH_B200_LIB), the libraries alternating A B A B (two processes each).  Shapes (randomly initialised, 32 k
tokens each): bert-base padded 128x256, 85x384, 64x512 and packed lengths uniform in [129, 512] (seed 11); t5-base
(GTR: mean pooling) padded 64x512 and the same packed mix; a MiniLM-L12 shape (hidden 384, 12 x 32-wide heads) padded
64x512.  A process times ROUNDS encodes of each shape after a warm-up (CUDA events), then takes the device time of its
long-sequence attention kernel over one encode (torch.profiler, per layer: attn_stream_kernel, or attn_long_kernel,
which took the 129 - 512-token sequences in builds before attn_stream_kernel did).  Reported per library and shape: the
median over all its rounds, the medians of its two processes (their difference is the run-to-run spread), and the max
rel-L2 of its reps against the first library's.
After a warm-up every round times each contender once, the order rotating from round to round; reported are medians.
The card's name, power limit and max SM clock are read in the same process (read-only query)."""
import json
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from openmatch_b200.encoder import CudaEncoder  # noqa: E402

LAYERS, H, HEADS, F, VOCAB, MAX_POS = 24, 1024, 16, 4096, 250002, 8194


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        smi = r.stdout.strip().splitlines()[:1]
    except (OSError, subprocess.SubprocessError):
        smi = []
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": smi}


def workloads():
    rng = np.random.default_rng(7)
    mix = []
    while sum(mix) < 32000:
        mix.append(int(rng.integers(513, 8193)))
    return {"4x8192": np.full(4, 8192, np.int32), "docmix": np.array(mix, np.int32)}


def model():
    from transformers import XLMRobertaConfig, XLMRobertaModel
    torch.manual_seed(0)
    cfg = XLMRobertaConfig(vocab_size=VOCAB, hidden_size=H, num_hidden_layers=LAYERS, num_attention_heads=HEADS,
                           intermediate_size=F, max_position_embeddings=MAX_POS, type_vocab_size=1, pad_token_id=1,
                           attn_implementation="sdpa")
    with torch.device("cuda"):
        return XLMRobertaModel(cfg).eval()


def batch(lens, seed=1):
    L = int(lens.max())
    ids = torch.randint(3, VOCAB, (len(lens), L), generator=torch.Generator().manual_seed(seed))
    ids[:, 0] = 0
    mask = (torch.arange(L)[None] < torch.from_numpy(lens).long()[:, None]).long()
    ids = torch.where(mask.bool(), ids, torch.ones_like(ids)).cuda()
    return ids, mask.cuda()


def timed(runs, rounds):
    names = list(runs)
    for _ in range(2):
        for n in names:
            runs[n]()
    torch.cuda.synchronize()
    times = {n: [] for n in names}
    for r in range(rounds):
        order = names[r % len(names):] + names[:r % len(names)]
        ev = {n: (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for n in names}
        for n in order:
            ev[n][0].record()
            runs[n]()
            ev[n][1].record()
        torch.cuda.synchronize()
        for n in names:
            times[n].append(ev[n][0].elapsed_time(ev[n][1]))
    return {n: (float(np.median(t)), [min(t), max(t)]) for n, t in times.items()}


def kernel_times(fn, names):
    """device time (ms) per kernel whose name contains one of `names`, over one call of fn"""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {n: 0.0 for n in names}
    total = 0.0
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        total += t
        for n in names:
            if n in e.key:
                out[n] += t / 1e3
    out["all_kernels"] = total / 1e3
    return out


def e2e(rounds):
    lm = model()
    enc = CudaEncoder.from_hf(lm, pooling="first", normalize=True)
    enc_mean = CudaEncoder.from_hf(lm, pooling="mean", normalize=True)
    records = []
    for name, lens in workloads().items():
        ids, mask = batch(lens)
        tokens = ids[mask.bool()]
        outs = {}

        def hf():
            with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
                h = lm(input_ids=ids, attention_mask=mask).last_hidden_state
            outs["hf"] = torch.nn.functional.normalize(h[:, 0].float(), dim=1)

        def om():
            outs["om"] = enc.encode_packed(tokens, lens)

        t = timed({"hf_bf16_sdpa": hf, "om_encode_packed": om}, rounds)
        rel = float(((outs["om"].double() - outs["hf"].double()).norm(dim=1) / outs["hf"].double().norm(dim=1)).max())
        rec = dict(workload=name, docs=len(lens), tokens=int(lens.sum()), padded_tokens=int(ids.numel()), rounds=rounds,
                   reps_max_rel_l2_om_vs_hf=rel)
        for n, (ms, mm) in t.items():
            rec["ms_" + n] = ms
            rec["ms_minmax_" + n] = mm
            rec["docs_per_s_" + n] = len(lens) / ms * 1e3
            rec["tokens_per_s_" + n] = float(lens.sum()) / ms * 1e3
        rec["speedup_om_vs_hf"] = rec["ms_hf_bf16_sdpa"] / rec["ms_om_encode_packed"]
        enc_mean.encode_packed(tokens, lens)
        kt = kernel_times(lambda: enc_mean.encode_packed(tokens, lens), ["pool_packed_kernel", "attn_stream_kernel"])
        rec["mean_pooled_encode_kernel_ms"] = kt
        rec["pool_packed_share_of_mean_encode"] = kt["pool_packed_kernel"] / kt["all_kernels"]
        records.append(rec)
        print(json.dumps(rec), flush=True)
    return records


def attn(rounds):
    lm = model()
    enc = CudaEncoder.from_hf(lm, pooling="first", normalize=True)
    del lm
    torch.cuda.empty_cache()
    B, L, dh = 4, 8192, 64
    flop = 4.0 * L * L * dh * HEADS * B  # per layer
    lens = np.full(B, L, np.int32)
    ids, _ = batch(lens)
    tokens = ids.reshape(-1)
    enc.encode_packed(tokens, lens)
    kt = kernel_times(lambda: enc.encode_packed(tokens, lens), ["attn_stream_kernel"])
    stream_ms = kt["attn_stream_kernel"] / LAYERS
    g = torch.Generator(device="cuda").manual_seed(3)
    q, k, v = (torch.randn(B, HEADS, L, dh, device="cuda", dtype=torch.bfloat16, generator=g) for _ in range(3))
    from torch.nn.attention import SDPBackend, sdpa_kernel

    def flash():
        with sdpa_kernel(SDPBackend.FLASH_ATTENTION):
            torch.nn.functional.scaled_dot_product_attention(q, k, v)

    t = timed({"sdpa_flash": flash}, rounds)
    rec = dict(shape="[4, 16, 8192, 64] bf16", flop_per_layer=flop, rounds=rounds,
               attn_stream_ms_per_layer=stream_ms, attn_stream_tflops=flop / stream_ms / 1e9,
               sdpa_flash_ms=t["sdpa_flash"][0], sdpa_flash_ms_minmax=t["sdpa_flash"][1],
               sdpa_flash_tflops=flop / t["sdpa_flash"][0] / 1e9, encode_kernel_ms=kt)
    print(json.dumps(rec), flush=True)
    return [rec]


def libs_shapes():
    from openmatch_b200 import synthetic
    rng = np.random.default_rng(11)
    mix = []
    while sum(mix) < 32000:
        mix.append(int(rng.integers(129, 513)))
    mix = np.array(mix, np.int32)
    minilm = dict(synthetic.BERT_BASE, hidden=384, heads=12, ffn=1536)
    t5 = dict(synthetic.T5_BASE)
    bert = dict(synthetic.BERT_BASE)
    return [("bert-base", bert, "first", "padded", 128, 256), ("bert-base", bert, "first", "padded", 85, 384),
            ("bert-base", bert, "first", "padded", 64, 512), ("bert-base", bert, "first", "packed", mix, None),
            ("t5-base", t5, "mean", "padded", 64, 512), ("t5-base", t5, "mean", "packed", mix, None),
            ("minilm-l12", minilm, "first", "padded", 64, 512)]


def libs_child(rounds, out_path):
    """one process of the libs mode: every shape on the library OPENMATCH_B200_LIB names"""
    from openmatch_b200 import synthetic
    encoders, records, reps = {}, [], {}
    for model_name, spec, pooling, layout, a, b in libs_shapes():
        if model_name not in encoders:
            sd = (synthetic.t5_state_dict if spec["arch"] == "t5" else synthetic.bert_state_dict)(spec, seed=0)
            encoders[model_name] = CudaEncoder(spec, sd, pooling=pooling, normalize=True, max_batch_tokens=40960)
        enc = encoders[model_name]
        bert = spec["arch"] == "bert"
        if layout == "padded":
            ids, mask = synthetic.token_batch(a, b, spec["vocab"], seed=5, bert=bert, device="cuda")
            shape = "%s padded %dx%d" % (model_name, a, b)
            fn = lambda: enc.encode(ids, mask)  # noqa: E731
        else:
            g = torch.Generator().manual_seed(5)
            tokens = torch.randint(1000, spec["vocab"], (int(a.sum()),), generator=g).cuda()
            shape = "%s packed [129, 512] x %d" % (model_name, len(a))
            fn = lambda: enc.encode_packed(tokens, a)  # noqa: E731
        for _ in range(2):
            fn()
        ms = []
        for _ in range(rounds):
            ev = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ev[0].record()
            fn()
            ev[1].record()
            torch.cuda.synchronize()
            ms.append(ev[0].elapsed_time(ev[1]))
        kt = kernel_times(fn, ["attn_long_kernel", "attn_stream_kernel"])
        attn_ms = (kt["attn_long_kernel"] + kt["attn_stream_kernel"]) / spec["layers"]
        reps[shape] = fn().cpu()
        records.append(dict(shape=shape, tokens=int(a.sum()) if layout == "packed" else a * b,
                            encode_ms=float(np.median(ms)),
                            attn_ms_per_layer=attn_ms, encode_ms_all=ms))
    torch.save(reps, out_path + ".reps.pt")
    with open(out_path, "w") as f:
        json.dump(records, f)


def libs(rounds, named):
    """the libs mode: NAME=LIB ... each in processes of its own, alternating"""
    libs_ = [nl.split("=", 1) for nl in named]
    runs = {n: [] for n, _ in libs_}
    tmp = tempfile.mkdtemp(prefix="encode_long_probe_")
    for k in range(2):
        for n, lib in libs_:
            out = os.path.join(tmp, "%s_%d.json" % (n, k))
            env = dict(os.environ, OPENMATCH_B200_LIB=os.path.abspath(lib))
            subprocess.run([sys.executable, os.path.abspath(__file__), "libs-child", str(rounds), out], env=env,
                           check=True)
            with open(out) as f:
                runs[n].append(json.load(f))
    ref = torch.load(os.path.join(tmp, "%s_0.json.reps.pt" % libs_[0][0]))
    records = []
    for i, first in enumerate(runs[libs_[0][0]][0]):
        rec = dict(shape=first["shape"], tokens=first["tokens"], rounds_per_process=rounds)
        for n, _ in libs_:
            procs = [r[i] for r in runs[n]]
            reps = torch.load(os.path.join(tmp, "%s_0.json.reps.pt" % n))[first["shape"]].double()
            want = ref[first["shape"]].double()
            rec[n] = dict(encode_ms=float(np.median(sum((p["encode_ms_all"] for p in procs), []))),
                          encode_ms_per_process=[p["encode_ms"] for p in procs],
                          attn_ms_per_layer=float(np.median([p["attn_ms_per_layer"] for p in procs])),
                          attn_ms_per_layer_per_process=[p["attn_ms_per_layer"] for p in procs],
                          reps_max_rel_l2_vs_first=float(((reps - want).norm(dim=1) / want.norm(dim=1)).max()))
        records.append(rec)
        print(json.dumps(rec), flush=True)
    shutil.rmtree(tmp)
    return records


def main():
    mode = sys.argv[1] if len(sys.argv) > 1 else "e2e"
    if mode == "libs-child":
        libs_child(int(sys.argv[2]), sys.argv[3])
        return
    rounds = int(sys.argv[2]) if len(sys.argv) > 2 else 10
    out_path = sys.argv[3] if len(sys.argv) > 3 else None
    runs = {"e2e": lambda: e2e(rounds), "attn": lambda: attn(rounds), "libs": lambda: libs(rounds, sys.argv[4:])}
    result = {"gpu": gpu_info(), "mode": mode, "records": runs[mode]()}
    print(json.dumps(result))
    if out_path:
        os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
        with open(out_path, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
