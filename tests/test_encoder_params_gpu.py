"""The parameter contract of om_encoder_set_weight / om_encoder_finalize, through the C ABI: the names a handle takes
(exactly, with or without the "bert." / "roberta." prefix), the ones it ignores (return value 1) or refuses, the
missing-parameter message of finalize, and that a finalized handle takes no more weights and keeps encoding the same
reps."""
import ctypes

import pytest
import torch

from openmatch_b200 import synthetic

pytestmark = pytest.mark.gpu

H, F, HEAD_OUT = 128, 256, 16
SPECS = {
    "bert": dict(arch="bert", layers=2, hidden=H, heads=2, ffn=F, vocab=1200, max_pos=128, type_vocab=2, ln_eps=1e-12),
    "hd32": dict(arch="bert", layers=2, hidden=H, heads=4, ffn=F, vocab=1200, max_pos=128, type_vocab=2, ln_eps=1e-12),
    "roberta": dict(arch="roberta", layers=2, hidden=H, heads=2, ffn=F, vocab=1200, max_pos=130, type_vocab=1,
                    ln_eps=1e-5),
    "t5": dict(arch="t5", layers=2, hidden=H, heads=2, ffn=F, vocab=1200, ln_eps=1e-6, rel_buckets=32,
               rel_max_distance=128),
}
OM_ESTATE, OM_EINVAL = -5, -1


@pytest.fixture(scope="module")
def lib():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from openmatch_b200 import _lib
    return _lib.load()


@pytest.fixture
def make(lib):
    """make(kind, head) -> a fresh handle, destroyed at teardown"""
    from openmatch_b200 import _lib
    from openmatch_b200.encoder import _ARCHS
    handles = []

    def make_(kind, head=False):
        s = SPECS[kind]
        desc = _lib.EncoderDesc(arch=_ARCHS[s["arch"]], layers=s["layers"], hidden=s["hidden"], heads=s["heads"],
                                ffn=s["ffn"], vocab=s["vocab"], max_pos=s.get("max_pos", 0),
                                type_vocab=s.get("type_vocab", 0), ln_eps=s["ln_eps"], pooling=_lib.OM_POOL_FIRST,
                                has_head=int(head), head_out=HEAD_OUT if head else 0, normalize=0, rel_buckets=32,
                                rel_max_distance=128, max_batch_tokens=1024)
        h = ctypes.c_void_p()
        assert lib.om_encoder_create(ctypes.byref(desc), ctypes.byref(h)) == 0
        handles.append(h)
        return h

    yield make_
    for h in handles:
        lib.om_encoder_destroy(h)


def _state_dict(kind, seed=0):
    s = SPECS[kind]
    return synthetic.t5_state_dict(s, seed) if s["arch"] == "t5" else synthetic.bert_state_dict(s, seed)


def _set(lib, h, name, t):
    """-> (return code, error message when negative)"""
    from openmatch_b200 import _lib
    t = t.detach().to(torch.float32).contiguous()
    shape = (ctypes.c_int64 * t.dim())(*t.shape)
    rc = lib.om_encoder_set_weight(h, name.encode(), t.data_ptr(), _lib.OM_HOST, shape, t.dim())
    return rc, lib.om_last_error().decode() if rc < 0 else ""


def _load(lib, h, sd, prefix=""):
    for name, t in sd.items():
        assert _set(lib, h, prefix + name, t) == (0, ""), name


def _finalize(lib, h):
    rc = lib.om_encoder_finalize(h)
    return rc, lib.om_last_error().decode() if rc < 0 else ""


def _encode(lib, h):
    """reps of a fixed padded batch (4 x 64, ragged mask) through om_encode"""
    g = torch.Generator().manual_seed(7)
    ids = torch.randint(2, SPECS["bert"]["vocab"], (4, 64), generator=g)
    mask = torch.ones(4, 64, dtype=torch.int64)
    for b, n in enumerate((64, 40, 17, 3)):
        mask[b, n:] = 0
    ids, mask = ids.cuda(), mask.cuda()
    out = torch.empty(4, lib.om_encoder_rep_dim(h), dtype=torch.float32, device="cuda")
    assert lib.om_encode(h, ids.data_ptr(), mask.data_ptr(), None, 4, 64, out.data_ptr(), 0, out.stride(0), None,
                         torch.cuda.current_stream().cuda_stream) == 0, lib.om_last_error()
    torch.cuda.synchronize()
    assert torch.isfinite(out).all()
    return out.cpu()


@pytest.mark.parametrize("kind,prefix", [("bert", ""), ("bert", "bert."), ("hd32", ""), ("roberta", ""),
                                         ("roberta", "roberta."), ("t5", "")])
def test_every_parameter_is_accepted(lib, make, kind, prefix):
    h = make(kind, head=True)
    sd = _state_dict(kind)
    if kind == "t5":  # T5EncoderModel's name of the tied embedding
        sd["encoder.embed_tokens.weight"] = sd.pop("shared.weight")
    _load(lib, h, sd, prefix)
    head_name = "linear.weight" if kind == "t5" else "head.linear.weight"  # LinearHead's own state_dict name, or ours
    assert _set(lib, h, head_name, torch.randn(HEAD_OUT, H) * 0.1) == (0, "")
    assert _finalize(lib, h) == (0, "")
    assert _encode(lib, h).shape == (4, HEAD_OUT)


@pytest.mark.parametrize("kind,head,name,shape", [
    ("bert", False, "pooler.dense.weight", (H, H)),
    ("bert", False, "bert.pooler.dense.bias", (H,)),
    ("roberta", False, "roberta.pooler.dense.weight", (H, H)),
    ("bert", False, "head.linear.weight", (HEAD_OUT, H)),
    ("t5", False, "linear.weight", (HEAD_OUT, H)),
    ("bert", False, "encoder.layer.2.attention.self.query.weight", (H, H)),
    ("bert", True, "encoder.layer.9.output.dense.bias", (H,)),
    ("bert", False, "encoder.block.0.layer.0.SelfAttention.q.weight", (H, H)),
    ("t5", False, "encoder.block.1.layer.0.SelfAttention.relative_attention_bias.weight", (32, 2)),
    ("t5", False, "encoder.block.2.layer.0.SelfAttention.q.weight", (H, H)),
    ("t5", False, "encoder.block.2.layer.1.DenseReluDense.wi_0.weight", (F, H)),
    ("t5", False, "decoder.block.0.layer.0.SelfAttention.q.weight", (H, H)),
    ("t5", False, "encoder.layer.0.attention.self.query.weight", (H, H)),
])
def test_ignored_names_return_1(lib, make, kind, head, name, shape):
    assert _set(lib, make(kind, head), name, torch.randn(*shape)) == (1, "")


@pytest.mark.parametrize("kind,head,name,shape", [
    ("bert", False, "embeddings.word_embeddings.weight", (1200, H + 1)),
    ("bert", False, "bert.encoder.layer.1.attention.self.key.weight", (H, 64)),
    ("bert", False, "encoder.layer.0.attention.self.value.bias", (1, H)),
    ("hd32", False, "encoder.layer.1.intermediate.dense.weight", (H, F)),
    ("roberta", False, "roberta.embeddings.position_embeddings.weight", (128, H)),
    ("bert", True, "head.linear.weight", (HEAD_OUT + 1, H)),
    ("t5", False, "encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight", (2, 32)),
    ("t5", False, "encoder.block.1.layer.1.DenseReluDense.wo.weight", (F, H)),
    ("t5", True, "linear.weight", (H,)),
])
def test_wrong_shape_names_the_parameter(lib, make, kind, head, name, shape):
    rc, msg = _set(lib, make(kind, head), name, torch.randn(*shape))
    assert rc == OM_EINVAL and "'%s'" % name in msg, msg


@pytest.mark.parametrize("name", ["encoder.block.0.layer.1.DenseReluDense.wi_0.weight",
                                  "encoder.block.1.layer.1.DenseReluDense.wi_1.weight"])
def test_gated_t5_is_refused(lib, make, name):
    rc, msg = _set(lib, make("t5"), name, torch.randn(F, H))
    assert rc == OM_EINVAL and "gated" in msg, msg


@pytest.mark.parametrize("kind,head,drop,listed", [
    ("bert", True, ["encoder.layer.1.attention.self.key.weight", "embeddings.LayerNorm.bias",
                    "encoder.layer.0.intermediate.dense.bias"],
     "4 parameter(s) missing: embeddings.LayerNorm.bias, encoder.layer.0.intermediate.dense.bias, "
     "encoder.layer.1.attention.self.key.weight, head.linear.weight"),
    ("roberta", False, ["encoder.layer.1.output.LayerNorm.bias", "encoder.layer.0.attention.self.value.bias",
                        "embeddings.word_embeddings.weight", "encoder.layer.0.attention.output.dense.weight",
                        "encoder.layer.0.attention.self.query.weight"],
     "5 parameter(s) missing: embeddings.word_embeddings.weight, encoder.layer.0.attention.self.query.weight, "
     "encoder.layer.0.attention.self.value.bias, encoder.layer.0.attention.output.dense.weight, ..."),
    ("t5", True, ["encoder.block.1.layer.1.layer_norm.weight",
                  "encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight", "shared.weight"],
     "4 parameter(s) missing: shared.weight, encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight, "
     "encoder.block.1.layer.1.layer_norm.weight, head.linear.weight"),
])
def test_missing_parameters_are_listed_in_order(lib, make, kind, head, drop, listed):
    h = make(kind, head)
    sd = _state_dict(kind)
    _load(lib, h, {k: v for k, v in sd.items() if k not in drop})
    assert _finalize(lib, h) == (OM_ESTATE, "om_encoder_finalize: " + listed)
    # the handle is still open: supplying what was missing makes finalize succeed
    _load(lib, h, {k: sd[k] for k in drop})
    if head:
        assert _set(lib, h, "head.linear.weight", torch.randn(HEAD_OUT, H) * 0.1) == (0, "")
    assert _finalize(lib, h) == (0, "")
    _encode(lib, h)


@pytest.mark.parametrize("kind", ["bert", "t5"])
def test_second_finalize_is_refused(lib, make, kind):
    h = make(kind)
    _load(lib, h, _state_dict(kind))
    assert _finalize(lib, h)[0] == 0
    want = _encode(lib, h)
    assert _finalize(lib, h)[0] == OM_ESTATE
    assert torch.equal(_encode(lib, h), want)


@pytest.mark.parametrize("kind,names", [
    ("bert", ["encoder.layer.0.attention.self.query.weight", "encoder.layer.1.output.dense.bias",
              "embeddings.word_embeddings.weight", "pooler.dense.weight"]),
    ("t5", ["encoder.block.0.layer.1.DenseReluDense.wi.weight", "encoder.final_layer_norm.weight",
            "encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight", "decoder.final_layer_norm.weight"]),
])
def test_set_weight_after_finalize_is_refused(lib, make, kind, names):
    """a finalized handle has folded its weights: a later set_weight (known name or not) changes nothing and the handle
    stays finalized"""
    h = make(kind)
    sd = _state_dict(kind)
    _load(lib, h, sd)
    assert _finalize(lib, h)[0] == 0
    want = _encode(lib, h)
    for name in names:
        t = torch.randn(*sd[name].shape) if name in sd else torch.randn(H)
        rc, msg = _set(lib, h, name, t)
        assert rc == OM_ESTATE and "after om_encoder_finalize" in msg, (name, rc, msg)
    assert torch.equal(_encode(lib, h), want)
    assert _finalize(lib, h)[0] == OM_ESTATE


@pytest.mark.parametrize("name,width", [("encoder.layer.0.attention.self.query.foo", H),
                                        ("encoder.layer.1.output.LayerNorm.gamma", H),
                                        ("bert.encoder.layer.0.intermediate.dense.beta", F)])
def test_inexact_name_is_ignored(lib, make, name, width):
    """names are matched exactly: a name that only shares a module prefix with a parameter uploads nothing"""
    sd = _state_dict("bert")
    ref, h = make("bert"), make("bert")
    _load(lib, ref, sd)
    _load(lib, h, sd)
    assert _set(lib, h, name, torch.randn(width) + 3.0) == (1, "")
    assert _finalize(lib, ref)[0] == 0 and _finalize(lib, h)[0] == 0
    assert torch.equal(_encode(lib, h), _encode(lib, ref))
