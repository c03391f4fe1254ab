"""CPU: decoding with a key / value cache (MultiHeadAttentionWithCache, TransformerDecoderLayer, TransformerDecoder).

* A plain-torch fp32 restatement of the reference forward reproduces tests/golden/decoder_cache_golden.pt (recorded from
  the unmodified reference) to 1e-5: the goldens and the cases mean what they say.
* The package's Python schedule (engine_layers.py), run on the emulated kernels of tests/emu_ops.py and
  tests/emu_decode_ops.py, reproduces them at bf16 tolerance: projection routing, cache layout and dtypes, masks, and
  the reference's quirks (cross_attention_mask dropped by TransformerDecoder, empty lists when nothing is requested,
  pre-norm without encoder states).
* mmb_attention_decode_splits covers the keys, is >= 1 and depends on its arguments alone.
* ptxas: the decode, combine and append kernels build for sm_90a without spills at their planned occupancy.
"""
import ctypes
import math
import os
import re
import shutil
import subprocess
import tempfile

import pytest
import torch
import torch.nn.functional as F

import decoder_cache_cases as DC
import emu_decode_ops
import emu_ops
from multimodal_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "multimodal_b200", "csrc", "attention_decode.cu")


@pytest.fixture(scope="module")
def gold():
    return torch.load(os.path.join(ROOT, "tests", "golden", "decoder_cache_golden.pt"), map_location="cpu",
                      weights_only=False)


def _ours():
    from multimodal_b200.modules.layers import multi_head_attention, transformer

    return DC.namespace(multi_head_attention, transformer)


# ---- plain fp32 restatement of the reference forward -------------------------------------------------------------
def _lin(x, lin):
    return F.linear(x, lin.weight, lin.bias)


def _ln(x, ln):
    return F.layer_norm(x.float(), ln.normalized_shape, ln.weight, ln.bias, ln.eps)


def r_mha(m, q, k, v, attn_mask=None, past=None, is_causal=False):
    B, Sq, d = q.shape
    H = m.num_heads
    hd = d // H
    Q = _lin(q, m.q_proj).view(B, -1, H, hd).transpose(1, 2)
    K = _lin(k, m.k_proj).view(B, -1, H, hd).transpose(1, 2)
    V = _lin(v, m.v_proj).view(B, -1, H, hd).transpose(1, 2)
    if past is not None:
        K, V = torch.cat([past[0], K], 2), torch.cat([past[1], V], 2)
    s = (Q @ K.transpose(-1, -2).to(Q.dtype)) / math.sqrt(hd)
    if attn_mask is not None:
        s = s.masked_fill(~attn_mask, float("-inf"))
    if is_causal:
        s = s.masked_fill(~torch.ones(Sq, K.shape[2], dtype=torch.bool).tril(), float("-inf"))
    o = (torch.softmax(s, -1) @ V.to(Q.dtype)).transpose(1, 2).reshape(B, Sq, d)
    return _lin(o, m.output_proj), (K, V)


def r_layer(m, x, enc=None, attention_mask=None, past=None):
    def mlp(h):
        seq = m.feedforward.model
        return _lin(F.gelu(_lin(h, seq[0])), seq[-1])

    if m.norm_first:
        a, kv = r_mha(m.attention, *([_ln(x, m.attention_layernorm)] * 3), attention_mask, past)
        h = a + x
        if m.use_cross_attention and enc is not None:
            h = r_mha(m.cross_attention, _ln(h, m.cross_attention_layernorm), enc, enc)[0] + h
        return h + mlp(_ln(h, m.feedforward_layernorm)), kv
    a, kv = r_mha(m.attention, x, x, x, attention_mask, past)
    h = _ln(a + x, m.attention_layernorm)
    if m.use_cross_attention:
        h = _ln(r_mha(m.cross_attention, h, enc, enc)[0] + h, m.cross_attention_layernorm)
    return _ln(h + mlp(h), m.feedforward_layernorm), kv


def r_run(m, name, inp):
    c = DC.CASES[name]
    if c["kind"] == "mha":
        out, (k, v) = r_mha(m, inp["query"], inp["key"], inp["value"], inp.get("attn_mask"), inp.get("past_key_value"),
                            inp.get("is_causal", False))
        return {"out": out, "k": k, "v": v} if c["use_cache"] else {"out": out}
    if c["kind"] == "layer":
        out, (k, v) = r_layer(m, inp["hidden_states"], inp.get("encoder_hidden_states"), inp.get("attention_mask"),
                              inp["past_key_value"])
        return {"out": out, "k": k, "v": v}
    x, res = inp["hidden_states"], {}
    for i, layer in enumerate(m.layer):
        res[f"hidden{i}"] = x
        x, (res[f"k{i}"], res[f"v{i}"]) = r_layer(layer, x, inp.get("encoder_hidden_states"), inp["attention_mask"],
                                                  inp["past_key_values"][i])
    res[f"hidden{len(m.layer)}"] = x
    res["out"] = _ln(x, m.final_layer_norm)
    return res


@pytest.mark.parametrize("name", list(DC.CASES))
def test_restatement_matches_reference_golden(gold, name):
    g = gold[name]
    m = DC.build(_ours(), name)
    assert sorted(m.state_dict()) == g["keys"]
    with torch.no_grad():
        res = r_run(m, name, g["inputs"])
    assert sorted(res) == sorted(g["results"])
    for k, ref in g["results"].items():
        assert res[k].dtype == ref.dtype and res[k].shape == ref.shape, k
        assert (res[k] - ref).abs().max().item() <= 1e-5, (name, k)


# ---- the package's schedule on emulated kernels -------------------------------------------------------------------
@pytest.fixture
def emulated(monkeypatch):
    from multimodal_b200 import engine_layers

    emu_ops.install(monkeypatch)
    emu_decode_ops.install(monkeypatch)
    monkeypatch.setattr(engine_layers, "_cuda", lambda t, what: None)


def _close(a, b, tol=2e-2):
    return (a.float() - b.float()).abs().max().item() <= tol * max(b.float().abs().max().item(), 1e-6)


@pytest.mark.parametrize("name", list(DC.CASES))
def test_schedule_on_emulated_kernels_matches_golden(gold, emulated, name):
    g = gold[name]
    m = DC.build(_ours(), name)
    inp = g["inputs"]
    with torch.no_grad():
        res = DC.run(m, name, inp)
    assert sorted(res) == sorted(g["results"])
    for k, ref in g["results"].items():
        assert res[k].dtype == ref.dtype and res[k].shape == ref.shape, (name, k, res[k].dtype, res[k].shape)
        assert _close(res[k], ref), (name, k)
    c = DC.CASES[name]
    if c.get("use_cache") or c["kind"] != "mha":
        for k, v in res.items():
            if k[0] in "kv" and k != "out":
                # the cache is the [B, H, S, hd] view of a row-major [B, S, H*hd] buffer, fresh on every call
                B, H, S, hd = v.shape
                assert v.stride() == (S * H * hd, hd, H * hd, 1), (k, v.stride())
                assert all(v.data_ptr() != t.data_ptr() for t in _tensors(inp))


def _tensors(x):
    if torch.is_tensor(x):
        return [x]
    if isinstance(x, dict):
        return [t for v in x.values() for t in _tensors(v)]
    if isinstance(x, (list, tuple)):
        return [t for v in x for t in _tensors(v)]
    return []


def test_goldens_keep_shared_inputs_shared(gold):
    """query is key is value (self-attention) selects the packed projections; the fixture keeps that identity."""
    inp = gold["mha_self_past_d64"]["inputs"]
    assert inp["query"] is inp["key"] is inp["value"]
    inp = gold["mha_cross_d96"]["inputs"]
    assert inp["key"] is inp["value"] and inp["key"] is not inp["query"]


def test_quirks_and_errors(emulated):
    ns = _ours()
    m = DC.build(ns, "layer_post_cross_d128")
    x = torch.randn(1, 2, 256)
    with torch.no_grad(), pytest.raises(ValueError, match="encoder_hidden_states"):
        m(x)   # post-norm with cross-attention needs encoder states (the pre-norm layer skips the block instead)
    dec = DC.build(ns, "decoder_2l_d96")
    with torch.no_grad():
        o = dec(torch.randn(1, 2, 384), torch.randn(1, 3, 128))
    assert o.hidden_states == [] and o.current_key_values == []
    mha = DC.build(ns, "mha_cross_d96")
    with torch.no_grad():
        with pytest.raises(ValueError, match="same bsz"):
            mha(torch.randn(2, 1, 384), torch.randn(3, 4, 80), torch.randn(3, 4, 80))
        enc = torch.randn(1, 4, 80)
        with pytest.raises(NotImplementedError, match="boolean"):
            mha(torch.randn(1, 1, 384), enc, enc, attn_mask=torch.zeros(1, 4))
        with pytest.raises(NotImplementedError, match="per-head"):
            mha(torch.randn(1, 1, 384), enc, enc, attn_mask=torch.ones(1, 2, 1, 4, dtype=torch.bool))
    mha.dropout = 0.1
    mha.train()
    with torch.no_grad(), pytest.raises(NotImplementedError, match="dropout"):
        mha(torch.randn(1, 1, 384), enc, enc)
    mha.eval()
    with torch.no_grad():
        mha(torch.randn(1, 1, 384), enc, enc)   # dropout only matters in training mode


def test_forward_only_guard_under_grad_mode(emulated):
    from multimodal_b200._lib import MMBError

    mha = DC.build(_ours(), "mha_cross_d96")
    enc = torch.randn(1, 4, 80)
    with pytest.raises(MMBError, match="forward values only"):
        mha(torch.randn(1, 1, 384), enc, enc)


# ---- split count ----------------------------------------------------------------------------------------------------
def test_decode_splits_cover_the_keys_and_depend_on_the_shape_alone():
    lib = ctypes.CDLL(str(_lib.LIB_PATH))
    f = lib.mmb_attention_decode_splits
    f.restype, f.argtypes = ctypes.c_int, [ctypes.c_int] * 3
    src = open(SRC).read()
    const = {n: int(re.search(rf"constexpr int {n} = (\d+);", src).group(1))
             for n in ("DEC_BN", "DEC_MIN_BLOCKS_PER_SPLIT", "DEC_TARGET_CTAS", "DEC_MAX_SPLITS")}
    for B in (1, 2, 8, 32, 64, 1000):
        for H in (1, 8, 12, 16):
            for Skv in (1, 63, 64, 65, 77, 255, 256, 257, 1000, 4096, 4097, 65536, 10 ** 6):
                n = f(B, H, Skv)
                assert n == f(B, H, Skv) and 1 <= n <= const["DEC_MAX_SPLITS"]
                nblk = -(-Skv // const["DEC_BN"])
                per = -(-nblk // n)
                assert (n - 1) * per < nblk <= n * per, (B, H, Skv, n)     # every split holds a block, all blocks held
                if n > 1:
                    assert per >= const["DEC_MIN_BLOCKS_PER_SPLIT"] or nblk // n < const["DEC_MIN_BLOCKS_PER_SPLIT"] + 1
                    assert B * H * (n - 1) < const["DEC_TARGET_CTAS"] + B * H
    assert f(1, 12, 4096) == 16 and f(64, 12, 4096) == 1 and f(1, 12, 77) == 1
    assert f(0, 12, 64) == -22 and f(1, 12, 0) == -22


def test_decode_rejects_long_queries_and_misaligned_operands():
    lib = ctypes.CDLL(str(_lib.LIB_PATH))
    vp, ll, i32 = ctypes.c_void_p, ctypes.c_longlong, ctypes.c_int
    f = lib.mmb_attention_fwd_decode
    f.restype = i32
    f.argtypes = [vp, ll, ll, vp, ll, ll, vp, ll, ll, vp, ll, ll, vp, ll, ll, i32, i32, i32, i32, i32, i32,
                  ctypes.c_float, vp]
    q, k, v, o = 0x10000, 0x20000, 0x30000, 0x40000   # never dereferenced: every call below is refused before a launch
    args = lambda q=q, o=o, Sq=1, D=64: (q, 128, 128, k, 128, 128 * 100, v, 128, 128 * 100, o, 128, 128, None, 0, 0,
                                         1, Sq, 100, 2, D, 0, 0.125, None)
    assert f(*args(Sq=17)) == -95
    assert f(*args(D=80)) == -95
    assert f(*args(q=q + 8)) == -22 and f(*args(o=o + 2)) == -22


# ---- ptxas -----------------------------------------------------------------------------------------------------------
def _nvcc():
    p = shutil.which("nvcc")
    if p is None and os.path.exists("/usr/local/cuda/bin/nvcc"):
        p = "/usr/local/cuda/bin/nvcc"
    return p


@pytest.mark.skipif(_nvcc() is None, reason="nvcc not installed")
def test_decode_kernels_no_spills_and_planned_occupancy():
    with tempfile.TemporaryDirectory() as td:
        cmd = [_nvcc(), *_lib.NVCC_FLAGS, "-Xptxas", "-v", "-I", os.path.join(ROOT, "multimodal_b200", "csrc"),
               "-I", os.path.join(ROOT, "include"), "-c", SRC, "-o", os.path.join(td, "attention_decode.o")]
        out = subprocess.run(cmd, capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-2000:]
    log = out.stdout + out.stderr
    props = re.findall(r"Function properties for (\S+)\s*\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads", log)
    assert len(props) >= 6
    for fn, st, ld in props:
        assert int(st) == 0 and int(ld) == 0, (fn, st, ld)
    src = open(SRC).read()
    const = lambda n: int(re.search(rf"constexpr int {n} = (\d+);", src).group(1))
    seen = set()
    for block in log.split("Compiling entry function '")[1:]:
        fn = block.split("'", 1)[0]
        regs = int(re.search(r"Used (\d+) registers", block).group(1))
        m = re.search(r"attn_fwd_decode_kernelILi(\d+)E", fn)
        if m:
            D = int(m.group(1))
            threads = 32 * const(f"DEC_WARPS_D{D}")
            budget = 65536 // (threads * const(f"DEC_CTAS_PER_SM_D{D}"))
            assert regs <= min(budget, 255), (fn, regs, budget)
            # shared memory: 16 query rows + per warp DEC_STAGES stages of 64 K and 64 V rows, 2*D + 16 bytes each
            smem = 16 * (2 * D + 16) + const(f"DEC_WARPS_D{D}") * (2 * const("DEC_STAGES") * 64 * (2 * D + 16) + 16)
            assert smem * const(f"DEC_CTAS_PER_SM_D{D}") <= 228 * 1024, (D, smem)
            seen.add(D)
        else:
            assert regs <= 64, (fn, regs)   # combine / append: 256-thread (or 128) grids, full occupancy
    assert seen == {64, 96, 128}
