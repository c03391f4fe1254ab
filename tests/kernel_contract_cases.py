"""Contract checks of the HBM-bound kernels (casts, im2col, token assembly, LayerNorm, embeddings, L2 norm, activations,
gathers / scatters, losses, the key / value cache) and of every other kernel the CPU emulation restates, each against a
float64 reference written from include/mmb200.h.

``check_<op>(impl, device, case)`` builds the inputs of one shape case on the CPU from a fixed seed, moves them to
`device`, calls ``impl.<op>`` and compares the results with the float64 reference.  `impl` is ``multimodal_b200.ops``
(device cuda) or the CPU emulation of tests/emu_ops.py + tests/emu_decode_ops.py (device cpu), so the same check proves
the kernel and the emulation that the CPU schedule tests trust.  Inputs the kernel reads as bf16 are bf16 before the
reference is formed.  The references never call the emulation.

Tolerance classes (each check returns its compared outputs as ``{name: Rec}`` so that two implementations can be held
against each other under the same class):
  exact  bit-exact (NaN compared by position): casts, im2col, gathers / assembly / concat / split, scatter_rows_add,
         kv_cache_append, argmax_tokens, kmask_out.  Each rounds at most once or adds once in fp32.
  bf16   bf16 outputs of fp32 math: at most 1 bf16 ulp from bf16(ref64) and at least `min_equal` (99 %) of the elements
         equal to it, which catches round-toward-zero where a relative bar does not.
  bound  fp32 results: |got - ref64| <= bound, elementwise.  For reductions the bound is k * 2^-24 * sum|terms| with k
         the length of the kernel's longest summation chain (plus the roundings of the terms), derived in each check.
         Attention outputs (also bf16) get a per-element bound built from each row's own p, |v|, |dO|, |q|, |k|
         (_attn_bh), never from a global maximum, so a late causal row whose output is small is held to its own size.
Accumulating outputs (colsum, batch_sum, dgamma / dbeta / gsum, ce accum, dmask_token, the embedding tables, dq_f32)
start from non-zero buffers, so `+=` is checked rather than `=`; attention outputs start as NaN, so an element the
kernel leaves unwritten fails.

CASES maps every checked op to its shape cases.  A case with ``"gpu": True`` is sized for the GPU (grid caps, real
vocabularies, long sequences) and is skipped by the CPU run of the emulation.
"""
import contextlib
import math

import torch

U = 2.0 ** -24          # unit roundoff of fp32
F32, BF, F64 = torch.float32, torch.bfloat16, torch.float64
H100_SMS = 132          # SM count assumed for the chain lengths when no GPU is present (H100 SXM)


# ---- reference helpers ---------------------------------------------------------------------------------------------
def rne_bf16(x: torch.Tensor) -> torch.Tensor:
    """fp32 -> bf16, round to nearest even on the bit pattern (written out, not torch's cast); NaN stays NaN."""
    x = x.to(F32).contiguous()
    b = x.view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    r = ((b + 0x7FFF + ((b >> 16) & 1)) >> 16) & 0xFFFF
    r = torch.where(torch.isnan(x), torch.full_like(r, 0x7FC0), r)
    r = torch.where(r >= 0x8000, r - 0x10000, r).to(torch.int16)
    return r.view(BF)


def d64(t: torch.Tensor) -> torch.Tensor:
    return t.detach().cpu().to(F32).to(F64)


def _sms(device) -> int:
    dev = torch.device(device)
    if dev.type == "cuda":
        return torch.cuda.get_device_properties(dev).multi_processor_count
    return H100_SMS


def _cdiv(a, b):
    return -(-a // b)


def _gen(case):
    return torch.Generator().manual_seed(1000 + case.get("seed", 0))


def _ord16(t):
    i = t.contiguous().view(torch.int16).to(torch.int32) & 0xFFFF
    return torch.where(i >= 0x8000, -(i & 0x7FFF), i)


def _bits(t):
    if t.dtype == F32:
        return t.contiguous().view(torch.int32)
    if t.dtype == BF:
        return t.contiguous().view(torch.int16)
    return t


class Rec:
    """One compared output: the value (on the CPU), its class and the class's parameter; `ratio` is the largest
    |got - ref| / bound seen (bound class only)."""

    def __init__(self, kind, got, param=None, ratio=0.0):
        self.kind, self.got, self.param, self.ratio = kind, got, param, ratio


def assert_exact(name, got, ref):
    assert got.shape == ref.shape and got.dtype == ref.dtype, (name, got.shape, got.dtype, ref.shape, ref.dtype)
    if got.is_floating_point():
        gn, rn = torch.isnan(got.float()), torch.isnan(ref.float())
        assert torch.equal(gn, rn), f"{name}: NaN positions differ"
        bad = (_bits(got) != _bits(ref)) & ~gn
    else:
        bad = got != ref
    if bad.any():
        i = bad.nonzero()[0].tolist()
        raise AssertionError(f"{name}: {int(bad.sum())} of {bad.numel()} elements differ, first at {i}: "
                             f"got {got[tuple(i)].item()!r}, want {ref[tuple(i)].item()!r}")


def assert_bf16(name, got, ref64, min_equal=0.99, err=None):
    """At most 1 bf16 ulp from bf16(ref64), and at least `min_equal` of the elements equal to it.  err (optional): an
    elementwise bound of the fp32 value's own error before the rounding; where it spans more than a bf16 ulp (a result
    formed by cancellation) the element may instead lie anywhere within 1 ulp of [bf16(ref - err), bf16(ref + err)],
    and it does not count towards the equal fraction."""
    ref = rne_bf16(ref64.to(F32))
    assert got.dtype == BF and got.shape == ref.shape, (name, got.dtype, got.shape, ref.shape)
    assert torch.equal(torch.isnan(got.float()), torch.isnan(ref.float())), f"{name}: NaN positions differ"
    og = _ord16(got)
    dist = (og - _ord16(ref)).abs()
    ok = dist <= 1
    counted = torch.ones_like(ok)
    if err is not None:
        lo, hi = _ord16(rne_bf16((ref64 - err).to(F32))), _ord16(rne_bf16((ref64 + err).to(F32)))
        ok = ok | ((og >= lo - 1) & (og <= hi + 1))
        counted = lo == hi          # the fraction counts the elements whose fp32 value resolves to one bf16 value
    eq = (dist[counted] == 0).float().mean().item() if counted.any() else 1.0
    assert bool(ok.all()), \
        f"{name}: {int((~ok).sum())} elements more than 1 bf16 ulp from the reference (max {dist[~ok].max().item()})"
    assert eq >= min_equal, f"{name}: only {eq:.4f} of the elements equal bf16(ref64) (need {min_equal})"
    return eq


def assert_bound(name, got, ref64, bound):
    err = (got.detach().cpu().to(F64) - ref64).abs()
    bound = torch.as_tensor(bound, dtype=F64).expand_as(ref64)
    bad = ~(err <= bound)
    if bad.any():
        i = bad.nonzero()[0].tolist()
        raise AssertionError(f"{name}: {int(bad.sum())} of {bad.numel()} elements outside the bound, first at {i}: "
                             f"got {got.cpu()[tuple(i)].item()!r}, "
                             f"ref {ref64[tuple(i)].item()!r}, bound {bound[tuple(i)].item():.3e}")
    pos = bound > 0
    return (err[pos] / bound[pos]).max().item() if pos.any() else 0.0


class _Out:
    def __init__(self, op=None):
        self.op, self.rec = op, {}

    def exact(self, name, got, ref):
        got = got.detach().cpu()
        assert_exact(name, got, ref)
        self.rec[name] = Rec("exact", got)

    def bf16(self, name, got, ref64, min_equal=0.99, err=None):
        got = got.detach().cpu()
        eq = assert_bf16(name, got, ref64, min_equal, err)
        self.rec[name] = Rec("bf16", got, (min_equal, err), 1.0 - eq)

    def bound(self, name, got, ref64, bound, rnd=None):
        """rnd (optional): the output's own final rounding (u * |ref| for a bf16 result), added to the bound but kept
        out of the TIGHTENED factor and of the recorded ratio, which then is the largest share of the computation's
        bound that the error beyond that rounding uses."""
        got = got.detach().cpu()
        bound = (TIGHTENED.get(f"{self.op}.{name}", 1.0) * torch.as_tensor(bound, dtype=F64)).expand_as(ref64)
        total = bound if rnd is None else bound + rnd
        r = assert_bound(name, got, ref64, total)
        if rnd is not None:
            beyond = ((got.to(F64) - ref64).abs() - rnd).clamp_min(0)
            pos = bound > 0
            r = (beyond[pos] / bound[pos]).max().item() if pos.any() else 0.0
        self.rec[name] = Rec("bound", got, total.clone(), r)


def compare_recs(name, a: Rec, b: Rec, slack=0.0, where=None):
    """Holds two implementations' results of the same check against each other under the output's class.  slack widens
    a bound where the output sums another compared output that may legitimately differ (gsum over g_bf16, the GEMM's
    colsum over D0); where (bf16 class) restricts the comparison to the elements formed from identical inputs (the
    GEMM's act(D0) where the two D0 agree: each implementation met the contract on its own D0 everywhere)."""
    assert a.kind == b.kind
    if where is not None:
        assert a.kind == "bf16"
        err = a.param[1]
        a = Rec("bf16", a.got[where], (a.param[0], None if err is None else err[where]))
        b = Rec("bf16", b.got[where])
    if a.kind == "exact":
        assert_exact(name, a.got, b.got)
    elif a.kind == "bf16":
        min_equal, err = a.param
        assert_bf16(name, a.got, b.got.to(F64), min_equal, None if err is None else 2 * err)
    else:                     # bound: both lie within the bound of the same reference
        assert_bound(name, a.got, b.got.to(F64), 2 * a.param + slack)


# Bounds tightened from measurement: where the largest |got - ref| / bound over every case, measured on an H100 80GB HBM3
# (132 SMs) for the kernel and on the CPU for the emulation, was far below the derived k * 2^-24 * sum|terms| bound (for
# attention, _attn_bh's), the bar is about 3x the larger of the two measured maxima (factor applied to the derived bound).
# Every other bound is the derived one.  The kernels' bf16 attention outputs and gradients reach 0.48 - 0.87 of theirs
# (P rounded to bf16 in rows that one key dominates), and attention_probs 0.24, so those stay derived.
TIGHTENED = {
    "sum_scale.out": 0.01,                   # measured 0.0027 (kernel and emulation: the final rounding only)
    "gemm.D": 0.42,                          # EPI_F32, every case: 0.139 kernel, 0.141 emulation
    "gemm.D_acc": 0.6,                       # EPI_F32 D += result (TMA reduce-add, split-K, direct): 0.142 / 0.197
    "gemm.colsum": 0.33,                     # 0.111 / 0.110
    "colsum_bf16.out": 0.11,                 # 0.036 / 0.036
    "ce_labels.accum": 0.11,                 # 0.036 / 0.036
    "layernorm_bwd.gsum": 0.28,              # 0.091 / 0.091
    "vit_embed_ln_fwd.mean": 0.11,           # 0.034 / 0.026
    "vit_assemble_bwd.dmask_token": 0.17,    # 0.054 / 0.054
    "bert_embed_ln_bwd.dgamma": 0.11,        # 0.034 / 0.034
    "bert_embed_ln_bwd.dbeta": 0.27,         # 0.089 / 0.067
    "bert_embed_ln_bwd.dpos": 0.2,           # 0.065 / 0.062
    "bert_embed_ln_bwd.dtype": 0.1,          # 0.033 / 0.024
    "attention_fwd.lse": 0.11,               # 0.037 / 0.025
    "attention_fwd_kmask.lse": 0.1,          # 0.033 / 0.027
    "attention_bwd_generic.dq_f32": 0.063,   # 0.021 / 0.00047
    "contrastive_ce_stats.dscale": 0.14,     # 0.046 / 0.046
    "gemm_ce_stats.sum_e": 0.16,             # 0.051 / 0.035
    "gemm_ce_stats.sum_ex": 0.16,            # 0.051 / 0.034
    "gemm_ce_stats.sum_x": 0.17,             # 0.056 / 0.022
    "gemm_ce_stats.xlabel": 0.3,             # 0.097 / 0.037
    "ce_stats_reduce.dscale": 0.12,          # 0.018 / 0.040
    "linear_cross_entropy.row_loss": 0.15,   # 0.048 / 0.048
    "linear_cross_entropy.accum": 0.1,       # 0.033 / 0.024
}
# The GEMM epilogue's QuickGELU (common.cuh quick_gelu: x / 2 (1 + tanh.approx(0.851 x))), measured in fp32 on an H100
# 80GB HBM3 over every bf16 input against float64, as a multiple of the bf16 output rounding 2^-8 |ref|: 0.0037 for
# x > -1, 0.023 for -4 < x <= -1, and up to 256 for x <= -4 (the result is 0 where tanh.approx returns -1, e.g.
# x = -9.4375).  The derived bound _act_fwd_epi_err, absolute in |x| |t| 2^-10.987, holds everywhere (largest share 0.96).


# ---- special values --------------------------------------------------------------------------------------------------
_F32_SPECIAL_BITS = [
    0x00000000, 0x80000000,                  # +-0
    0x00000001, 0x80000001, 0x00008000,      # smallest subnormals, a subnormal tie (-> 0, even)
    0x00018000, 0x007FFFFF, 0x807FFFFF,      # subnormal tie (-> up), largest subnormal (-> smallest normal)
    0x7F800000, 0xFF800000,                  # +-inf
    0x7FC00000, 0xFFC00001, 0x7F800001,      # NaNs (quiet, negative quiet, signalling)
    0x7F7F8000, 0xFF7F8000, 0x7F7FFFFF,      # ties at the top (-> +-inf), FLT_MAX (-> inf)
    0x7F7F7FFF,                              # just below the tie (-> bf16 max)
    0x3F808000, 0x3F818000, 0x3F808001, 0x3F807FFF,   # 1 + 2^-8 tie (-> 1), tie (-> up), above / below a tie
]


def f32_specials():
    b = torch.tensor([v - (1 << 32) if v >= 1 << 31 else v for v in _F32_SPECIAL_BITS], dtype=torch.int32)
    return b.view(F32)


def _with_specials(x, sp):
    k = min(len(sp), x.numel())
    x = x.clone()
    x.view(-1)[:k] = sp[:k]
    return x


ACT_SPECIALS = torch.tensor([10.0, -10.0, 0.0, -0.0, 3.0, -3.0, 1.0, -1.0], dtype=F32)


# ---- casts -------------------------------------------------------------------------------------------------------------
def check_cast_bf16(impl, device, case):
    o = _Out("cast_bf16")
    n = case["n"]
    x = _with_specials(torch.randn(n, generator=_gen(case)) * 3, f32_specials())
    out = torch.empty(n, dtype=BF, device=device)
    impl.cast_bf16(x.to(device, copy=True), out)
    o.exact("out", out, rne_bf16(x))
    return o.rec


def check_cast_f32(impl, device, case):
    """Every bf16 bit pattern but one (an odd count exercises the scalar tail), in a shuffled order."""
    o = _Out("cast_f32")
    n = case["n"]
    bits = torch.arange(-32768, 32767, dtype=torch.int32)
    bits = bits[torch.randperm(bits.numel(), generator=_gen(case))][:n]
    src = bits.to(torch.int16).view(BF)
    out = torch.empty(n, dtype=F32, device=device)
    impl.cast_f32(src.to(device, copy=True), out)
    o.exact("out", out, (bits << 16).view(F32))
    return o.rec


# ---- patch im2col --------------------------------------------------------------------------------------------------------
def check_im2col(impl, device, case):
    o = _Out("im2col")
    B, H, W, ps, ld = case["B"], case["H"], case["W"], case["ps"], case["ld"]
    K, gh, gw = 3 * ps * ps, H // ps, W // ps
    img = torch.randn(B, 3, H, W, generator=_gen(case))
    buf = torch.full((B * gh * gw, ld), -7.0, dtype=BF, device=device)
    impl.im2col(img.to(device, copy=True), ps, buf[:, :K])
    ref = img.view(B, 3, gh, ps, gw, ps).permute(0, 2, 4, 1, 3, 5).reshape(B * gh * gw, K)
    got = buf.cpu()
    o.exact("out", got[:, :K], rne_bf16(ref))
    o.exact("pad", got[:, K:], torch.full((B * gh * gw, ld - K), -7.0, dtype=BF))
    return o.rec


# ---- LayerNorm -------------------------------------------------------------------------------------------------------
def _ln_ref(x64, gamma64, beta64, eps):
    mu = x64.mean(-1, keepdim=True)
    var = ((x64 - mu) ** 2).mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + eps)
    h = (x64 - mu) * rstd
    return h * gamma64 + beta64, mu.squeeze(-1), rstd.squeeze(-1), h


def _ln_fwd_bounds(x64, gamma64, beta64, eps, nv, in_err=None):
    """Bounds of the warp-per-row forward (ln_stats): mean = (sum of 4*nv values per lane, 5 shuffle levels) / d;
    var the same over squared deviations; rstd = rsqrtf(var + eps); out = (x - mean) * rstd * gamma + beta.
    in_err: elementwise absolute error of the kernel's input relative to x64 (fp32 sums formed in the kernel)."""
    out, mu, rstd, h = _ln_ref(x64, gamma64, beta64, eps)
    d = x64.shape[-1]
    k_mean = 4 * nv + 5 + 1
    k_var = 4 * nv + 5 + 3
    ax = x64.abs().mean(-1, keepdim=True)
    b_mean = k_mean * U * ax.squeeze(-1)
    b_rstd = (k_var / 2 + 3) * U * rstd
    g = gamma64.abs()
    b_out = U * (g * h.abs() * (k_var / 2 + 6) + k_mean * g * ax * rstd[:, None] + out.abs() + beta64.abs())
    if in_err is not None:
        me = in_err.mean(-1, keepdim=True)
        b_mean = b_mean + me.squeeze(-1)
        b_rstd = b_rstd + rstd * (h.abs() * in_err).mean(-1) * rstd
        b_out = b_out + g * rstd[:, None] * (in_err + me + h.abs() * (h.abs() * in_err).mean(-1, keepdim=True))
    return out, mu, rstd, b_out, b_mean, b_rstd


def check_add_layernorm_fwd(impl, device, case):
    o = _Out("add_layernorm_fwd")
    g = _gen(case)
    M, d, eps = case["M"], case["d"], 1e-5
    rpg, gather = case.get("rpg", 0), case.get("gather")
    R = M * rpg if rpg else M
    x = torch.randn(R, d, generator=g) * 2 + 0.5
    y = (torch.randn(R, d, generator=g) * 2).to(BF)
    gamma, beta = torch.randn(d, generator=g), torch.randn(d, generator=g)
    use_x, use_y = case.get("x", True), case.get("y", True)
    row_idx = torch.randint(0, max(rpg, 1), (M,), generator=g, dtype=torch.int32) if gather == "idx" else None
    tod = lambda t: None if t is None else t.to(device, copy=True)  # noqa: E731
    x_out = torch.full((M, d), 9.0, device=device)
    ln_bf16 = torch.empty(M, d, dtype=BF, device=device)
    ln_f32 = torch.empty(M, d, device=device)
    mean, rstd = torch.empty(M, device=device), torch.empty(M, device=device)
    impl.add_layernorm_fwd(tod(x) if use_x else None, tod(y) if use_y else None, x_out, ln_bf16, ln_f32, tod(gamma),
                           tod(beta), mean, rstd, M, d, eps, row_idx=tod(row_idx), rows_per_group=rpg)
    phys = torch.arange(M) * rpg + (row_idx.long() if row_idx is not None else 0) if rpg else torch.arange(M)
    xs = torch.zeros(M, d, dtype=F64)
    if use_x:
        xs = xs + d64(x)[phys]
    if use_y:
        xs = xs + d64(y)[phys]
    xr = xs.to(F32)                      # x_out: one fp32 add; the LayerNorm normalises the stored sum
    o.exact("x_out", x_out, xr)
    out, mu, rs, b_out, b_mean, b_rstd = _ln_fwd_bounds(xr.to(F64), d64(gamma), d64(beta), eps, d // 128)
    o.bound("mean", mean, mu, b_mean)
    o.bound("rstd", rstd, rs, b_rstd)
    o.bound("ln_f32", ln_f32, out, b_out)
    o.bf16("ln_bf16", ln_bf16, out, err=b_out)
    return o.rec


def check_vit_embed_ln_fwd(impl, device, case):
    o = _Out("vit_embed_ln_fwd")
    g = _gen(case)
    B, S, d, eps = case["B"], case["S"], case["d"], 1e-5
    patch = (torch.randn(B * (S - 1), d, generator=g) * 2).to(BF)
    cls, pos = torch.randn(d, generator=g), torch.randn(S, d, generator=g) * 0.5
    gamma, beta = torch.randn(d, generator=g), torch.randn(d, generator=g)
    x0 = torch.empty(B * S, d, device=device)
    mean, rstd = torch.empty(B * S, device=device), torch.empty(B * S, device=device)
    impl.vit_embed_ln_fwd(patch.to(device, copy=True), cls.to(device, copy=True), pos.to(device, copy=True), gamma.to(device, copy=True), beta.to(device, copy=True), x0, mean,
                          rstd, B, S, d, eps)
    t = torch.cat([d64(cls).view(1, 1, d).expand(B, 1, d), d64(patch).view(B, S - 1, d)], 1) + d64(pos).view(1, S, d)
    t = t.reshape(B * S, d)
    out, mu, rs, b_out, b_mean, b_rstd = _ln_fwd_bounds(t, d64(gamma), d64(beta), eps, d // 128, in_err=U * t.abs())
    o.bound("mean", mean, mu, b_mean)
    o.bound("rstd", rstd, rs, b_rstd)
    o.bound("x0", x0, out, b_out)
    return o.rec


def _ln_bwd_grid(M, d, sms):
    nv = d // 128
    per_sm = min(1536 // (nv * 32), 24)
    return min(sms * per_sm, M)


def _ln_bwd_ref(x64, dy64, mean64, rstd64, gamma64, nv):
    """dx of the one-CTA-per-row backward and its bound.  h = (x - mean) * rstd (2 roundings), dyg = dy * gamma (1),
    s1 / s2 = row sums over 4 (thread) + 5 (shuffle) + nv (cross-warp) terms, / d;
    dx = rstd * (dyg - s1 - h * s2) (+ g_in)."""
    d = x64.shape[-1]
    h = (x64 - mean64[:, None]) * rstd64[:, None]
    dyg = dy64 * gamma64
    s1 = dyg.mean(-1, keepdim=True)
    s2 = (dyg * h).mean(-1, keepdim=True)
    dx = rstd64[:, None] * (dyg - s1 - h * s2)
    k1 = 4 + 5 + nv + 1
    k2 = 4 + 5 + nv + 4
    a1 = dyg.abs().mean(-1, keepdim=True)
    a2 = (dyg * h).abs().mean(-1, keepdim=True)
    b = U * (rstd64[:, None] * (5 * (dyg.abs() + s1.abs() + (h * s2).abs()) + k1 * a1 + k2 * h.abs() * a2) + dx.abs())
    return dx, b, h


def check_layernorm_bwd(impl, device, case):
    o = _Out("layernorm_bwd")
    g = _gen(case)
    M, d = case["M"], case["d"]
    nv = d // 128
    rpg, gather = case.get("rpg", 0), case.get("gather")
    R = M * rpg if rpg else M
    x = torch.randn(M, d, generator=g) * 2 + 0.5
    x64 = d64(x)
    mu = x64.mean(-1)
    rs = 1.0 / torch.sqrt(((x64 - mu[:, None]) ** 2).mean(-1) + 1e-5)
    mean, rstd = mu.to(F32), rs.to(F32)
    gamma = torch.randn(d, generator=g)
    dyb = case.get("dy", "f32") == "bf16"
    dy = torch.randn(M, d, generator=g).to(BF if dyb else F32)
    alias, use_gin = case.get("alias", False), case.get("gin", True)
    row_idx = torch.randint(0, max(rpg, 1), (M,), generator=g, dtype=torch.int32) if gather == "idx" else None
    phys = torch.arange(M) * rpg + (row_idx.long() if row_idx is not None else 0) if rpg else torch.arange(M)
    gin = torch.randn(R, d, generator=g)
    dg0, db0, gs0 = torch.randn(d, generator=g), torch.randn(d, generator=g), torch.randn(d, generator=g)
    want_bf, want_gsum = case.get("g_bf16", True), case.get("gsum", True)

    G_in = gin.to(device, copy=True) if use_gin else None
    G_out = G_in if alias else torch.zeros(R, d, device=device)
    Gb = torch.zeros(R, d, dtype=BF, device=device) if want_bf else None
    dgamma, dbeta = dg0.to(device, copy=True), db0.to(device, copy=True)
    gsum = gs0.to(device, copy=True) if want_gsum else None
    impl.layernorm_bwd(x.to(device, copy=True), dy.to(device, copy=True) if dyb else None, None if dyb else dy.to(device, copy=True), mean.to(device, copy=True),
                       rstd.to(device, copy=True), gamma.to(device, copy=True), G_in, G_out, Gb, dgamma, dbeta, M, d,
                       row_idx=None if row_idx is None else row_idx.to(device, copy=True), rows_per_group=rpg, gsum=gsum)

    dy64 = d64(dy)
    dx, b_dx, h = _ln_bwd_ref(x64, dy64, d64(mean), d64(rstd), d64(gamma), nv)
    gin64 = d64(gin)
    ref_g = gin64.clone() if alias else torch.zeros(R, d, dtype=F64)
    b_g = torch.zeros(R, d, dtype=F64)
    ref_g[phys] = dx + (gin64[phys] if use_gin else 0)
    b_g[phys] = b_dx + U * ref_g[phys].abs()
    o.bound("g_out", G_out, ref_g, b_g)
    # dgamma / dbeta: per-CTA running sums over ceil(M / grid) rows, then reduce_partials (ceil(grid / 8) + 8 terms)
    # and the += into the caller's buffer; each term dy * h carries 3 roundings.
    grid = _ln_bwd_grid(M, d, _sms(device))
    k = _cdiv(M, grid) + _cdiv(grid, 8) + 8 + 1 + 3
    tg, tb = (dy64 * h).abs().sum(0) + d64(dg0).abs(), dy64.abs().sum(0) + d64(db0).abs()
    o.bound("dgamma", dgamma, d64(dg0) + (dy64 * h).sum(0), k * U * tg)
    o.bound("dbeta", dbeta, d64(db0) + dy64.sum(0), k * U * tb)
    if want_bf:
        gb = Gb.cpu()
        other = torch.ones(R, dtype=torch.bool)
        other[phys] = False
        o.bf16("g_bf16", gb[phys], ref_g[phys], err=b_g[phys])
        o.exact("g_bf16_untouched", gb[other], torch.zeros(int(other.sum()), d, dtype=BF))
        if want_gsum:   # the header's contract: the sum of the bf16-rounded g as stored
            terms = d64(gb[phys])
            o.bound("gsum", gsum, d64(gs0) + terms.sum(0), (k - 3) * U * (terms.abs().sum(0) + d64(gs0).abs()))
    return o.rec


def check_vit_embed_ln_bwd(impl, device, case):
    o = _Out("vit_embed_ln_bwd")
    g = _gen(case)
    B, S, d = case["B"], case["S"], case["d"]
    M, nv = B * S, d // 128
    patch = (torch.randn(B * (S - 1), d, generator=g) * 2).to(BF)
    cls, pos = torch.randn(d, generator=g), torch.randn(S, d, generator=g) * 0.5
    # the kernel re-assembles t = pos + (cls | patch) in fp32 (one rounding): the statistics belong to that t
    t = (torch.cat([d64(cls).view(1, 1, d).expand(B, 1, d), d64(patch).view(B, S - 1, d)], 1)
         + d64(pos).view(1, S, d)).reshape(M, d).to(F32).to(F64)
    mu = t.mean(-1)
    rs = 1.0 / torch.sqrt(((t - mu[:, None]) ** 2).mean(-1) + 1e-5)
    mean, rstd = mu.to(F32), rs.to(F32)
    gamma = torch.randn(d, generator=g)
    dy = torch.randn(M, d, generator=g)
    dg0, db0 = torch.randn(d, generator=g), torch.randn(d, generator=g)
    dt = torch.empty(M, d, device=device)
    dpatch = torch.empty(B * (S - 1), d, dtype=BF, device=device)
    dgamma, dbeta = dg0.to(device, copy=True), db0.to(device, copy=True)
    impl.vit_embed_ln_bwd(patch.to(device, copy=True), cls.to(device, copy=True), pos.to(device, copy=True), dy.to(device, copy=True), mean.to(device, copy=True),
                          rstd.to(device, copy=True), gamma.to(device, copy=True), dt, dpatch, dgamma, dbeta, B, S, d)
    dy64 = d64(dy)
    dx, b_dx, h = _ln_bwd_ref(t, dy64, d64(mean), d64(rstd), d64(gamma), nv)
    o.bound("dt_f32", dt, dx, b_dx)
    o.bf16("dpatch", dpatch, dx.view(B, S, d)[:, 1:].reshape(-1, d), err=b_dx.view(B, S, d)[:, 1:].reshape(-1, d))
    grid = _ln_bwd_grid(M, d, _sms(device))
    k = _cdiv(M, grid) + _cdiv(grid, 8) + 8 + 1 + 3
    o.bound("dgamma", dgamma, d64(dg0) + (dy64 * h).sum(0), k * U * ((dy64 * h).abs().sum(0) + d64(dg0).abs()))
    o.bound("dbeta", dbeta, d64(db0) + dy64.sum(0), k * U * (dy64.abs().sum(0) + d64(db0).abs()))
    return o.rec


# ---- column / batch sums ---------------------------------------------------------------------------------------------
def batch_sum_chunks(n, sms):
    """Number of batch chunks mmb_batch_sum splits the rows into when Bn is large (its blockIdx.y extent)."""
    bx = _cdiv(n // 4, 128)
    return _cdiv(sms * 4, bx)


def _resolve(v, n, device):
    if isinstance(v, tuple):   # ("chunks", delta): relative to the chunk count of this device
        return batch_sum_chunks(n, _sms(device)) + v[1]
    return v


def check_batch_sum(impl, device, case):
    o = _Out("batch_sum")
    g = _gen(case)
    n, ld = case["n"], case["ld"]
    Bn = _resolve(case["Bn"], n, device)
    inp = torch.randn(Bn, ld, generator=g)
    out0 = torch.randn(n + 4, generator=g)
    out = out0.to(device, copy=True)
    impl.batch_sum(inp.to(device, copy=True), out, Bn, ld, n)
    chunks = max(min(batch_sum_chunks(n, _sms(device)), Bn), 1)
    b_chunk = _cdiv(Bn, chunks)
    k = b_chunk + _cdiv(_cdiv(Bn, b_chunk), 8) + 8 + 1      # chunk chain, reduce_partials, the +=
    terms = d64(inp)[:, :n]
    ref = d64(out0).clone()
    ref[:n] += terms.sum(0)
    bnd = torch.zeros(n + 4, dtype=F64)
    bnd[:n] = k * U * (terms.abs().sum(0) + d64(out0)[:n].abs())
    o.bound("out", out, ref, bnd)
    return o.rec


def check_colsum_bf16(impl, device, case):
    o = _Out("colsum_bf16")
    g = _gen(case)
    M, N, ld = case["M"], case["N"], case["ld"]
    x = torch.randn(M, ld, generator=g).to(BF)
    out0 = torch.randn(N, generator=g)
    out = out0.to(device, copy=True)
    impl.colsum_bf16(x.to(device, copy=True), out, M, N, ld)
    bx = _cdiv(N, 256)
    chunks = _cdiv(_sms(device) * 6, bx)
    rpb = _cdiv(_cdiv(M, chunks), 8) * 8
    # per thread rpb / 8 rows, 8 row lanes in shared memory, reduce_partials over the row chunks, the +=
    k = _cdiv(rpb, 8) + 8 + _cdiv(_cdiv(M, rpb), 8) + 8 + 1
    terms = d64(x)[:, :N]
    o.bound("out", out, d64(out0) + terms.sum(0), k * U * (terms.abs().sum(0) + d64(out0).abs()))
    return o.rec


def check_sum_scale(impl, device, case):
    o = _Out("sum_scale")
    g = _gen(case)
    n, scale, acc = case["n"], case["scale"], case["accumulate"]
    inp = torch.randn(n, generator=g)
    out0 = torch.randn(1, generator=g)
    out = out0.to(device, copy=True)
    impl.sum_scale(inp.to(device, copy=True), n, scale, out, accumulate=acc)
    k = _cdiv(n, 256) + 5 + 8 + 2        # per thread, warp shuffles, 8 warp sums, * scale and +=
    s = d64(inp).sum()
    s32 = torch.tensor(scale, dtype=F32).to(F64)
    ref = (d64(out0) if acc else 0) + s * s32
    bnd = k * U * (d64(inp).abs().sum() * abs(s32.item()) + (d64(out0).abs() if acc else 0))
    o.bound("out", out, ref.view(1), torch.as_tensor(bnd, dtype=F64).view(1))
    return o.rec


def check_matmul_f32(impl, device, case):
    o = _Out("matmul_f32")
    g = _gen(case)
    M, N, K, ta, tb, acc, alpha = case["M"], case["N"], case["K"], case["ta"], case["tb"], case["acc"], case["alpha"]
    A = torch.randn(K, M, generator=g) if ta else torch.randn(M, K, generator=g)
    Bm = torch.randn(N, K, generator=g) if tb else torch.randn(K, N, generator=g)
    C0 = torch.randn(M, N, generator=g)
    C = C0.to(device, copy=True)
    impl.matmul_f32(A.to(device, copy=True), Bm.to(device, copy=True), ta=ta, tb=tb, out=C, alpha=alpha, accumulate=acc)
    a64 = d64(A).t() if ta else d64(A)
    b64 = d64(Bm).t() if tb else d64(Bm)
    ref = alpha * (a64 @ b64) + (d64(C0) if acc else 0)
    bnd = (K + 3) * U * (abs(alpha) * (a64.abs() @ b64.abs()) + (d64(C0).abs() if acc else 0))
    o.bound("C", C, ref, bnd)
    return o.rec


# ---- embeddings ------------------------------------------------------------------------------------------------------
def check_text_embed_fwd(impl, device, case):
    o = _Out("text_embed_fwd")
    g = _gen(case)
    B, S, d, V = case["B"], case["S"], case["d"], case["V"]
    tok = torch.randint(0, V, (B, S), generator=g)
    tok[0, 0], tok[-1, -1] = 0, V - 1
    emb, pos = torch.randn(V, d, generator=g), torch.randn(S, d, generator=g)
    x = torch.empty(B * S, d, device=device)
    impl.text_embed_fwd(tok.to(device, copy=True), emb.to(device, copy=True), pos.to(device, copy=True), x, B, S, d, V)
    o.exact("x", x, (d64(emb)[tok] + d64(pos).view(1, S, d)).reshape(B * S, d).to(F32))
    return o.rec


def check_text_embed_bwd(impl, device, case):
    """Padding: the tail of every sequence is token 0, so thousands of rows add into one table row."""
    o = _Out("text_embed_bwd")
    g = _gen(case)
    B, S, d, V = case["B"], case["S"], case["d"], case["V"]
    tok = torch.randint(1, V, (B, S), generator=g)
    lens = torch.randint(1, S + 1, (B,), generator=g)
    tok[torch.arange(S).view(1, S) >= lens.view(B, 1) * case.get("keep", 1.0)] = 0
    grad = torch.randn(B * S, d, generator=g)
    demb0 = torch.randn(V, d, generator=g) * 0.1
    demb = demb0.to(device, copy=True)
    impl.text_embed_bwd(tok.to(device, copy=True), grad.to(device, copy=True), demb, B, S, d)
    flat = tok.view(-1)
    ref = d64(demb0).index_add(0, flat, d64(grad))
    mag = d64(demb0).abs().index_add(0, flat, d64(grad).abs())
    # one CTA adds the rows of a token id in row order: the chain is that id's count + 1
    cnt = torch.bincount(flat, minlength=V).to(F64).view(V, 1)
    o.bound("demb", demb, ref, (cnt + 1) * U * mag)
    return o.rec


def check_argmax_tokens(impl, device, case):
    o = _Out("argmax_tokens")
    g = _gen(case)
    B, S = case["B"], case["S"]
    tok = torch.randint(0, case.get("V", 49408), (B, S), generator=g)
    tok[0] = 7                                     # all equal: the first index
    if B > 1:
        tok[1, S // 3] = tok[1, S - 1] = 10 ** 6   # a tie: the first of them
    if B > 2:
        tok[2, -1] = 10 ** 6 + 1
    idx = torch.empty(B, dtype=torch.int32, device=device)
    impl.argmax_tokens(tok.to(device, copy=True), idx, B, S)
    first = [next(s for s in range(S) if tok[b, s] == tok[b].max()) for b in range(B)]
    o.exact("idx", idx, torch.tensor(first, dtype=torch.int32))
    return o.rec


def check_coca_text_embed_fwd(impl, device, case):
    o = _Out("coca_text_embed_fwd")
    g = _gen(case)
    B, S, d, V, with_cls = case["B"], case["S"], case["d"], case["V"], case["cls"]
    T = S - 1 if with_cls else S
    ids = torch.randint(0, V, (B, T), generator=g)
    emb, cls, pos = torch.randn(V, d, generator=g), torch.randn(d, generator=g), torch.randn(S + 3, d, generator=g)
    x = torch.empty(B * S, d, device=device)
    impl.coca_text_embed_fwd(ids.to(device, copy=True), emb.to(device, copy=True), cls.to(device, copy=True) if with_cls else None, pos.to(device, copy=True), x,
                             B, S, d, V)
    e = d64(emb)[ids]
    if with_cls:
        e = torch.cat([e, d64(cls).view(1, 1, d).expand(B, 1, d)], 1)
    o.exact("x", x, (e + d64(pos)[:S].view(1, S, d)).reshape(B * S, d).to(F32))
    return o.rec


def _bert_inputs(case):
    g = _gen(case)
    B, S, d, V, P, T = case["B"], case["S"], case["d"], case["V"], case["S"] + 5, 2
    ids = torch.randint(0, V, (B, S), generator=g)
    ids[:, -3:] = case.get("pad", 0)
    tt = torch.randint(0, T, (B, S), generator=g) if case.get("types", True) else None
    word, pos, typ = torch.randn(V, d, generator=g), torch.randn(P, d, generator=g), torch.randn(T, d, generator=g)
    gamma, beta = torch.randn(d, generator=g), torch.randn(d, generator=g)
    return g, ids, tt, word, pos, typ, gamma, beta


def _bert_sum(ids, tt, word, pos, typ, S):
    t0 = tt if tt is not None else torch.zeros_like(ids)
    e = d64(word)[ids] + d64(pos)[:S].unsqueeze(0) + d64(typ)[t0]
    mag = d64(word)[ids].abs() + d64(pos)[:S].unsqueeze(0).abs() + d64(typ)[t0].abs()
    return e.reshape(-1, e.shape[-1]), mag.reshape(-1, e.shape[-1]), t0


def check_bert_embed_ln_fwd(impl, device, case):
    o = _Out("bert_embed_ln_fwd")
    _, ids, tt, word, pos, typ, gamma, beta = _bert_inputs(case)
    B, S, d, V, pad = case["B"], case["S"], case["d"], case["V"], case.get("pad", 0)
    x = torch.empty(B * S, d, device=device)
    km = torch.full((B * S,), 7, dtype=torch.uint8, device=device)
    tod = lambda t: None if t is None else t.to(device, copy=True)  # noqa: E731
    impl.bert_embed_ln_fwd(tod(ids), tod(tt), tod(word), tod(pos), tod(typ), tod(gamma), tod(beta), x, km, pad, B, S,
                           d, V, 1e-12)
    e, mag, _ = _bert_sum(ids, tt, word, pos, typ, S)
    out, _, _, b_out, _, _ = _ln_fwd_bounds(e, d64(gamma), d64(beta), 1e-12, d // 128, in_err=2 * U * mag)
    o.bound("x", x, out, b_out)
    o.exact("kmask_out", km, (ids != pad).to(torch.uint8).view(-1))
    return o.rec


def check_bert_embed_ln_bwd(impl, device, case):
    """The statistics are recomputed in fp32 from the tables, and everything lands in fp32 atomics (any order)."""
    o = _Out("bert_embed_ln_bwd")
    g, ids, tt, word, pos, typ, gamma, _ = _bert_inputs(case)
    B, S, d, V = case["B"], case["S"], case["d"], case["V"]
    M, nv = B * S, d // 128
    dy = torch.randn(M, d, generator=g)
    dw0, dp0, dt0 = torch.randn(V, d, generator=g), torch.randn(S + 5, d, generator=g), torch.randn(2, d, generator=g)
    dg0, db0 = torch.randn(d, generator=g), torch.randn(d, generator=g)
    bufs = [t.to(device, copy=True) for t in (dw0, dp0, dt0, dg0, db0)]
    tod = lambda t: None if t is None else t.to(device, copy=True)  # noqa: E731
    impl.bert_embed_ln_bwd(tod(ids), tod(tt), tod(word), tod(pos), tod(typ), tod(gamma), tod(dy), *bufs, B, S, d, V,
                           1e-12)
    e, mag, t0 = _bert_sum(ids, tt, word, pos, typ, S)
    _, mu, rs, h = _ln_ref(e, d64(gamma), torch.zeros(d, dtype=F64), 1e-12)
    dy64 = d64(dy)
    dx, b_dx, _ = _ln_bwd_ref(e, dy64, mu, rs, d64(gamma), nv)
    # the recomputed xhat is off by the forward's statistics error: widen dx by its effect (|d dx / d xhat| <= rstd *
    # (|s2| + |dyg| / d + ...), folded into one term per row)
    _, _, _, b_h, _, _ = _ln_fwd_bounds(e, torch.ones(d, dtype=F64), torch.zeros(d, dtype=F64), 1e-12, nv,
                                        in_err=2 * U * mag)
    dyg = dy64 * d64(gamma)
    b_dx = b_dx + rs[:, None] * (dyg * h).abs().mean(-1, keepdim=True) * b_h \
        + rs[:, None] * (dyg.abs().mean(-1, keepdim=True) * b_h.mean(-1, keepdim=True)) * 2
    flat_ids, flat_pos, flat_t = ids.reshape(-1), torch.arange(S).repeat(B), t0.reshape(-1)
    for name, buf, init, index in (("dword", bufs[0], dw0, flat_ids), ("dpos", bufs[1], dp0, flat_pos),
                                   ("dtype", bufs[2], dt0, flat_t)):
        ref = d64(init).index_add(0, index, dx)
        cnt = torch.bincount(index, minlength=init.shape[0]).to(F64).view(-1, 1)
        bnd = d64(torch.zeros_like(init)).index_add(0, index, b_dx) \
            + (cnt + 1) * U * d64(init).abs().index_add(0, index, dx.abs())
        o.bound(name, buf, ref, bnd)
    k = M + 4      # per-warp register sums and one atomic per warp, in any order: at most M + 1 additions
    o.bound("dgamma", bufs[3], d64(dg0) + (dy64 * h).sum(0),
            k * U * ((dy64 * h).abs().sum(0) + d64(dg0).abs()) + (dy64.abs() * b_h).sum(0))
    o.bound("dbeta", bufs[4], d64(db0) + dy64.sum(0), k * U * (dy64.abs().sum(0) + d64(db0).abs()))
    return o.rec


# ---- L2 normalisation ------------------------------------------------------------------------------------------------
def check_l2norm_fwd(impl, device, case):
    o = _Out("l2norm_fwd")
    g = _gen(case)
    B, E, eps = case["B"], case["E"], 1e-12
    x = torch.randn(B, E, generator=g) * 3
    if case.get("zero_row") is not None:
        x[case["zero_row"]] = 0
    y = torch.empty(B, E, device=device)
    yb = torch.empty(B, E, dtype=BF, device=device)
    inv = torch.empty(B, device=device)
    impl.l2norm_fwd(x.to(device, copy=True), y, yb, inv, B, E, eps)
    x64 = d64(x)
    eps32 = torch.tensor(eps, dtype=F32).item()
    inv64 = 1.0 / torch.clamp_min(x64.norm(dim=1), eps32)
    k = _cdiv(E, 32) + 5 + 1           # per-lane squares, shuffles
    o.bound("inv_norm", inv, inv64, (k / 2 + 3) * U * inv64)
    y64 = x64 * inv64[:, None]
    o.bound("y", y, y64, (k / 2 + 4) * U * y64.abs())
    o.bf16("y_bf16", yb, y64, err=(k / 2 + 4) * U * y64.abs())
    return o.rec


def check_l2norm_bwd(impl, device, case):
    o = _Out("l2norm_bwd")
    g = _gen(case)
    B, E = case["B"], case["E"]
    x = torch.randn(B, E, generator=g)
    y = (x / x.norm(dim=1, keepdim=True)).to(F32)
    inv = torch.rand(B, generator=g) + 0.2
    dy = torch.randn(B, E, generator=g)
    dx = torch.empty(B, E, device=device)
    dxb = torch.empty(B, E, dtype=BF, device=device)
    impl.l2norm_bwd(dy.to(device, copy=True), y.to(device, copy=True), inv.to(device, copy=True), dx, dxb, B, E)
    y64, dy64, inv64 = d64(y), d64(dy), d64(inv)[:, None]
    s = (y64 * dy64).sum(1, keepdim=True)
    ref = inv64 * (dy64 - y64 * s)
    k = _cdiv(E, 32) + 5 + 1
    bnd = U * (inv64 * (3 * (dy64.abs() + (y64 * s).abs()) + k * y64.abs() * (y64 * dy64).abs().sum(1, keepdim=True))
               + ref.abs())
    o.bound("dx", dx, ref, bnd)
    o.bf16("dx_bf16", dxb, ref, err=bnd)
    return o.rec


# ---- activations -------------------------------------------------------------------------------------------------------
_RSQRT2 = 1.0 / math.sqrt(2.0)


def _phi_cdf(x64):
    return 0.5 * torch.special.erfc(-x64 * _RSQRT2)


def _act64(x64, kind):
    if kind == 0:
        return x64 * torch.sigmoid(1.702 * x64)
    return x64 * _phi_cdf(x64)


def _act_grad64(x64, kind):
    if kind == 0:
        s = torch.sigmoid(1.702 * x64)
        return s * (1 + 1.702 * x64 * (1 - s))
    return _phi_cdf(x64) + x64 * torch.exp(-0.5 * x64 * x64) / math.sqrt(2 * math.pi)


TANH_APPROX = 2.0 ** -10.987   # maximum relative error of tanh.approx.f32 (PTX ISA)


def _quick_gelu_tanh(x64):
    """u = 0.851 x, t = tanh(u) and the absolute error of the kernels' t = tanh.approx(fl(0.851f x)) (common.cuh
    quick_gelu / quick_gelu_grad): the approximation's TANH_APPROX |t| plus u's rounding (2 U |u|: the constant and the
    product) carried through dt / du = 1 - t^2."""
    u = 0.851 * x64
    t = torch.tanh(u)
    return u, t, TANH_APPROX * t.abs() + 2 * U * u.abs() * (1 - t * t)


def _act_fwd_epi_err(x64, kind):
    """Absolute error of the GEMM epilogue's act(x) in fp32 (common.cuh act_fn).  QuickGELU = fmaf(h, t, h), h = x / 2:
    |h| times t's error plus the fmaf's rounding; GELU-erf as check_act_fwd."""
    if kind == 0:
        _, _, et = _quick_gelu_tanh(x64)
        return 0.5 * x64.abs() * et + U * _act64(x64, 0).abs()
    return 4 * U * _act64(x64, 1).abs() + 8 * U * x64.abs()


def _act_grad_err(x64, kind):
    """Absolute error of the kernels' act'(x) in fp32 (common.cuh act_grad).  QuickGELU': 0.5 (1 + t + u (1 - t^2)),
    whose derivative in t is 0.5 (1 - 2 u t), plus the roundings of the three fmaf; GELU-erf': Phi(x) = 0.5 (1 + erf)
    carries an absolute error of a few ulp of 1, exp of -x^2/2 a relative one ~ x^2 u."""
    if kind == 0:
        u, t, et = _quick_gelu_tanh(x64)
        return 0.5 * (1 - 2 * u * t).abs() * et + 8 * U * (1 + u.abs())
    return 8 * U + (8 + x64 * x64) * U * (x64 * torch.exp(-0.5 * x64 * x64)).abs()


def _act_input(case, n):
    x = torch.randn(n, generator=_gen(case)) * 3
    return _with_specials(x, ACT_SPECIALS)


def check_act_fwd(impl, device, case):
    """QuickGELU: x / (1 + exp(-1.702 x)) with an approximate exp whose argument error grows with |x|; exact GELU:
    0.5 x (1 + erf(x / sqrt 2)), where 1 + erf cancels for negative x (an absolute error of a few ulp of |x|)."""
    o = _Out("act_fwd")
    n, kind = case["n"], case["kind"]
    x = _act_input(case, n)
    y = impl.act_fwd(x.to(device, copy=True), kind)
    x64 = d64(x)
    ref = _act64(x64, kind)
    if kind == 0:
        bnd = (2.5 * 1.702 * x64.abs() + 8) * U * ref.abs()
    else:
        bnd = 4 * U * ref.abs() + 8 * U * x64.abs()
    o.bound("y", y, ref, bnd)
    return o.rec


def check_tanh_(impl, device, case):
    o = _Out("tanh_")
    n = case["n"]
    x = _act_input(case, n)
    xd = x.to(device, copy=True)
    impl.tanh_(xd)
    ref = torch.tanh(d64(x))
    o.bound("x", xd, ref, 4 * U * ref.abs())
    o.exact("signed_zeros", xd.cpu()[2:4], torch.tensor([0.0, -0.0]))
    return o.rec


def check_tanh_bwd(impl, device, case):
    o = _Out("tanh_bwd")
    g = _gen(case)
    n = case["n"]
    y = torch.tanh(torch.randn(n, generator=g) * 2)
    dy = torch.randn(n, generator=g)
    dx = torch.empty(n, device=device)
    dxb = torch.empty(n, dtype=BF, device=device)
    impl.tanh_bwd(dy.to(device, copy=True), y.to(device, copy=True), dx, dxb)
    y64, dy64 = d64(y), d64(dy)
    ref = dy64 * (1 - y64 * y64)
    bnd = 3 * U * dy64.abs() * ((1 - y64 * y64).abs() + y64 * y64)
    o.bound("dx", dx, ref, bnd)
    o.bf16("dx_bf16", dxb, ref, err=bnd)
    return o.rec


def check_act_bwd(impl, device, case):
    o = _Out("act_bwd")
    g = _gen(case)
    n, kind = case["n"], case["kind"]
    pre = _act_input(case, n).to(BF)
    dy = torch.randn(n, generator=g).to(BF)
    dx = torch.empty(n, dtype=BF, device=device)
    impl.act_bwd(dy.to(device, copy=True), pre.to(device, copy=True), dx, kind)
    x64, dy64 = d64(pre), d64(dy)
    o.bf16("dx", dx, dy64 * _act_grad64(x64, kind), case.get("min_equal", 0.99),
           err=dy64.abs() * _act_grad_err(x64, kind))
    return o.rec


# ---- gathers, scatters, token assembly -----------------------------------------------------------------------------------
def check_gather_rows_cast(impl, device, case):
    o = _Out("gather_rows_cast")
    B, rpg, row, d = case["B"], case["rpg"], case["row"], case["d"]
    x = torch.randn(B * rpg, d, generator=_gen(case))
    out = torch.empty(B, d, dtype=BF, device=device)
    impl.gather_rows_cast(x.to(device, copy=True), out, B, rpg, row, d)
    o.exact("out", out, rne_bf16(x.view(B, rpg, d)[:, row]))
    return o.rec


def check_gather_rows_idx_cast(impl, device, case):
    o = _Out("gather_rows_idx_cast")
    g = _gen(case)
    R, ld, d, n = case["R"], case["ld"], case["d"], case["n"]
    buf = torch.randn(R, ld, generator=g)
    idx = torch.randint(0, R, (n,), generator=g)
    if n > 2:
        idx[1] = idx[0]            # repeated rows
        idx[-1] = R - 1
    out = torch.empty(n, d, dtype=BF, device=device)
    impl.gather_rows_idx_cast(buf.to(device, copy=True)[:, :d], idx.to(device, copy=True), out, d)
    o.exact("out", out, rne_bf16(buf[idx, :d]))
    return o.rec


def check_scatter_rows_add(impl, device, case):
    o = _Out("scatter_rows_add")
    g = _gen(case)
    B, rpg, row, d = case["B"], case["rpg"], case["row"], case["d"]
    src = torch.randn(B, d, generator=g)
    dst0 = torch.randn(B * rpg, d, generator=g)
    dst = dst0.to(device, copy=True)
    impl.scatter_rows_add(src.to(device, copy=True), dst, B, rpg, row, d)
    ref = d64(dst0).view(B, rpg, d).clone()
    ref[:, row] += d64(src)
    o.exact("dst", dst, ref.view(B * rpg, d).to(F32))
    return o.rec


def check_scatter_rows_idx_add(impl, device, case):
    """fp32 atomics: repeated rows add in any order, so each destination row gets (count + 1) * u * sum|terms|."""
    o = _Out("scatter_rows_idx_add")
    g = _gen(case)
    R, ld, d, n = case["R"], case["ld"], case["d"], case["n"]
    src = torch.randn(n, d, generator=g)
    idx = torch.randint(0, R, (n,), generator=g)
    if n > 3:
        idx[: n // 3] = idx[0]
    buf0 = torch.randn(R, ld, generator=g)
    buf = buf0.to(device, copy=True)
    impl.scatter_rows_idx_add(src.to(device, copy=True), idx.to(device, copy=True), buf[:, :d], d)
    ref = d64(buf0).clone()
    ref[:, :d] = ref[:, :d].index_add(0, idx, d64(src))
    cnt = torch.bincount(idx, minlength=R).to(F64).view(R, 1)
    bnd = torch.zeros(R, ld, dtype=F64)
    bnd[:, :d] = (cnt + 1) * U * d64(buf0)[:, :d].abs().index_add(0, idx, d64(src).abs())
    o.bound("dst", buf, ref, bnd)
    return o.rec


def check_concat_tokens(impl, device, case):
    o = _Out("concat_tokens")
    g = _gen(case)
    B, Sa, Sb, d, with_cls = case["B"], case["Sa"], case["Sb"], case["d"], case["cls"]
    cls = torch.randn(d, generator=g)
    a, b = torch.randn(B * Sa, d, generator=g), torch.randn(B * Sb, d, generator=g)
    So = (1 if with_cls else 0) + Sa + Sb
    out = torch.empty(B * So, d, device=device)
    ad = a.to(device, copy=True)
    impl.concat_tokens(cls.to(device, copy=True) if with_cls else None, ad, b.to(device, copy=True) if Sb else ad, out, B, Sa, Sb, d)
    parts = ([cls.view(1, 1, d).expand(B, 1, d)] if with_cls else []) + [a.view(B, Sa, d), b.view(B, Sb, d)]
    o.exact("out", out, torch.cat(parts, 1).reshape(B * So, d))
    return o.rec


def check_split_tokens_cast(impl, device, case):
    o = _Out("split_tokens_cast")
    B, Sa, Sb, d, has_cls = case["B"], case["Sa"], case["Sb"], case["d"], case["cls"]
    off = 1 if has_cls else 0
    gr = torch.randn(B * (off + Sa + Sb), d, generator=_gen(case))
    a = torch.empty(B * Sa, d, dtype=BF, device=device)
    b = torch.empty(B * Sb, d, dtype=BF, device=device) if Sb else None
    impl.split_tokens_cast(gr.to(device, copy=True), a, b, B, Sa, Sb, d, has_cls=has_cls)
    gv = gr.view(B, off + Sa + Sb, d)
    o.exact("a", a, rne_bf16(gv[:, off:off + Sa].reshape(-1, d)))
    if Sb:
        o.exact("b", b, rne_bf16(gv[:, off + Sa:].reshape(-1, d)))
    return o.rec


def check_vit_assemble_fwd(impl, device, case):
    o = _Out("vit_assemble_fwd")
    g = _gen(case)
    B, S, d, with_cls, masked = case["B"], case["S"], case["d"], case["cls"], case["mask"]
    off = 1 if with_cls else 0
    P = S - off
    patch = torch.randn(B * P, d, generator=g).to(BF)
    cls, pos, mtok = torch.randn(d, generator=g), torch.randn(S, d, generator=g), torch.randn(d, generator=g)
    pm = (torch.rand(B * P, generator=g) < 0.4).to(torch.uint8)
    x = torch.empty(B * S, d, device=device)
    tod = lambda t: t.to(device, copy=True)  # noqa: E731
    impl.vit_assemble_fwd(tod(patch), tod(cls) if with_cls else None, tod(pos), tod(mtok) if masked else None,
                          tod(pm) if masked else None, x, B, S, d)
    e = d64(patch).view(B, P, d)
    if masked:
        e = torch.where(pm.view(B, P, 1).bool(), d64(mtok).view(1, 1, d), e)
    if with_cls:
        e = torch.cat([d64(cls).view(1, 1, d).expand(B, 1, d), e], 1)
    o.exact("x", x, (e + d64(pos).view(1, S, d)).reshape(B * S, d).to(F32))
    return o.rec


def check_vit_assemble_bwd(impl, device, case):
    o = _Out("vit_assemble_bwd")
    g = _gen(case)
    B, S, d, has_cls, masked = case["B"], case["S"], case["d"], case["cls"], case["mask"]
    off = 1 if has_cls else 0
    P = S - off
    gr = torch.randn(B * S, d, generator=g)
    pm = (torch.rand(B * P, generator=g) < 0.4).to(torch.uint8)
    dm0 = torch.randn(d, generator=g)
    dpatch = torch.empty(B * P, d, dtype=BF, device=device)
    dm = dm0.to(device, copy=True)
    impl.vit_assemble_bwd(gr.to(device, copy=True), pm.to(device, copy=True) if masked else None, dpatch, dm if masked else None, B, S, d,
                          has_cls=has_cls)
    gp = gr.view(B, S, d)[:, off:].reshape(B * P, d)
    if masked:
        keep = ~pm.bool().view(-1, 1)
        o.exact("dpatch", dpatch, torch.where(keep, rne_bf16(gp), torch.zeros((), dtype=BF)))
        terms = d64(gp)[pm.bool()]
        k = 16 + _cdiv(B * P, 16) + 1      # a 16-row strip per thread, then one atomic per strip
        o.bound("dmask_token", dm, d64(dm0) + terms.sum(0), k * U * (terms.abs().sum(0) + d64(dm0).abs()))
    else:
        o.exact("dpatch", dpatch, rne_bf16(gp))
        o.exact("dmask_token_untouched", dm, dm0)
    return o.rec


def check_zero_(impl, device, case):
    o = _Out("zero_")
    t = torch.randn(case["n"], generator=_gen(case)).to(device, copy=True)
    impl.zero_(t)
    o.exact("t", t, torch.zeros(case["n"]))
    return o.rec


def check_kv_cache_append(impl, device, case):
    o = _Out("kv_cache_append")
    g = _gen(case)
    B, H, Sp, Sn, hd = case["B"], case["H"], case["Sp"], case["Sn"], case["hd"]
    past_dt, out_dt, want_bf = case["past"], case["out"], case["out_bf16"]
    d = H * hd
    past = None
    if Sp:   # stored [B, Sp, H, hd]: a [B, H, Sp, hd] view with non-contiguous strides
        past = torch.randn(B, Sp, H, hd, generator=g).to(past_dt).transpose(1, 2)
    newbuf = torch.randn(B * Sn, d + 8, generator=g).to(BF)
    out = torch.empty(B * (Sp + Sn) * d, dtype=out_dt, device=device) if out_dt is not None else None
    outb = torch.empty(B * (Sp + Sn) * d, dtype=BF, device=device) if want_bf else None
    impl.kv_cache_append(None if past is None else past.to(device, copy=True), newbuf.to(device, copy=True)[:, :d], out, outb, B=B, H=H,
                         Sp=Sp, Sn=Sn, head_dim=hd)
    new = newbuf[:, :d].to(F32).view(B, Sn, d)
    cat = new if past is None else torch.cat([past.to(F32).transpose(1, 2).reshape(B, Sp, d), new], 1)
    cat = cat.reshape(-1)
    if out is not None:
        o.exact("out", out, cat if out_dt == F32 else rne_bf16(cat))
    if outb is not None:
        o.exact("out_bf16", outb, rne_bf16(cat))
    return o.rec


# ---- losses --------------------------------------------------------------------------------------------------------------
def _ce_inputs(case):
    g = _gen(case)
    M, V, stride, ignore = case["M"], case["V"], case["stride"], case.get("ignore", -100)
    logits = torch.randn(M, V, generator=g) * case.get("scale", 3.0)
    lab = torch.randint(0, V, (M,), generator=g)
    lab[0] = V - 1
    nig = case.get("n_ignored", 0)
    if nig:
        lab[torch.randperm(M, generator=g)[:nig]] = ignore
    labels = torch.full((M * stride,), 12345, dtype=torch.int64)   # the other slots of a strided label view
    labels[::stride] = lab
    return g, logits, lab, labels, ignore


def check_ce_labels(impl, device, case):
    """row loss = max + log(sum exp(x - max)) - x[label] with an approximate exp (relative error ~(2 + 1.44 |z|) u for
    argument z) summed over ceil(V / 256) + 5 + 8 terms; accum[0] adds the kept rows through reduce_partials."""
    o = _Out("ce_labels")
    g, logits, lab, labels, ignore = _ce_inputs(case)
    M, V, stride = case["M"], case["V"], case["stride"]
    row_loss = torch.full((M,), 5.0, device=device)
    acc0 = torch.tensor([1.5, 2.0])
    accum = acc0.to(device, copy=True)
    impl.ce_labels(logits.to(device, copy=True), labels.to(device, copy=True), stride, ignore, M, V, row_loss, accum)
    l64 = d64(logits)
    keep = lab != ignore
    lse = torch.logsumexp(l64, 1)
    mx = l64.max(1).values
    nll = torch.where(keep, lse - l64.gather(1, lab.clamp(0, V - 1).view(-1, 1)).squeeze(1), torch.zeros((), dtype=F64))
    zspan = (mx - l64.min(1).values)
    k = _cdiv(V, 256) + 5 + 8 + 4
    b_row = U * ((k + 2 + 1.5 * zspan) + 2 * (mx.abs() + lse.abs() + l64.abs().max(1).values))
    b_row = torch.where(keep, b_row, torch.zeros((), dtype=F64))
    o.bound("row_loss", row_loss, nll, b_row)
    kr = _cdiv(M, 8) + 8 + 1
    o.bound("accum", accum, torch.stack([d64(acc0)[0] + nll.sum(), d64(acc0)[1] + keep.sum().to(F64)]),
            torch.stack([b_row.sum() + kr * U * (nll.abs().sum() + abs(acc0[0].item())), torch.zeros((), dtype=F64)]))
    return o.rec


def check_ce_labels_bwd(impl, device, case):
    o = _Out("ce_labels_bwd")
    g, logits, lab, labels, ignore = _ce_inputs(case)
    M, V, stride = case["M"], case["V"], case["stride"]
    keep = lab != ignore
    count = float(keep.sum())
    accum = torch.tensor([3.0, count])
    gscale = torch.tensor([0.75]) if case.get("gscale") else None
    dl = torch.empty(M, V, dtype=BF, device=device)
    impl.ce_labels_bwd(logits.to(device, copy=True), labels.to(device, copy=True), stride, ignore, M, V, accum.to(device, copy=True), 1.25, dl,
                       gscale=None if gscale is None else gscale.to(device, copy=True))
    l64 = d64(logits)
    p = torch.softmax(l64, 1)
    oh = torch.zeros(M, V, dtype=F64)
    oh[torch.arange(M)[keep], lab[keep]] = 1
    w = 1.25 * (0.75 if gscale is not None else 1.0) / max(count, 1.0)
    zspan = (l64.max(1).values - l64.min(1).values).view(-1, 1)
    k = _cdiv(V, 256) + 5 + 8 + 4
    err = abs(w) * ((k + 2 + 1.5 * zspan) * U * p + 2 * U * (p - oh).abs()) * keep.view(-1, 1)
    o.bf16("dlogits", dl, w * (p - oh) * keep.view(-1, 1), err=err)
    return o.rec


# ---- GEMM: every instantiation gemm_launch dispatches, its fused epilogues, tile boundaries and operand pitches ----------
# A case names the epilogue ("epi": bf16 / act / dact / f32), the operand layouts (a_mn, b_mn), the activation (act:
# 0 QuickGELU, 1 GELU-erf), alpha, bias, colsum, split-K (splits), "pad" extra columns on every pitch and, for fp32,
# the output's first column "col0" in its buffer (1: a base off 16 bytes, written with direct stores).
# Operands: A scaled by 3 / sqrt(K) (pre-activations of a few units, where the activations bend), bf16 before the
# float64 products are formed (_gemm64), stored at pitches rounded up to 8 elements past extent + pad with the padding
# NaN: a read of it poisons the result.  Outputs are [M, N] views one row into [M + 2, ld] buffers of a sentinel bit
# pattern: every element outside [M, N] must come back unchanged.
# Bounds (S = the split count the dispatch forms):
#   acc     the fp32 accumulation and the fmaf that applies alpha and bias, (K + S + 3) U (|alpha| sum|a||b| + |bias|);
#   D0      bf16 (EPI_BF16, the ACT pre-activation): within 1 bf16 ulp of bf16(alpha A B^T + bias), err = acc;
#   D1      act(D0) of the implementation's own stored bf16 D0 (mmb200.h: D1 = bf16(act(D0))), err = _act_fwd_epi_err;
#   DACT    alpha acc act'(aux): err = (acc + U |alpha acc|) |act'| + |alpha acc| _act_grad_err;
#   colsum  colsum0 + sum_m of the stored D0: k U sum|terms| with k = 2 (rows per thread) + 3 (shuffle levels) +
#           8 (warps) + ceil(P / 8) + 8 + 1 (reduce_partials over P = ceil(M / 128) row blocks);
#   fp32    D = alpha acc + bias within acc, and D_acc = C0 + alpha acc + bias within acc + (K + S + 3) U |C0|.
_SENT_BF16 = 0x4B39
_SENT_F32 = 0x4B39A5C3
_EPI = {"bf16": 0, "act": 1, "dact": 2, "f32": 3}


def _ld8(n):
    return _cdiv(n, 8) * 8


def _nan_padded(x, ld):
    """x [rows, cols] bf16 stored in a [rows, ld] buffer whose padding columns are NaN."""
    buf = torch.full((x.shape[0], ld), NAN, dtype=BF)
    buf[:, :x.shape[1]] = x
    return buf


def _gemm_splits(K, splits, epi):
    """The split count gemm_dispatch forms: clamped to [1, k-blocks], one for bf16 epilogues, then whole k-block runs."""
    kb = _cdiv(K, 64)
    s = 1 if epi != "f32" else min(max(splits, 1), kb)
    return _cdiv(kb, _cdiv(kb, s))


def _sentinel_out(M, N, ld, col0, dtype, device, inner=None):
    """The [M, N] view at row 1, column col0 of a [M + 2, ld] buffer filled with the sentinel (inner: its values)."""
    if dtype == BF:
        buf = torch.full((M + 2, ld), _SENT_BF16, dtype=torch.int16).view(BF)
    else:
        buf = torch.full((M + 2, ld), _SENT_F32, dtype=torch.int32).view(F32)
    if inner is not None:
        buf[1:M + 1, col0:col0 + N] = inner
    buf = buf.to(device, copy=True)
    return buf, buf[1:M + 1, col0:col0 + N]


def _check_outside(o, name, buf, M, N, col0):
    got = buf.detach().cpu()
    keep = torch.ones(got.shape, dtype=torch.bool)
    keep[1:M + 1, col0:col0 + N] = False
    want = _SENT_BF16 if got.dtype == BF else _SENT_F32
    o.exact(name, _bits(got)[keep], torch.full((int(keep.sum()),), want, dtype=_bits(got).dtype))


def check_gemm(impl, device, case):
    o = _Out("gemm")
    g = _gen(case)
    M, N, K = case["M"], case["N"], case["K"]
    epi, act, a_mn, b_mn = case["epi"], case.get("act", 0), case.get("a_mn", 0), case.get("b_mn", 0)
    alpha, pad, col0 = case.get("alpha", 1.0), case.get("pad", 0), case.get("col0", 0)
    S = _gemm_splits(K, case.get("splits", 1), epi)
    use_bias = case.get("bias", epi != "dact")
    use_colsum = case.get("colsum", epi in ("bf16", "dact"))
    A = (torch.randn(M, K, generator=g) * (3 / math.sqrt(K))).to(BF)
    Bm = torch.randn(N, K, generator=g).to(BF)
    bias = torch.randn(N, generator=g)
    As = _nan_padded(A.t() if a_mn else A, _ld8((M if a_mn else K) + pad))
    Bs = _nan_padded(Bm.t() if b_mn else Bm, _ld8((N if b_mn else K) + pad))
    Ad = As.to(device, copy=True)[:, :(M if a_mn else K)]
    Bd = Bs.to(device, copy=True)[:, :(N if b_mn else K)]
    tod = lambda t: t.to(device, copy=True)  # noqa: E731
    acc, mag = _gemm64(A, Bm)
    mag = mag / ((K + 3) * U)
    b64 = d64(bias) if use_bias else torch.zeros(N, dtype=F64)
    ref = alpha * acc + b64
    e_acc = (K + S + 3) * U * (abs(alpha) * mag + b64.abs())
    kw = dict(a_mn=bool(a_mn), b_mn=bool(b_mn), epilogue=_EPI[epi], alpha=alpha, act=act, splits=case.get("splits", 1),
              bias=tod(bias) if use_bias else None)
    ld = (_ld8 if epi != "f32" else lambda n: _cdiv(n, 4) * 4)(col0 + N + pad)

    if epi == "f32":
        C0 = torch.randn(M, N, generator=g)
        buf, D = _sentinel_out(M, N, ld, col0, F32, device)
        buf_acc, D_acc = _sentinel_out(M, N, ld, col0, F32, device, inner=C0)
        with _gemm_mode(impl, case):
            impl.gemm(Ad, Bd, out=D, **kw)
            impl.gemm(Ad, Bd, out=D_acc, accumulate=True, **kw)
        o.bound("D", D, ref, e_acc)
        o.bound("D_acc", D_acc, ref + d64(C0), e_acc + (K + S + 3) * U * d64(C0).abs())
        _check_outside(o, "D_outside", buf, M, N, col0)
        _check_outside(o, "D_acc_outside", buf_acc, M, N, col0)
        return o.rec

    cs0 = torch.randn(N, generator=g)
    cs = tod(cs0) if use_colsum else None
    buf0, D0 = _sentinel_out(M, N, ld, 0, BF, device)
    if epi == "act":
        buf1, D1 = _sentinel_out(M, N, ld, 0, BF, device)
        with _gemm_mode(impl, case):
            impl.gemm(Ad, Bd, out=D0, out2=D1, **kw)
    elif epi == "dact":
        aux = (torch.randn(M, N, generator=g) * 2).to(BF)
        auxd = tod(_nan_padded(aux, _ld8(N + pad)))[:, :N]
        with _gemm_mode(impl, case):
            impl.gemm(Ad, Bd, out=D0, aux=auxd, colsum=cs, **kw)
    else:
        with _gemm_mode(impl, case):
            impl.gemm(Ad, Bd, out=D0, colsum=cs, **kw)

    if epi == "dact":
        x64 = d64(aux)
        gr = _act_grad64(x64, act)
        o.bf16("D0", D0, ref * gr, err=(e_acc + U * ref.abs()) * gr.abs() + ref.abs() * _act_grad_err(x64, act))
    else:
        o.bf16("D0", D0, ref, err=e_acc)
    _check_outside(o, "D0_outside", buf0, M, N, 0)
    if epi == "act":
        pre = d64(D0)
        o.bf16("D1", D1, _act64(pre, act), err=_act_fwd_epi_err(pre, act))
        _check_outside(o, "D1_outside", buf1, M, N, 0)
    if use_colsum:
        terms = d64(D0)
        k = 2 + 3 + 8 + _cdiv(_cdiv(M, 128), 8) + 8 + 1
        o.bound("colsum", cs, d64(cs0) + terms.sum(0), k * U * (terms.abs().sum(0) + d64(cs0).abs()))
    return o.rec


# ---- attention -------------------------------------------------------------------------------------------------------
u = 2.0 ** -8           # unit roundoff of bf16: one rounding moves a value by at most u of itself
EX2 = 2.0 ** -21        # relative error of the kernels' exponential (exp2f / ex2.approx.ftz.f32: 2 ulp)
TINY_P = 2.0 ** -126    # a p that ex2.approx.ftz or a bf16 / fp32 rounding flushes to zero is at most this
LOG2E, LN2 = 1.0 / math.log(2.0), math.log(2.0)
NAN = float("nan")


def _refdev():
    """The float64 references run on the GPU when there is one: S = 4097 needs [S, S] float64 matrices."""
    return torch.device("cuda") if torch.cuda.is_available() else torch.device("cpu")


def _attn_bh(q, k, v, allow, scale, dout=None, o_used=None, lse_used=None, probs=False):
    """Float64 attention of one (batch, head) and the derived bound of every output element.  q [Sq, D], k / v [Skv, D],
    dout [Sq, D] (float64, on one device), allow bool [Sq, Skv], scale the fp32 value the kernel is given.  o_used /
    lse_used: the bf16 O and the lse a backward (or attention_probs) is handed; None where it forms them itself.  Every
    bound is row-local: built from the row's (or key's) own p, |v|, |dO|, |q|, |k|.  U = 2^-24, u = 2^-8.

    Scores, in log2 units (s2 = q.k * scale * log2e, which the kernels exponentiate with exp2):
      es_ij = scale*log2e*(D+2)*U*sum_d|q_id k_jd|    the fp32 dot product (exact bf16 products, D additions)
              + 8U*(|s2_ij| + M_i + log2(Skv + 1))    scale*log2e, the product, s2 - m or s2 - lse2 (|lse2| <= M + log2 Skv)
      M_i = max over visible j of |s2_ij|.
    A kernel's p_ij = 2^(s2_ij - m_i) / l_i then has the relative error
      dp_ij = ln2*es_ij + EX2 + 2U + dl_i,
      dl_i  = nr*(EX2 + 2U + 2U*ln2*M_i) + (nr + 136)*U
    from nr = ceil(Skv/64) + 2 running-max rescales 2^(m_old - m_new) (one per 64-key block, one for the decode
    kernel's combine of its splits) and the fp32 sum l of positive terms (64 adds per block, the block chain, 64 split
    partials, 8 reduction levels).  A p below 2^-126 may flush to zero: TINY_P, absolute.
    O_id = sum_j p_ij v_jd with P rounded to bf16 for the PV product (u) and fp32 sums of at most Skv + 18 adds:
      |dO_id| <= (u + (Skv+18)*U)*A_id + sum_j p_ij*dp_ij*(|v_jd| + |O_id|) + TINY_P*sum_j visible |v_jd|,
      A_id = sum_j p_ij*|v_jd|, plus u*|O_id| for the bf16 output.  (The normaliser l sums the unrounded fp32 p.)
    lse_i = (m_i + log2 l_i)*ln2:
      |dlse_i| <= ln2*sum_j p_ij*es_ij + dl_i + 4U*(|lse_i| + ln2*M_i) + 2U*log2(Skv + 1);  -inf for a row with no
      visible key.
    Backward.  p is recomputed from the lse (dlse: the actual error of the lse handed in, or the bound above where the
    kernel forms it): dpb_ij = ln2*es_ij + dlse_i*(1 + dlse_i) + EX2 + 2U.
      dP_ij = dO_i . v_j, exact products and fp32 sums: edP_ij = (D+2)*U*sum_d|dO_id v_jd|.
      D_i = rowsum(dO * O~) over the bf16 O~ handed in (packed and resident kernels) or sum_j p_ij dP_ij (generic
      streamed backward).  One bound covers both:
        bD_i = sum_d|dO_id|*|O~_id - O_id| + sum_j p_ij*(dpb_ij*|dP_ij| + edP_ij)
               + (Skv + D + 8)*U*(sum_d|dO_id O~_id| + sum_j p_ij*|dP_ij|).
      dS_ij = p_ij*(dP_ij - D_i), rounded to bf16 before the dQ / dK products:
        edS_ij = p_ij*((dpb_ij + 3U + u)*|dP_ij - D_i| + (1 + u)*(edP_ij + bD_i)) + TINY_P*(|dP_ij| + |D_i|).
      dQ = scale*dS K, dK = scale*dS^T Q, dV = P^T dO (P bf16), fp32 sums of at most Skv + 18 / Sq + 18 adds:
        bdQ = scale*(edS |K| + (Skv+18)*U*|dS| |K|), bdK = scale*(edS^T |Q| + (Sq+18)*U*|dS|^T |Q|),
        bdV = (p*(dpb + u))^T |dO| + (Sq+18)*U*p^T |dO| + TINY_P*visible^T |dO|,
      plus u*|x| for the bf16 outputs (not for the fp32 dq_f32 of batch-shared queries).
    The returned b* entries leave out those final bf16 roundings: the checks pass them to _Out.bound as `rnd`.
    attention_probs: |dp_ij| <= p_ij*(ln2*es_ij + dlse_i*(1 + dlse_i) + EX2 + 2U) + TINY_P; exactly 0 where masked,
    causal-future or the row is empty."""
    Sq, D = q.shape
    Skv = k.shape[0]
    zero = torch.zeros((), dtype=F64, device=q.device)
    vis = allow.any(1, keepdim=True)
    fa = allow.to(F64)
    s = (q @ k.t()) * scale
    s2a = (s * LOG2E).abs()
    sm = s.masked_fill(~allow, float("-inf"))
    lse = torch.logsumexp(sm, 1, keepdim=True)
    p = torch.where(allow, torch.exp(sm - torch.where(vis, lse, zero)), zero)
    M = torch.where(allow, s2a, zero).amax(1, keepdim=True)
    l2s = math.log2(Skv + 1)
    es = scale * LOG2E * (D + 2) * U * (q.abs() @ k.abs().t()) + 8 * U * (s2a + M + l2s)
    nr = _cdiv(Skv, 64) + 2
    dl = nr * (EX2 + 2 * U + 2 * U * LN2 * M) + (nr + 136) * U
    dp = LN2 * es + EX2 + 2 * U + dl
    av = v.abs()
    O = p @ v
    pd = p * dp
    b_o = (u + (Skv + 18) * U) * (p @ av) + pd @ av + pd.sum(1, keepdim=True) * O.abs() + TINY_P * (fa @ av)
    b_lse = LN2 * (p * es).sum(1, keepdim=True) + dl + 4 * U * (lse.abs() + LN2 * M) + 2 * U * l2s
    r = {"O": O, "bO": b_o, "lse": lse.squeeze(1), "blse": torch.where(vis, b_lse, zero).squeeze(1),
         "vis": vis.squeeze(1)}
    if lse_used is not None:
        dlse = torch.where(vis, (lse_used.view(-1, 1) - lse).abs(), zero)
    else:
        dlse = torch.where(vis, b_lse, zero)
    dpb = LN2 * es + dlse * (1 + dlse) + EX2 + 2 * U
    if probs:
        r["P"] = p
        r["bP"] = p * dpb + TINY_P * fa
    if dout is None:
        return r
    dO = dout
    aq, ak, adO = q.abs(), k.abs(), dO.abs()
    dP = dO @ v.t()
    edP = (D + 2) * U * (adO @ av.t())
    Ou = O if o_used is None else o_used
    Dv = (dO * O).sum(1, keepdim=True)
    b_d = ((adO * (Ou - O).abs()).sum(1, keepdim=True) + (p * (dpb * dP.abs() + edP)).sum(1, keepdim=True)
           + (Skv + D + 8) * U * ((dO * Ou).abs().sum(1, keepdim=True) + (p * dP.abs()).sum(1, keepdim=True)))
    dS = p * (dP - Dv)
    e_ds = p * ((dpb + 3 * U + u) * (dP - Dv).abs() + (1 + u) * (edP + b_d)) + TINY_P * fa * (dP.abs() + Dv.abs())
    dQ, dK, dV = scale * (dS @ k), scale * (dS.t() @ q), p.t() @ dO
    r["dQ"], r["dK"], r["dV"] = dQ, dK, dV
    r["bdQ"] = scale * (e_ds @ ak + (Skv + 18) * U * (dS.abs() @ ak))
    r["bdK"] = scale * (e_ds.t() @ aq + (Sq + 18) * U * (dS.abs().t() @ aq))
    r["bdV"] = (p * (dpb + u)).t() @ adO + (Sq + 18) * U * (p.t() @ adO) + TINY_P * (fa.t() @ adO)
    return r


def _attn_ref(q, k, v, scale, causal, kmask=None, mask=None, dout=None, o_used=None, lse_used=None, probs=False):
    """_attn_bh over every (batch, head), one at a time on the reference device.  q [Bq, Sq, H, D] (Bq = 1: the
    queries are shared across the batch), k / v [B, Skv, H, D], dout / o_used [B, Sq, H, D] bf16; kmask [B, Skv] and
    mask [B, Sq, Skv] as the kernels read them (1 = attend); causal is top-left (j <= i); lse_used [B, H, Sq].
    Returns CPU float64 tensors [B, H, ...]."""
    B, Skv, H, D = k.shape
    Sq = q.shape[1]
    dev = _refdev()
    scale = float(torch.tensor(scale, dtype=F32))
    base = torch.ones(Sq, Skv, dtype=torch.bool, device=dev)
    if causal:
        base = base.tril()
    res = {}
    pick = lambda t, b, h: None if t is None else t[b, :, h].to(dev).to(F64)  # noqa: E731
    for b in range(B):
        allow = base
        if kmask is not None:
            allow = allow & kmask[b].to(dev).bool().view(1, Skv)
        if mask is not None:
            allow = allow & mask[b].to(dev).bool()
        for h in range(H):
            r = _attn_bh(pick(q, b if q.shape[0] > 1 else 0, h), pick(k, b, h), pick(v, b, h), allow, scale,
                         dout=pick(dout, b, h), o_used=pick(o_used, b, h),
                         lse_used=None if lse_used is None else lse_used[b, h].to(dev).to(F64), probs=probs)
            for name, val in r.items():
                if name not in res:
                    res[name] = torch.empty((B, H) + tuple(val.shape), dtype=val.dtype)
                res[name][b, h] = val.cpu()
    return res


def _rows(t):
    """[B, H, S, D] -> the kernels' [B*S, H*D] row layout."""
    B, H, S, D = t.shape
    return t.permute(0, 2, 1, 3).reshape(B * S, H * D)


def _attn_qkvd(case, g, B, Bq, Sq, Skv, H, D, scale):
    """q [Bq, Sq, H, D], k / v [B, Skv, H, D], dO [B, Sq, H, D] in bf16: N(0, 0.7^2), moved by case["inputs"]:
      flat     as drawn (scores of standard deviation ~0.5: the running max barely moves);
      peaked   q scaled to a score standard deviation of 10, so the scores span about +-30 and most 2^(s - m) underflow;
      rising   a shared direction (column 0 of every head): q_i0 = 4 and k_j0 a per-key offset growing with j, so the
               running max climbs in every 64-key block (by 3 per block, at most 40 over the row);
      falling  the same direction with a +8 offset on the first 64 keys only: the maximum lies in the first block;
      offset   V and dO shifted by 4: dP and D = rowsum(dO * O) share a large part that cancels in dP - D."""
    kind = case.get("inputs", "flat")
    q = torch.randn(Bq, Sq, H, D, generator=g) * 0.7
    k = torch.randn(B, Skv, H, D, generator=g) * 0.7
    v = torch.randn(B, Skv, H, D, generator=g) * 0.7
    do = torch.randn(B, Sq, H, D, generator=g) * 0.7
    if kind == "peaked":
        q = q * (10 / (scale * 0.49 * math.sqrt(D)))
    elif kind in ("rising", "falling"):
        q[..., 0] = 4.0
        j = torch.arange(Skv, dtype=F32)
        off = j * (min(3.0, 40.0 / _cdiv(Skv, 64)) / 64) if kind == "rising" else torch.where(j < 64, 8.0, 0.0)
        k[..., 0] = (off / (4.0 * scale)).view(1, Skv, 1)
    elif kind == "offset":
        v, do = v + 4.0, do + 4.0
    else:
        assert kind == "flat", kind
    return q.to(BF), k.to(BF), v.to(BF), do.to(BF)


def _key_mask(case, g, B, S):
    """uint8 [B, S] key mask: ~80 % of the keys visible, key 0 visible, the last key of sequence 0 masked (a masked key
    in the last, partial block), then case["kmask"]:
      late   no visible key before 197 (the first lies several 64-key blocks in);
      holes  keys 64..191 masked (whole blocks between visible keys);
      empty  the last sequence has no visible key;
      key0   key 0 masked (with causal: row 0 sees no key, the later rows do)."""
    m = (torch.rand(B, S, generator=g) < 0.8).to(torch.uint8)
    m[:, 0] = 1
    m[0, -1] = 0
    kind = "rand" if case["kmask"] is True else case["kmask"]
    if kind == "late":
        m[:, :197] = 0
        m[:, -1] = 1
    elif kind == "holes":
        m[:, 64:192] = 0
    elif kind == "empty":
        m[-1] = 0
    elif kind == "key0":
        m[:, 0] = 0
    else:
        assert kind == "rand", kind
    return m


def _packed_inputs(case):
    """The packed self-attention operands: qkv bf16 [B*S, 3*H*64], kmask (or None), dO [B*S, H*64], and the
    [B, S, H, 64] q, k, v, dO the reference takes."""
    g = _gen(case)
    B, S, H = case["B"], case["S"], case["H"]
    q, k, v, do = _attn_qkvd(case, g, B, B, S, S, H, 64, case.get("scale", 0.125))
    km = _key_mask(case, g, B, S) if case.get("kmask") else None
    qkv = torch.cat([t.reshape(B * S, H * 64) for t in (q, k, v)], 1)
    return qkv, km, do.reshape(B * S, H * 64), (q, k, v, do)


def _bound_bf16(o, name, got, ref, bound):
    """A bf16 attention output: the derived bound of its computation, plus its final rounding u * |ref|."""
    o.bound(name, got, ref, bound, rnd=u * ref.abs())


def _check_lse(o, lse, r):
    vis = r["vis"].reshape(-1)
    got = lse.detach().cpu().reshape(-1)
    o.bound("lse", got[vis], r["lse"].reshape(-1)[vis], r["blse"].reshape(-1)[vis])
    o.exact("lse_empty", got[~vis], torch.full((int((~vis).sum()),), float("-inf")))


def _packed_fwd(impl, device, case, qkv, km):
    B, S, H = case["B"], case["S"], case["H"]
    out = torch.full((B * S, H * 64), NAN, dtype=BF, device=device)
    lse = torch.full((B * H * S,), NAN, device=device)
    qd = qkv.to(device, copy=True)
    kd = None if km is None else km.to(device, copy=True)
    if km is not None:
        impl.attention_fwd_kmask(qd, out, lse, kd, B, S, H, case["causal"], case.get("scale", 0.125))
    else:
        impl.attention_fwd(qd, out, lse, B, S, H, case["causal"], case.get("scale", 0.125))
    return qd, kd, out, lse


def _check_attention_fwd(impl, device, case, op):
    o = _Out(op)
    B, S, H = case["B"], case["S"], case["H"]
    qkv, km, _, (q, k, v, _) = _packed_inputs(case)
    _, _, out, lse = _packed_fwd(impl, device, case, qkv, km)
    r = _attn_ref(q, k, v, case.get("scale", 0.125), case["causal"], kmask=km)
    _bound_bf16(o, "out", out, _rows(r["O"]), _rows(r["bO"]))
    _check_lse(o, lse, r)
    return o.rec


def check_attention_fwd(impl, device, case):
    return _check_attention_fwd(impl, device, case, "attention_fwd")


def check_attention_fwd_kmask(impl, device, case):
    return _check_attention_fwd(impl, device, case, "attention_fwd_kmask")


def _check_attention_bwd(impl, device, case, op):
    """The backward of the implementation's own forward: D and p are formed from the O and lse that forward wrote, so
    the bound takes their actual errors."""
    o = _Out(op)
    B, S, H, causal, scale = case["B"], case["S"], case["H"], case["causal"], case.get("scale", 0.125)
    d = H * 64
    qkv, km, dout, (q, k, v, do) = _packed_inputs(case)
    qd, kd, out, lse = _packed_fwd(impl, device, case, qkv, km)
    dqkv = torch.full((B * S, 3 * d), NAN, dtype=BF, device=device)
    if km is not None:
        impl.attention_bwd_kmask(qd, out, dout.to(device, copy=True), lse, dqkv, kd, B, S, H, causal, scale)
    else:
        impl.attention_bwd(qd, out, dout.to(device, copy=True), lse, dqkv, B, S, H, causal, scale)
    r = _attn_ref(q, k, v, scale, causal, kmask=km, dout=do, o_used=out.cpu().view(B, S, H, 64),
                  lse_used=lse.cpu().view(B, H, S))
    got = dqkv.cpu()
    for i, name in enumerate(("dq", "dk", "dv")):
        _bound_bf16(o, name, got[:, i * d:(i + 1) * d], _rows(r["d" + name[1].upper()]),
                    _rows(r["bd" + name[1].upper()]))
    return o.rec


def check_attention_bwd(impl, device, case):
    return _check_attention_bwd(impl, device, case, "attention_bwd")


def check_attention_bwd_kmask(impl, device, case):
    return _check_attention_bwd(impl, device, case, "attention_bwd_kmask")


def check_attention_probs(impl, device, case):
    o = _Out("attention_probs")
    B, S, H, causal, scale = case["B"], case["S"], case["H"], case["causal"], case.get("scale", 0.125)
    qkv, km, _, (q, k, v, _) = _packed_inputs(case)
    qd, kd, _, lse = _packed_fwd(impl, device, case, qkv, km)
    probs = torch.full((B, H, S, S), NAN, device=device)
    impl.attention_probs(qd, lse, kd, probs, B, S, H, causal, scale)
    r = _attn_ref(q, k, v, scale, causal, kmask=km, lse_used=lse.cpu().view(B, H, S), probs=True)
    o.bound("probs", probs, r["P"], r["bP"])
    return o.rec


def _mask_kind(case):
    """A general case's mask: None, "kpad" ([B, Skv]; True is its short form) or "full" ([B, Sq, Skv])."""
    m = case.get("mask")
    return "kpad" if m is True else m


def _generic_inputs(case):
    """Operands of the general kernels.  case: B, Sq, Skv, H, hd; scale (default 1/sqrt(hd)); causal; mask "kpad"
    ([B, Skv], with keys hide = (lo, hi) masked) or "full" ([B, Sq, Skv] with query row 1 of batch 0 empty); shared_q
    (bsq = 0); pitch (q rows in a wider buffer, k / v the halves of one packed [B*Skv, 2*H*hd] buffer)."""
    g = _gen(case)
    B, Sq, Skv, H, hd = case["B"], case["Sq"], case["Skv"], case["H"], case["hd"]
    scale = case.get("scale", 1 / math.sqrt(hd))
    Bq = 1 if case.get("shared_q") else B
    q, k, v, do = _attn_qkvd(case, g, B, Bq, Sq, Skv, H, hd, scale)
    mask = None
    if _mask_kind(case) == "kpad":
        mask = (torch.rand(B, Skv, generator=g) < 0.7).to(torch.uint8)
        mask[:, 0] = 1
        if "hide" in case:
            mask[:, case["hide"][0]:case["hide"][1]] = 0
    elif _mask_kind(case) == "full":
        mask = (torch.rand(B, Sq, Skv, generator=g) < 0.7).to(torch.uint8)
        mask[:, :, 0] = 1
        mask[0, min(1, Sq - 1)] = 0
    return scale, q, k, v, do, mask


def _generic_call(case, device, q, k, v, mask):
    """Device buffers and keyword arguments of one general-attention call."""
    B, Sq, Skv, H, hd = case["B"], case["Sq"], case["Skv"], case["H"], case["hd"]
    d = H * hd
    Bq = q.shape[0]
    pad = 64 if case.get("pitch") else 0
    qb = torch.zeros(Bq * Sq, d + pad, dtype=BF)
    qb[:, :d] = q.reshape(Bq * Sq, d)
    qd = qb.to(device)[:, :d]
    if case.get("pitch"):
        kv = torch.cat([k.reshape(B * Skv, d), v.reshape(B * Skv, d)], 1).to(device)
        kd, vd = kv[:, :d], kv[:, d:]
    else:
        kd, vd = k.reshape(B * Skv, d).to(device), v.reshape(B * Skv, d).to(device)
    md = None if mask is None else mask.to(device, copy=True)
    kw = dict(B=B, Sq=Sq, Skv=Skv, H=H, head_dim=hd, bsq=0 if Bq == 1 and case.get("shared_q") else Sq * qd.stride(0),
              bsk=Skv * kd.stride(0), bsv=Skv * vd.stride(0), bso=Sq * d,
              scale=case.get("scale", 1 / math.sqrt(hd)), mask=md,
              mask_bs=0 if mask is None else mask[0].numel(), mask_qs=Skv if _mask_kind(case) == "full" else 0,
              causal=case.get("causal", False))
    return qd, kd, vd, kw


def _check_generic_fwd(impl, device, case, op):
    o = _Out(op)
    B, Sq, H, hd = case["B"], case["Sq"], case["H"], case["hd"]
    scale, q, k, v, _, mask = _generic_inputs(case)
    qd, kd, vd, kw = _generic_call(case, device, q, k, v, mask)
    out = torch.full((B * Sq, H * hd), NAN, dtype=BF, device=device)
    getattr(impl, op)(qd, kd, vd, out, **kw)
    kp = mask if _mask_kind(case) == "kpad" else None
    fm = mask if _mask_kind(case) == "full" else None
    r = _attn_ref(q, k, v, scale, case.get("causal", False), kmask=kp, mask=fm)
    _bound_bf16(o, "out", out, _rows(r["O"]), _rows(r["bO"]))
    if op == "attention_fwd_decode" and hasattr(impl, "attention_decode_splits"):
        assert impl.attention_decode_splits(B, H, case["Skv"]) == case.get("splits", 1), case
    return o.rec


def check_attention_fwd_generic(impl, device, case):
    return _check_generic_fwd(impl, device, case, "attention_fwd_generic")


def check_attention_fwd_decode(impl, device, case):
    """Also asserts, on the kernel, the number of key splits the case was built to exercise (one unless it names
    more)."""
    return _check_generic_fwd(impl, device, case, "attention_fwd_decode")


def check_attention_bwd_generic(impl, device, case):
    """Batch-shared queries (shared_q) return their gradient summed over the batch in dq_f32, which starts non-zero:
    dq_f32 = init + sum_b dQ_b in fp32, (B + 2)*U*(sum_b |dQ_b| + |init|) for the adds on top of each dQ_b's own bound."""
    o = _Out("attention_bwd_generic")
    B, Sq, Skv, H, hd = case["B"], case["Sq"], case["Skv"], case["H"], case["hd"]
    d = H * hd
    scale, q, k, v, do, mask = _generic_inputs(case)
    qd, kd, vd, kw = _generic_call(case, device, q, k, v, mask)
    shared = bool(case.get("shared_q"))
    dqb = torch.full((qd.shape[0], qd.stride(0)), NAN, dtype=BF, device=device)
    dkv = torch.full((B * Skv, kd.stride(0)), NAN, dtype=BF, device=device)
    dk = dkv[:, :d]
    dv = dkv[:, d:] if case.get("pitch") else torch.full((B * Skv, d), NAN, dtype=BF, device=device)
    dq32_0 = torch.randn(Sq, d, generator=_gen(case)) if shared else None
    dq32 = None if dq32_0 is None else dq32_0.to(device, copy=True)
    impl.attention_bwd_generic(qd, kd, vd, do.reshape(B * Sq, d).to(device, copy=True), dk, dv,
                               dq=None if shared and B > 1 else dqb[:, :d], dq_f32=dq32, **kw)
    kp = mask if _mask_kind(case) == "kpad" else None
    fm = mask if _mask_kind(case) == "full" else None
    r = _attn_ref(q, k, v, scale, case.get("causal", False), kmask=kp, mask=fm, dout=do)
    if shared:
        dq_sum = d64(dq32_0) + _rows(r["dQ"].sum(0, keepdim=True))
        b = _rows(r["bdQ"].sum(0, keepdim=True)) \
            + (B + 2) * U * (_rows(r["dQ"].abs().sum(0, keepdim=True)) + d64(dq32_0).abs())
        o.bound("dq_f32", dq32, dq_sum, b)
    if not shared or B == 1:
        _bound_bf16(o, "dq", dqb[:, :d], _rows(r["dQ"]), _rows(r["bdQ"]))
    _bound_bf16(o, "dk", dk, _rows(r["dK"]), _rows(r["bdK"]))
    _bound_bf16(o, "dv", dv, _rows(r["dV"]), _rows(r["bdV"]))
    return o.rec


# Attention cases.  Lengths sit at the kernels' switches: packed self-attention runs resident kernels at S <= 384
# (a staged backward at S <= 224) and streamed ones above; 64-key blocks and 128-row tiles end partially at 17, 65,
# 129, 225, 385, 577, 1025, 4097.  B*H = 144 > 132 SMs makes CTAs loop over (batch, head) items.  The general kernels
# switch from resident to streamed at S = 512 / 336 / 256 for head_dim 64 / 96 / 128.  The decode kernel runs one
# split (with the direct bf16 store) up to Skv = 319 at any B*H, two uneven splits of 5 and 4 key blocks at
# Skv = 513 and small B*H, and 61 splits of 17 blocks (the last short) at Skv = 65573, B = H = 1 (the 64-split cap).
# Every op has scales that are not powers of two (0.1, 0.3, 1/sqrt(96), 1/sqrt(128)) in at least a third of its cases.
_PACKED = [
    {"B": 2, "S": 40, "H": 2, "causal": True},
    {"B": 2, "S": 1, "H": 2, "causal": False, "scale": 0.1},
    {"B": 2, "S": 17, "H": 2, "causal": True, "inputs": "peaked"},
    {"B": 1, "S": 64, "H": 2, "causal": False, "scale": 0.3, "inputs": "rising"},
    {"B": 2, "S": 65, "H": 1, "causal": True, "scale": 0.1, "inputs": "falling"},
    {"B": 1, "S": 129, "H": 2, "causal": False, "inputs": "rising"},
    {"B": 1, "S": 129, "H": 1, "causal": True, "scale": 0.1, "inputs": "offset"},
    {"B": 1, "S": 224, "H": 1, "causal": True, "scale": 0.3},
    {"B": 1, "S": 225, "H": 1, "causal": False, "scale": 0.1, "inputs": "peaked"},
    {"B": 2, "S": 384, "H": 3, "causal": True, "inputs": "rising", "gpu": True},
    {"B": 2, "S": 385, "H": 2, "causal": False, "scale": 0.1, "inputs": "peaked", "gpu": True},
    {"B": 1, "S": 577, "H": 2, "causal": True, "scale": 0.3, "inputs": "falling", "gpu": True},
    {"B": 1, "S": 1025, "H": 2, "causal": False, "inputs": "offset", "gpu": True},
    {"B": 1, "S": 4097, "H": 1, "causal": True, "scale": 0.1, "gpu": True},
    {"B": 12, "S": 65, "H": 12, "causal": True, "scale": 0.3, "gpu": True},
    {"B": 12, "S": 385, "H": 12, "causal": False, "inputs": "rising", "gpu": True},
]
_KMASKED = [
    {"B": 2, "S": 40, "H": 2, "causal": False, "kmask": True},
    {"B": 2, "S": 1, "H": 1, "causal": False, "kmask": "rand"},
    {"B": 2, "S": 17, "H": 1, "causal": True, "kmask": "key0", "scale": 0.3},
    {"B": 2, "S": 65, "H": 2, "causal": False, "kmask": "rand", "scale": 0.1},
    {"B": 3, "S": 129, "H": 1, "causal": False, "kmask": "empty", "scale": 0.3, "inputs": "rising"},
    {"B": 1, "S": 225, "H": 2, "causal": True, "kmask": "late", "inputs": "peaked"},
    {"B": 1, "S": 225, "H": 1, "causal": False, "kmask": "holes", "scale": 0.1, "inputs": "offset"},
    {"B": 2, "S": 385, "H": 2, "causal": True, "kmask": "key0", "scale": 0.3, "inputs": "falling", "gpu": True},
    {"B": 2, "S": 577, "H": 2, "causal": False, "kmask": "late", "scale": 0.1, "gpu": True},
    {"B": 2, "S": 1025, "H": 1, "causal": True, "kmask": "holes", "inputs": "rising", "gpu": True},
    {"B": 3, "S": 4097, "H": 1, "causal": True, "kmask": "empty", "scale": 0.1, "inputs": "offset", "gpu": True},
    {"B": 12, "S": 224, "H": 12, "causal": False, "kmask": "rand", "scale": 0.3, "inputs": "peaked", "gpu": True},
]
_GENERIC = [
    {"B": 2, "Sq": 16, "Skv": 40, "H": 2, "hd": 64, "mask": True},
    {"B": 2, "Sq": 16, "Skv": 40, "H": 2, "hd": 96},
    {"B": 2, "Sq": 16, "Skv": 40, "H": 2, "hd": 64, "mask": "kpad", "scale": 0.3},
    {"B": 2, "Sq": 33, "Skv": 70, "H": 1, "hd": 96, "mask": "full", "inputs": "peaked"},
    {"B": 1, "Sq": 70, "Skv": 33, "H": 2, "hd": 128, "causal": True, "inputs": "rising"},            # Sq > Skv
    {"B": 3, "Sq": 20, "Skv": 150, "H": 1, "hd": 64, "causal": True, "shared_q": True, "pitch": True,
     "inputs": "falling"},                                                                           # Sq < Skv
    {"B": 1, "Sq": 256, "Skv": 256, "H": 1, "hd": 128, "inputs": "offset", "scale": 0.1},           # resident
    {"B": 1, "Sq": 257, "Skv": 257, "H": 1, "hd": 128, "mask": "full", "causal": True},             # streamed
    {"B": 1, "Sq": 336, "Skv": 336, "H": 1, "hd": 96, "causal": True, "inputs": "rising"},          # resident
    {"B": 2, "Sq": 337, "Skv": 337, "H": 1, "hd": 96, "mask": "kpad", "pitch": True, "inputs": "offset"},
    {"B": 1, "Sq": 512, "Skv": 512, "H": 2, "hd": 64, "causal": True, "scale": 0.1, "gpu": True},
    {"B": 1, "Sq": 513, "Skv": 513, "H": 2, "hd": 64, "mask": "full", "inputs": "peaked", "gpu": True},
    {"B": 2, "Sq": 150, "Skv": 800, "H": 2, "hd": 64, "causal": True, "mask": "kpad", "scale": 0.3,
     "inputs": "rising", "gpu": True},                                                               # streamed, Sq < Skv
    {"B": 100, "Sq": 300, "Skv": 300, "H": 1, "hd": 128, "shared_q": True, "pitch": True, "gpu": True},  # 50 dQ chunks
]
_STREAMED = {  # mmb_attention_generic_streamed of each general case
    (16, 40, 64): 0, (16, 40, 96): 0, (33, 70, 96): 0, (70, 33, 128): 0, (20, 150, 64): 0, (256, 256, 128): 0, (257, 257, 128): 1,
    (336, 336, 96): 0, (337, 337, 96): 1, (512, 512, 64): 0, (513, 513, 64): 1, (150, 800, 64): 1, (300, 300, 128): 1}
_DECODE = [
    {"B": 2, "Sq": 3, "Skv": 100, "H": 2, "hd": 64, "mask": True},
    {"B": 2, "Sq": 1, "Skv": 1, "H": 2, "hd": 64, "splits": 1},
    {"B": 2, "Sq": 5, "Skv": 255, "H": 2, "hd": 96, "mask": "kpad", "scale": 0.1, "inputs": "rising", "splits": 1},
    {"B": 1, "Sq": 16, "Skv": 257, "H": 2, "hd": 128, "causal": True, "scale": 0.3, "inputs": "peaked", "splits": 1},
    {"B": 1, "Sq": 3, "Skv": 513, "H": 1, "hd": 64, "scale": 0.1, "inputs": "rising", "splits": 2},
    {"B": 2, "Sq": 4, "Skv": 513, "H": 2, "hd": 96, "mask": "kpad", "hide": (0, 320), "splits": 2},  # split 0 empty
    {"B": 1, "Sq": 1, "Skv": 65573, "H": 1, "hd": 64, "inputs": "rising", "splits": 61, "gpu": True},
    {"B": 1, "Sq": 16, "Skv": 65573, "H": 1, "hd": 128, "mask": "kpad", "hide": (3 * 1088, 11 * 1088), "scale": 0.1,
     "splits": 61, "gpu": True},
    {"B": 1, "Sq": 5, "Skv": 65573, "H": 1, "hd": 96, "causal": True, "scale": 0.3, "inputs": "peaked", "splits": 61,
     "gpu": True},                                                                                   # 60 empty splits
]
_PROBS = [
    {"B": 2, "S": 65, "H": 2, "causal": True, "kmask": "key0", "scale": 0.1},
    {"B": 1, "S": 129, "H": 1, "causal": False, "inputs": "peaked"},
    {"B": 2, "S": 40, "H": 1, "causal": False, "kmask": "empty", "scale": 0.3},
    {"B": 1, "S": 384, "H": 2, "causal": False, "kmask": "rand", "inputs": "rising", "gpu": True},
    {"B": 2, "S": 577, "H": 2, "causal": True, "kmask": "empty", "scale": 0.1, "gpu": True},
    {"B": 1, "S": 1025, "H": 1, "causal": True, "scale": 0.3, "inputs": "falling", "gpu": True},
]

# ---- temperature-scaled cross-entropy: materialised (loss.cu) and fused into the similarity GEMM (gemm.cu) ---------------
# The references are written from include/mmb200.h and contrastive_loss_with_temperature.py:81-107: logits
# x = exp(log_scale) * sims (T64 = exp(log_scale) in float64), row loss (1 - eps) (lse - x_label) + eps (lse - mean x),
# d loss / d sims = w T (softmax - t), t = (1 - eps) onehot(label) + eps / N, plus the other direction's transposed term
# on [col_lo, col_hi); d loss / d log_scale = sum (p - t) x = E_p[x] - (1 - eps) x_label - eps mean(x).
# Error terms of the bounds, each built from the row's (or element's) own values:
#   T       __expf(log_scale): (2 + floor(1.173 |log_scale|)) ulp (CUDA C++ Programming Guide, intrinsic functions);
#   x       the fp32 GEMM accumulation (K + 3) U sum|a||b| (as check_gemm) times T, plus x's own roundings;
#   exp     __expf(z) in loss.cu: (2 + floor(1.173 |z|)) ulp; ex2.approx in the GEMM epilogues: EX2, with the fmaf
#           argument a T2 - m2 (T2 = T log2e rounded) rounded once;
#   log     logf: 1 ulp (no fast-math);
#   merges  32 columns per lane and the two-level quad merge in EPI_CE_STATS (each level rescales by one ex2), the
#           ceil(n_parts / 32) + 5 chain of ce_stats_reduce, 256-thread block sums of ceil(N / 256) + 5 + 8 in loss.cu,
#           reduce_partials' ceil(rows / 8) + 8 + 1 for the scalar accumulators;
#   dscale  formed by cancellation: bounded with sum |terms|, never with the result.
_LS_CLIP, _LS_MAX = math.log(1 / 0.07), math.log(100.0)     # the initial logit scale and its clamp


def _expf_rel(z):
    """Relative error of __expf(z): the CUDA C++ Programming Guide bounds it by 2 + floor(1.173 |z|) ulp, and one ulp is
    at most 2^-23 of the value."""
    z = torch.as_tensor(z, dtype=F64)
    return (2 + torch.floor(1.173 * z.abs())) * 2 * U


def _f32(v):
    return float(torch.tensor(v, dtype=F32))


@contextlib.contextmanager
def _gemm_mode(impl, case):
    """Forces the GEMM kernel variant of case["gemm_mode"] (0: one CTA per 128 x 256 tile, 1: 2-CTA clusters) for the
    real kernels; the automatic choice takes clusters only at M >= 512 with enough tiles.  The emulation has one path."""
    if "gemm_mode" not in case or getattr(impl, "__name__", None) != "multimodal_b200.ops":
        yield
        return
    from multimodal_b200 import _lib

    assert _lib.lib().mmb_gemm_set_mode(case["gemm_mode"], 8) == 0
    try:
        yield
    finally:
        _lib.lib().mmb_gemm_set_mode(-1, 0)


def _pair(case, g, M, N, K, lab):
    """bf16 operands of a similarity GEMM, A [M, K] and B [N, K], of the kind case["inputs"]:
      norm  unit rows (the loss's L2-normalised embeddings);
      raw   N(0, 1) rows: logits of several hundred at the clamped temperature;
      peak  unit rows, A_i a noisy copy of B's row lab[i] (where that is a row of B): one column dominates its row;
      flat  unit rows, A scaled by 1e-3: a row's logits all but equal."""
    kind = case.get("inputs", "norm")
    A, Bm = torch.randn(M, K, generator=g), torch.randn(N, K, generator=g)
    if kind != "raw":
        A, Bm = A / A.norm(dim=1, keepdim=True), Bm / Bm.norm(dim=1, keepdim=True)
    if kind == "peak":
        ok = (lab >= 0) & (lab < N)
        A[ok] = Bm[lab[ok]] + 0.1 * A[ok]
        A = A / A.norm(dim=1, keepdim=True)
    elif kind == "flat":
        A = A * 1e-3
    else:
        assert kind in ("norm", "raw"), kind
    return A.to(BF), Bm.to(BF)


def _mask_weights(g, n, zero=(), one=()):
    """Masked-mean weights mask_i / count(mask) of a boolean row mask (contrastive_loss_with_temperature.py:97-100),
    ~70 % of the rows kept, the rows in `zero` dropped (weight 0) and those in `one` kept."""
    m = torch.rand(n, generator=g) < 0.7
    m[list(zero)] = False
    m[list(one)] = True
    return (m.to(F64) / m.sum()).to(F32)


def _gemm64(A, Bm):
    """float64 A B^T of bf16 operands and its fp32-accumulation bound (K + 3) U sum|a||b|, on the CPU."""
    dev = _refdev()
    a, b = d64(A).to(dev), d64(Bm).to(dev)
    return (a @ b.t()).cpu(), ((A.shape[1] + 3) * U * (a.abs() @ b.abs().t())).cpu()


def _exp_term_err(Wt, x, ex, L, e, t):
    """Error of one W (2^(a T2 - L log2e) - t) term of the EPI_CE_GRAD epilogue (or of W (__expf(x - L) - t) in
    loss.cu with ex = x's error): e = exp(x - L) in float64; the fmaf argument and L log2e round once each; W = lw T w
    carries T's error and two products."""
    rho = ex + 2 * U * L.abs() + U * (x - L).abs() + EX2 + _expf_rel(x - L)
    return Wt.abs() * (e * rho + U * (e + t) + TINY_P) + Wt.abs() * 3 * U * (e - t).abs()


def _sims(case, g, rows, N, off):
    """fp32 similarity rows [rows, ld] (the columns past N NaN: the kernels must not read them) of bf16 embeddings of
    width 64 in the case's input kind, the label column of row i at off + i."""
    A, Bm = _pair(case, g, rows, N, 64, off + torch.arange(rows))
    s = torch.full((rows, case.get("ld", N)), NAN)
    s[:, :N] = (d64(A) @ d64(Bm).t()).to(F32)
    return s


def _lse_stats(x, ex, k):
    """Row log-sum-exp of loss.cu over the fp32 logits with errors ex: the row max cancels (the same max enters the
    exponent and the result), each __expf(x - max) has its own relative error, the block sum k roundings, logf 1 ulp,
    the final add."""
    lse = torch.logsumexp(x, 1)
    p = torch.exp(x - lse[:, None])
    z = x - x.amax(1, keepdim=True)
    b = (p * (ex + U * z.abs() + _expf_rel(z))).sum(1) + k * U + 2 * U * (lse - x.amax(1)).abs() + U * lse.abs() \
        + x.shape[1] * TINY_P
    return lse, p, b


def check_contrastive_ce_stats(impl, device, case):
    o = _Out("contrastive_ce_stats")
    g = _gen(case)
    rows, N, off, eps, lw = case["rows"], case["N"], case.get("off", 0), _f32(case.get("eps", 0.0)), 0.5
    sims = _sims(case, g, rows, N, off)
    ls = torch.tensor([case.get("ls", _LS_CLIP)], dtype=F32)
    rw = _mask_weights(g, rows, zero=(0,), one=(rows - 1,)) if case.get("rw") else None
    d0 = torch.tensor([0.375])
    row_loss, lse = torch.full((rows,), NAN, device=device), torch.full((rows,), NAN, device=device)
    dscale = d0.to(device, copy=True)
    logits = torch.full(sims.shape, NAN, device=device) if case.get("logits") else None
    impl.contrastive_ce_stats(sims.to(device, copy=True), ls.to(device, copy=True), rows, N, off, eps, lw, row_loss,
                              lse, dscale, logits, None if rw is None else rw.to(device, copy=True))
    T64, eT = math.exp(ls.item()), _expf_rel(ls.item()).item()
    x = T64 * d64(sims)[:, :N]
    ex = (eT + 2 * U) * x.abs()                       # T's error and the product's rounding
    k = _cdiv(N, 256) + 5 + 8
    ar = torch.arange(rows)
    lab = off + ar
    lse64, p, b_lse = _lse_stats(x, ex, k)
    xl, mean = x[ar, lab], x.mean(1)
    b_mean = ex.mean(1) + (k + 1) * U * x.abs().mean(1)
    loss = (1 - eps) * (lse64 - xl) + eps * (lse64 - mean)
    b_loss = b_lse + ex[ar, lab] + eps * b_mean + 3 * U * (lse64.abs() + xl.abs() + mean.abs()) + U * loss.abs()
    wrow = d64(rw) if rw is not None else torch.full((rows,), 1.0 / rows, dtype=F64)
    if rw is not None:
        o.bound("row_loss", row_loss, loss * wrow * rows, b_loss * wrow * rows + 3 * U * (loss * wrow * rows).abs())
    else:
        o.bound("row_loss", row_loss, loss, b_loss)
    o.bound("lse", lse, lse64, b_lse)
    if logits is not None:
        got = logits.cpu()
        o.bound("logits", got[:, :N], x, ex)
        o.exact("logits_pad", got[:, N:], torch.full((rows, sims.shape[1] - N), NAN))
    # d loss / d log_scale: per row sum_j (p - t) x over the block chain, * lw * wrow, then reduce_partials and the +=
    t = torch.full((rows, N), eps / N, dtype=F64)
    t[ar, lab] += 1 - eps
    gl = p - t
    e_gl = p * (ex + b_lse[:, None] + U * (x - lse64[:, None]).abs() + _expf_rel(x - lse64[:, None])) + 2 * U * (p + t)
    part = (gl * x).sum(1) * lw * wrow
    b_part = ((e_gl * x.abs() + gl.abs() * ex).sum(1) + (k + 2) * U * (gl * x).abs().sum(1)) * lw * wrow \
        + 3 * U * part.abs()
    kr = _cdiv(rows, 8) + 8 + 1
    o.bound("dscale", dscale, d64(d0) + part.sum(), b_part.sum() + kr * U * (part.abs().sum() + abs(d0.item())))
    return o.rec


def check_contrastive_ce_grad(impl, device, case):
    """lse_row is the fp32-rounded float64 row LSE; lse_col that of the other direction's rows (here: the column's LSE
    over these rows, widened to N rows); col_w-weight-0 columns carry a non-finite lse_col when case["bad"]."""
    o = _Out("contrastive_ce_grad")
    g = _gen(case)
    rows, N, off, eps, lw = case["rows"], case["N"], case.get("off", 0), _f32(case.get("eps", 0.0)), 0.5
    sims = _sims(case, g, rows, N, off)
    ld = sims.shape[1]
    ls = torch.tensor([case.get("ls", _LS_CLIP)], dtype=F32)
    T64, eT = math.exp(ls.item()), _expf_rel(ls.item()).item()
    x = T64 * d64(sims)[:, :N]
    lse_row = torch.logsumexp(x, 1).to(F32)
    lse_col = (torch.logsumexp(x, 0) + math.log(N / rows)).to(F32)
    cw = rw = None
    if case.get("rw"):
        cw = _mask_weights(g, N, zero=(0, off), one=(off + rows - 1,))
        rw = cw[off:off + rows].clone()
        if case.get("bad"):
            z = (cw == 0).nonzero().view(-1)
            lse_col[z] = torch.tensor([NAN, float("-inf"), float("inf")])[torch.arange(z.numel()) % 3]
    lo, hi = {"none": (0, 0), "local": (off, off + rows), "global": (0, N),
              "inner": (off // 2 + 3, N - 5)}[case.get("mode", "global")]
    want = case.get("out", "both")
    dbf = torch.full((rows, ld), NAN, dtype=BF, device=device) if want != "f32" else None
    d32 = torch.full((rows, ld), NAN, device=device) if want != "bf16" else None
    tod = lambda t: None if t is None else t.to(device, copy=True)  # noqa: E731
    impl.contrastive_ce_grad(tod(sims), tod(ls), rows, N, off, eps, lw, tod(lse_row),
                             None if hi <= lo else tod(lse_col), lo, hi, dbf, d32, tod(rw), tod(cw))
    ar = torch.arange(rows)
    t = torch.full((rows, N), eps / N, dtype=F64)
    t[ar, off + ar] += 1 - eps
    ex = (eT + 2 * U) * x.abs()
    L1 = d64(lse_row)[:, None]
    W1 = (lw * T64 * (d64(rw) if rw is not None else torch.full((rows,), 1.0 / rows, dtype=F64)))[:, None]
    e1 = torch.exp(x - L1)
    ref = W1 * (e1 - t)
    err = _exp_term_err(W1, x, ex, L1, e1, t)
    j = torch.arange(N)
    W2 = lw * T64 * (d64(cw) if cw is not None else torch.full((N,), 1.0 / rows, dtype=F64))
    W2 = torch.where((j >= lo) & (j < hi), W2, torch.zeros((), dtype=F64))[None, :]
    L2 = torch.where(W2 != 0, d64(lse_col)[None, :], torch.zeros((), dtype=F64))
    e2 = torch.exp(x - L2)
    on = W2 != 0
    ref = ref + torch.where(on, W2 * (e2 - t), torch.zeros((), dtype=F64))
    err = err + torch.where(on, _exp_term_err(W2, x, ex, L2, e2, t), torch.zeros((), dtype=F64)) + U * ref.abs()
    if dbf is not None:
        got = dbf.cpu()
        o.bf16("dsims_bf16", got[:, :N], ref, err=err)
        o.exact("dsims_bf16_pad", got[:, N:], torch.full((rows, ld - N), NAN, dtype=BF))
    if d32 is not None:
        got = d32.cpu()
        o.bound("dsims_f32", got[:, :N], ref, err)
        o.exact("dsims_f32_pad", got[:, N:], torch.full((rows, ld - N), NAN))
    return o.rec


def _stats_launches(case, M):
    """The launches of one fused-statistics case: (first B row, label0, part0) each over N = case["N"] columns.  World 1:
    one launch with case["label0"] (default 0) at case["part0"] (default 0).  World W > 1 restates
    engine_loss.contrastive_schedule on rank `rank` (B = M = N): one launch per peer r over its column block,
    label0 = rank*B - r*B (negative, or >= N, when the label lies in another block), part0 = r * npp."""
    N, W = case["N"], case.get("world", 1)
    if W == 1:
        return [(0, case.get("label0", 0), case.get("part0", 0))]
    assert M == N
    rank, npp = case["rank"], _cdiv(N, 128)
    return [(r * N, rank * M - r * N, r * npp) for r in range(W)]


def check_gemm_ce_stats(impl, device, case):
    """Every float4 part {max, sum e^(x - max), sum e^(x - max) x, sum x} of every launch, the sums re-expressed
    relative to the float64 part maximum (the kernel's own maximum is checked first, so a part is compared at the scale
    it was formed at); parts no launch owns and xlabel entries whose label column no launch holds stay NaN."""
    from multimodal_b200 import _lib

    o = _Out("gemm_ce_stats")
    g = _gen(case)
    M, N, K, W = case["M"], case["N"], case["K"], case.get("world", 1)
    npp = _cdiv(N, 128)
    assert _lib.lib().mmb_gemm_ce_num_parts(N) == npp
    launches = _stats_launches(case, M)
    glab = torch.arange(M) + (case["rank"] * M if W > 1 else case.get("label0", 0))
    A, Bfull = _pair(case, g, M, W * N, K, glab)
    ls = torch.tensor([case.get("ls", _LS_CLIP)], dtype=F32)
    P = max(p0 for _, _, p0 in launches) + npp + 1                 # one spare part past the last launch's
    part = torch.full((M, P, 4), NAN, device=device)
    xlabel = torch.full((M,), NAN, device=device)
    Ad, lsd = A.to(device, copy=True), ls.to(device, copy=True)
    with _gemm_mode(impl, case):
        for b0, label0, part0 in launches:
            impl.gemm_ce_stats(Ad, Bfull[b0:b0 + N].to(device, copy=True), lsd, label0, part, part0, xlabel)
    got = part.cpu()
    g64 = got.to(F64)
    T64, eT = math.exp(ls.item()), _expf_rel(ls.item()).item()
    written = torch.zeros(M, P, dtype=torch.bool)
    cols = {k: ([], [], []) for k in ("max", "sum_e", "sum_ex", "sum_x")}    # got, ref, bound per part
    xl_ref, xl_b = torch.full((M,), NAN, dtype=F64), torch.zeros(M, dtype=F64)
    ar = torch.arange(M)
    for b0, label0, part0 in launches:
        acc, eacc = _gemm64(A, Bfull[b0:b0 + N])
        x = T64 * acc
        ex = T64 * eacc + (eT + 3 * U) * x.abs()
        for p in range(npp):
            xs, es = x[:, 128 * p:128 * (p + 1)], ex[:, 128 * p:128 * (p + 1)]
            q = g64[:, part0 + p]
            written[:, part0 + p] = True
            mref, m = xs.amax(1), q[:, 0]
            R = xs.abs().amax(1)
            cols["max"][0].append(m), cols["max"][1].append(mref)
            cols["max"][2].append(es.amax(1) + 5 * U * mref.abs())
            e = torch.exp(xs - m[:, None])
            rho = es + U * (xs - m[:, None]).abs() + 3 * U * m.abs()[:, None] + EX2
            merge = 32 * U + 2 * (EX2 + 3 * U + 2 * U * R)
            shift = torch.exp(m - mref)
            eref = torch.exp(xs - mref[:, None])
            for name, val, ref, b in (
                    ("sum_e", q[:, 1], eref.sum(1), (e * rho).sum(1) + merge * e.sum(1) + 128 * TINY_P),
                    ("sum_ex", q[:, 2], (eref * xs).sum(1),
                     (e * (rho * xs.abs() + es)).sum(1) + (merge + U) * (e * xs.abs()).sum(1) + 128 * TINY_P * R)):
                cols[name][0].append(val * shift), cols[name][1].append(ref), cols[name][2].append(b * shift)
            cols["sum_x"][0].append(q[:, 3]), cols["sum_x"][1].append(xs.sum(1))
            cols["sum_x"][2].append(es.sum(1) + 34 * U * xs.abs().sum(1))
        lab = label0 + ar
        hit = (lab >= 0) & (lab < N)
        xl_ref[hit], xl_b[hit] = x[ar[hit], lab[hit]], ex[ar[hit], lab[hit]]
    for name, (gv, rv, bv) in cols.items():
        o.bound(name, torch.stack(gv, 1), torch.stack(rv, 1), torch.stack(bv, 1))
    o.exact("untouched", got[~written], torch.full((int((~written).sum()), 4), NAN))
    has = ~torch.isnan(xl_ref)
    gx = xlabel.cpu()
    o.bound("xlabel", gx[has], xl_ref[has], xl_b[has])
    o.exact("xlabel_untouched", gx[~has], torch.full((int((~has).sum()),), NAN))
    return o.rec


def _logit_rows(case, g, rows, N, lab):
    """float64 logits [rows, N] of the kind case["inputs"]: norm (the clamped-free CLIP scale times cosine similarities
    of 64-wide unit rows), raw (N(0, 30^2)), peak (norm plus 60 at the label column), flat (14.3 + 1e-3 N(0, 1))."""
    kind = case.get("inputs", "norm")
    z = torch.randn(rows, N, generator=g, dtype=F64)
    if kind == "raw":
        return 30 * z
    if kind == "flat":
        return 14.3 + 1e-3 * z
    x = z / 8 / 0.07
    if kind == "peak":
        x[torch.arange(rows), lab] += 60
    else:
        assert kind == "norm", kind
    return x


def check_ce_stats_reduce(impl, device, case):
    """Parts formed in float64 per 128 columns of each of `world` launches of B columns (n_parts = world * npp,
    n_total = world * B), rounded to fp32: the reduce's own contract, apart from the GEMM's.  A spare part past n_parts
    is NaN and must not be read."""
    o = _Out("ce_stats_reduce")
    g = _gen(case)
    rows, B, W, eps, lw = case["rows"], case["B"], case.get("world", 1), _f32(case.get("eps", 0.0)), 0.5
    N, npp = W * B, _cdiv(B, 128)
    n_parts = W * npp
    ar = torch.arange(rows)
    lab = (min(1, W - 1) * rows + ar) % N
    x = _logit_rows(case, g, rows, N, lab)
    parts = []
    for r in range(W):
        for p in range(npp):
            xs = x[:, r * B + 128 * p:r * B + min(128 * (p + 1), B)]
            m = xs.amax(1)
            e = torch.exp(xs - m[:, None])
            parts.append(torch.stack([m, e.sum(1), (e * xs).sum(1), xs.sum(1)], -1))
    part = torch.full((rows, n_parts + 1, 4), NAN)
    part[:, :n_parts] = torch.stack(parts, 1).to(F32)
    xl = x[ar, lab].to(F32)
    rw = _mask_weights(g, rows, zero=(0,), one=(rows - 1,)) if case.get("rw") else None
    d0 = torch.tensor([0.375])
    row_loss, lse = torch.full((rows,), NAN, device=device), torch.full((rows,), NAN, device=device)
    dscale = d0.to(device, copy=True)
    tod = lambda t: None if t is None else t.to(device, copy=True)  # noqa: E731
    impl.ce_stats_reduce(tod(part), n_parts, tod(xl), rows, N, eps, lw, tod(rw), row_loss, lse, dscale)
    m, y, z, w = d64(part[:, :n_parts]).unbind(-1)
    mx = m.amax(1, keepdim=True)
    f = torch.exp(m - mx)
    S = (y * f).sum(1)
    lse64 = mx.squeeze(1) + torch.log(S)
    Ex = (z * f).sum(1) / S
    mean = w.sum(1) / N
    xl64 = d64(xl)
    kc = _cdiv(n_parts, 32) + 5
    eta = _expf_rel(m - mx) + U * (m - mx).abs() + U
    rel_S = (y * f * eta).sum(1) / S + kc * U
    b_lse = rel_S + 2 * U * torch.log(S).abs() + U * lse64.abs()
    ez = z.abs() * f
    b_E = ((ez * eta).sum(1) + kc * U * ez.sum(1)) / S + Ex.abs() * rel_S + 2 * U * Ex.abs()
    b_mean = (kc + 1) * U * w.abs().sum(1) / N
    loss = (1 - eps) * (lse64 - xl64) + eps * (lse64 - mean)
    b_loss = b_lse + eps * b_mean + 3 * U * (lse64.abs() + xl64.abs() + mean.abs()) + U * loss.abs()
    wrow = d64(rw) if rw is not None else torch.full((rows,), 1.0 / rows, dtype=F64)
    if rw is not None:
        o.bound("row_loss", row_loss, loss * wrow * rows, b_loss * wrow * rows + 3 * U * (loss * wrow * rows).abs())
    else:
        o.bound("row_loss", row_loss, loss, b_loss)
    o.bound("lse", lse, lse64, b_lse)
    dpart = (Ex - (1 - eps) * xl64 - eps * mean) * lw * wrow
    b_dp = (b_E + eps * b_mean + 3 * U * (Ex.abs() + xl64.abs() + mean.abs())) * lw * wrow + 3 * U * dpart.abs()
    kr = _cdiv(rows, 8) + 8 + 1
    o.bound("dscale", dscale, d64(d0) + dpart.sum(), b_dp.sum() + kr * U * (dpart.abs().sum() + abs(d0.item())))
    return o.rec


def check_gemm_ce_grad(impl, device, case):
    """engine_loss.contrastive_schedule's gradient launches on rank `rank` of `world` (B rows, N = world * B): one per
    peer block r with label0 = rank*B - r*B, the transposed range clipped to the block and lse_col / col_w sliced to
    it, each writing a column slice of one NaN-filled dsims buffer wider than [B, N] in both dimensions.  lse_row and
    lse_col are the fp32-rounded float64 row LSEs of the two directions.  case["refused"]: a launch over an N that is
    not a multiple of 8 (a bf16 output) raises MMBError and writes nothing."""
    from multimodal_b200._lib import MMBError

    o = _Out("gemm_ce_grad")
    g = _gen(case)
    B, K, W = case["B"], case["K"], case.get("world", 1)
    rank = case.get("rank", 0)
    N, lab = W * B, rank * B
    eps, lw = _f32(case.get("eps", 0.0)), 0.5
    a_all, b_all = _pair(case, g, N, N, K, torch.arange(N))
    A = a_all[lab:lab + B]
    ls = torch.tensor([case.get("ls", _LS_CLIP)], dtype=F32)
    T64, eT = math.exp(ls.item()), _expf_rel(ls.item()).item()
    acc, eacc = _gemm64(A, b_all)
    x = T64 * acc
    lse_row = torch.logsumexp(x, 1).to(F32)
    lse_col = torch.logsumexp(T64 * _gemm64(b_all, a_all)[0], 1).to(F32)
    cw = rw = None
    if case.get("rw"):
        cw = torch.cat([_mask_weights(g, B, zero=(0,), one=(B - 1,)) for _ in range(W)])
        rw = cw[lab:lab + B].clone()
        if case.get("bad"):
            z = (cw == 0).nonzero().view(-1)
            lse_col[z] = torch.tensor([NAN, float("-inf"), float("inf")])[torch.arange(z.numel()) % 3]
    mode = case.get("mode", "global")
    lo, hi = {"none": (0, 0), "local": (lab, lab + B), "global": (0, N), "inner": (lab // 2 + 3, N - 5)}[mode]
    tod = lambda t: None if t is None else t.to(device, copy=True)  # noqa: E731
    Ad, lsd, lrd, rwd, cwd = tod(A), tod(ls), tod(lse_row), tod(rw), tod(cw)
    LBd = None if mode == "none" else tod(lse_col)
    DS = torch.full((B + 3, N + 16), NAN, dtype=BF, device=device)
    if case.get("refused"):
        try:
            impl.gemm_ce_grad(Ad, tod(b_all), lsd, lab, N, B, eps, lw, lrd, rwd, LBd, cwd, lo, hi, DS[:B, :N])
        except MMBError:
            o.exact("untouched", DS.cpu(), torch.full(DS.shape, NAN, dtype=BF))
            return o.rec
        raise AssertionError(f"gemm_ce_grad accepted a bf16 output of {N} columns")
    with _gemm_mode(impl, case):
        for r in range(W):
            c0 = r * B
            clo, chi = min(max(lo - c0, 0), B), min(max(hi - c0, 0), B)
            sl = slice(c0, c0 + B)
            impl.gemm_ce_grad(Ad, tod(b_all[sl]), lsd, lab - c0, N, B, eps, lw, lrd, rwd,
                              LBd[sl] if (LBd is not None and chi > clo) else None,
                              cwd[sl] if cwd is not None else None, clo, chi, DS[:B, sl])
    ar = torch.arange(B)
    t = torch.full((B, N), eps / N, dtype=F64)
    t[ar, lab + ar] += 1 - eps
    ex = T64 * eacc + (eT + 3 * U) * x.abs()
    L1 = d64(lse_row)[:, None]
    W1 = (lw * T64 * (d64(rw) if rw is not None else torch.full((B,), 1.0 / B, dtype=F64)))[:, None]
    e1 = torch.exp(x - L1)
    ref = W1 * (e1 - t)
    err = _exp_term_err(W1, x, ex, L1, e1, t)
    j = torch.arange(N)
    W2 = lw * T64 * (d64(cw) if cw is not None else torch.full((N,), 1.0 / B, dtype=F64))
    W2 = torch.where((j >= lo) & (j < hi), W2, torch.zeros((), dtype=F64))[None, :]
    on = W2 != 0
    L2 = torch.where(on, d64(lse_col)[None, :], torch.zeros((), dtype=F64))
    e2 = torch.exp(x - L2)
    ref = ref + torch.where(on, W2 * (e2 - t), torch.zeros((), dtype=F64))
    err = err + torch.where(on, _exp_term_err(W2, x, ex, L2, e2, t), torch.zeros((), dtype=F64)) + U * ref.abs()
    got = DS.cpu()
    o.bf16("dsims", got[:B, :N], ref, err=err)
    o.exact("untouched", torch.cat([got[B:].reshape(-1), got[:B, N:].reshape(-1)]),
            torch.full((3 * (N + 16) + 16 * B,), NAN, dtype=BF))
    return o.rec


def check_linear_cross_entropy(impl, device, case):
    """Linear (no bias) -> CrossEntropy(ignore_index) over a vocabulary: the fused statistics GEMM with explicit labels
    (T = __expf(0)) and ce_labels_reduce.  Its lse carries the EPI_CE_STATS errors (per-element x and ex2 errors, the
    max mismatch m2 ln2 vs the stored max, 32 + quad-merge roundings) and the reduce's (__expf of m_p - max, its
    ceil(n_parts / 32) + 5 chain, logf)."""
    o = _Out("linear_cross_entropy")
    g = _gen(case)
    M, V, K, ignore = case["M"], case["V"], case["K"], case.get("ignore", -100)
    h = torch.randn(M, K, generator=g).to(BF)
    w = (torch.randn(V, K, generator=g) * (3.0 / math.sqrt(K))).to(BF)
    lab = torch.randint(1 if ignore == 0 else 0, V, (M,), generator=g)
    lab[0] = V - 1
    nig = M if case.get("n_ignored") == "all" else case.get("n_ignored", 0)
    lab[torch.randperm(M, generator=g)[:nig]] = ignore
    acc0 = torch.tensor([1.5, 2.0])
    accum = acc0.to(device, copy=True)
    row_loss = torch.full((M,), NAN, device=device)
    with _gemm_mode(impl, case):
        impl.linear_cross_entropy(h.to(device, copy=True), w.to(device, copy=True),
                                  lab.to(torch.int32).to(device), ignore, accum, row_loss)
    x, eacc = _gemm64(h, w)
    ex = eacc + (_expf_rel(0.0).item() + 3 * U) * x.abs()
    keep = lab != ignore
    lse = torch.logsumexp(x, 1)
    p = torch.exp(x - lse[:, None])
    mx, R = x.amax(1), x.abs().amax(1)
    span = mx - x.amin(1)
    kc = _cdiv(_cdiv(V, 128), 32) + 5
    b_lse = (p * ex).sum(1) + U * span + 3 * U * R + EX2 + 32 * U + 2 * (EX2 + 3 * U + 2 * U * R) \
        + _expf_rel(span) + U * span + U + kc * U + 2 * U * (lse - mx).abs() + U * lse.abs() + V * TINY_P
    ar = torch.arange(M)
    lc = lab.clamp(0, V - 1)
    xl = x[ar, lc]
    zero = torch.zeros((), dtype=F64)
    nll = torch.where(keep, lse - xl, zero)
    b_row = torch.where(keep, b_lse + ex[ar, lc] + 2 * U * (lse.abs() + xl.abs()) + U * nll.abs(), zero)
    o.bound("row_loss", row_loss, nll, b_row)
    kr = _cdiv(M, 8) + 8 + 1
    o.bound("accum", accum, torch.stack([d64(acc0)[0] + nll.sum(), d64(acc0)[1] + keep.sum().to(F64)]),
            torch.stack([b_row.sum() + kr * U * (nll.abs().sum() + abs(acc0[0].item())), zero]))
    return o.rec


def _both_modes(cases):
    return [dict(c, gemm_mode=m) for c in cases for m in (0, 1)]


_CONTRASTIVE_STATS = [
    {"rows": 7, "N": 7, "off": 0, "eps": 0.1},
    {"rows": 5, "N": 256, "off": 251, "eps": 0.05, "rw": True, "ld": 264, "logits": True, "ls": _LS_MAX},
    {"rows": 9, "N": 300, "off": 100, "inputs": "raw", "logits": True},
    {"rows": 6, "N": 70, "off": 64, "eps": 0.1, "rw": True, "inputs": "peak", "ls": _LS_MAX, "ld": 77},
    {"rows": 4, "N": 600, "off": 596, "eps": 0.05, "inputs": "flat"},
    {"rows": 300, "N": 1024, "off": 724, "eps": 0.1},
    {"rows": 1000, "N": 4000, "off": 3000, "eps": 0.1, "gpu": True},
    {"rows": 257, "N": 1032, "rw": True, "inputs": "peak", "eps": 0.1, "ls": _LS_MAX, "logits": True, "gpu": True},
]
_CONTRASTIVE_GRAD = [
    {"rows": 6, "N": 20, "off": 8, "mode": "none", "eps": 0.1},
    {"rows": 6, "N": 20, "off": 8, "mode": "local", "rw": True, "out": "f32"},
    {"rows": 5, "N": 300, "off": 295, "mode": "global", "eps": 0.05, "rw": True, "bad": True, "ld": 304,
     "ls": _LS_MAX},
    {"rows": 8, "N": 256, "mode": "inner", "inputs": "peak", "eps": 0.1, "out": "bf16"},
    {"rows": 7, "N": 64, "off": 57, "mode": "global", "inputs": "raw", "rw": True, "bad": True},
    {"rows": 4, "N": 130, "off": 3, "mode": "global", "inputs": "flat"},
    {"rows": 300, "N": 1024, "off": 724, "mode": "global", "rw": True, "bad": True, "eps": 0.1, "gpu": True},
]
# M 1 .. 1000 and N 64 .. 1032 on both sides of the 128-column part and 256-column tile boundaries (N = 130: a second
# half of one column; N = 255: one half present in the last tile), K tails shorter than one 64-deep k-block, world 2 / 3
# launch sets, and a 2000 x 2600 case with more tiles than SMs in either mode (the persistent grid loops).
_GEMM_CE_STATS = _both_modes([
    {"M": 1, "N": 64, "K": 8},
    {"M": 127, "N": 130, "K": 72, "inputs": "raw", "label0": 3, "part0": 1},
    {"M": 129, "N": 255, "K": 136, "inputs": "peak", "ls": _LS_MAX},
    {"M": 64, "N": 64, "K": 72, "world": 3, "rank": 1, "inputs": "peak"},
    {"M": 130, "N": 130, "K": 8, "world": 2, "rank": 1, "inputs": "flat", "ls": _LS_MAX},
    {"M": 255, "N": 256, "K": 768, "gpu": True},
    {"M": 257, "N": 600, "K": 136, "inputs": "raw", "label0": -100, "gpu": True},
    {"M": 1000, "N": 1032, "K": 768, "inputs": "peak", "ls": _LS_MAX, "gpu": True},
    {"M": 264, "N": 264, "K": 136, "world": 3, "rank": 2, "gpu": True},
    {"M": 2000, "N": 2600, "K": 136, "gpu": True},
])
_CE_STATS_REDUCE = [
    {"rows": 5, "B": 200, "world": 3, "eps": 0.1},
    {"rows": 8, "B": 130, "world": 2, "rw": True, "inputs": "raw"},
    {"rows": 3, "B": 64, "eps": 0.05, "inputs": "peak"},
    {"rows": 6, "B": 1032, "world": 4, "eps": 0.1, "rw": True, "inputs": "flat"},       # 36 parts: two per lane
    {"rows": 1000, "B": 1032, "world": 2, "eps": 0.1, "gpu": True},
    {"rows": 300, "B": 4096, "world": 2, "rw": True, "eps": 0.05, "inputs": "raw", "gpu": True},
]
_GEMM_CE_GRAD = _both_modes([
    {"B": 64, "K": 72, "mode": "global", "eps": 0.1, "rw": True, "bad": True},
    {"B": 64, "K": 8, "world": 3, "rank": 1, "mode": "local", "eps": 0.05, "inputs": "peak"},
    {"B": 128, "K": 136, "world": 2, "rank": 1, "mode": "inner", "eps": 0.1, "rw": True, "bad": True, "ls": _LS_MAX},
    {"B": 136, "K": 72, "world": 2, "mode": "none", "inputs": "raw"},
    {"B": 64, "K": 72, "world": 2, "mode": "inner", "eps": 0.05},
    {"B": 8, "K": 8, "world": 3, "rank": 2, "mode": "global", "eps": 0.1, "inputs": "flat"},
    {"B": 256, "K": 768, "world": 2, "rank": 1, "mode": "global", "eps": 0.1, "rw": True, "bad": True, "gpu": True},
    {"B": 1032, "K": 136, "inputs": "peak", "ls": _LS_MAX, "gpu": True},
    {"B": 600, "K": 136, "world": 3, "rank": 2, "mode": "inner", "eps": 0.05, "inputs": "raw", "gpu": True},
    {"B": 2600, "K": 72, "mode": "local", "eps": 0.1, "gpu": True},
]) + [{"B": 255, "K": 72, "refused": True}]
_LINEAR_CE = _both_modes([
    {"M": 6, "V": 49408, "K": 8, "ignore": 0, "n_ignored": 2},
    {"M": 5, "V": 1001, "K": 72},
    {"M": 4, "V": 49408, "K": 72, "n_ignored": "all"},
    {"M": 127, "V": 255, "K": 136, "ignore": 0, "n_ignored": 20},
    {"M": 257, "V": 49408, "K": 136, "ignore": 0, "n_ignored": 40, "gpu": True},
    {"M": 1000, "V": 1001, "K": 768, "n_ignored": 100, "gpu": True},
])

# The ten (a_mn, b_mn, epilogue, act) instantiations gemm_launch dispatches, split-K on the two wgrad layouts.
GEMM_KINDS = [
    {"epi": "bf16"}, {"epi": "act", "act": 0}, {"epi": "act", "act": 1}, {"epi": "f32"},
    {"epi": "bf16", "b_mn": 1}, {"epi": "dact", "b_mn": 1, "act": 0}, {"epi": "dact", "b_mn": 1, "act": 1},
    {"epi": "f32", "b_mn": 1}, {"epi": "f32", "a_mn": 1, "b_mn": 1, "splits": 3}, {"epi": "f32", "a_mn": 1, "splits": 2},
]


def _gemm_kind_key(c):
    return c.get("a_mn", 0), c.get("b_mn", 0), _EPI[c["epi"]], c.get("act", 0) if c["epi"] in ("act", "dact") else 0


def _gc(M, N, K, kind, **kw):
    return {"M": M, "N": N, "K": K, **GEMM_KINDS[kind], **kw}


# Edges, each in both variants: M below 64 (the second consumer warpgroup has no rows) and on both sides of 64, 128 and
# 256, M <= 128 in a cluster (the peer CTA has no rows), N = 8 and one 8-column chunk past 64 / 256, fp32 N = 4 mod 8,
# K = 8, 64, 65 and tails shorter than one k-block, alpha 1 / 0.125 / -0.5 with and without bias, NaN-padded operand
# pitches, fp32 outputs off 16 bytes (direct stores, also under split-K).
_GEMM_EDGES = [
    _gc(40, 264, 72, 0, alpha=0.125, pad=8),
    _gc(65, 72, 65, 1, alpha=-0.5),
    _gc(127, 8, 8, 2, pad=16),
    _gc(129, 260, 200, 3, alpha=-0.5, col0=1, pad=4),
    _gc(100, 520, 64, 4, bias=False, pad=8),
    _gc(257, 136, 136, 5, alpha=0.125, pad=8),
    _gc(64, 264, 72, 6, alpha=-0.5),
    _gc(255, 68, 8, 7, bias=False, pad=4),
    _gc(136, 12, 392, 8, alpha=0.125, pad=8),
    _gc(264, 200, 136, 9, col0=1),
    _gc(63, 328, 65, 0, bias=False, colsum=True, alpha=-0.5),
    _gc(128, 72, 64, 1, bias=False, pad=8),
    _gc(256, 264, 130, 5, alpha=-0.5, pad=8),
    _gc(48, 260, 200, 8, alpha=-0.5, splits=4),
    _gc(300, 516, 200, 3, bias=False, col0=1),       # an fp32 column slice: base 4 bytes past a 16-byte boundary
]
# Persistent loops: every CTA (cluster) of a 132-SM H100 runs >= 3 tiles, and N = 1032 (five 256-column tiles, the
# last 8 columns wide) puts a partial-N tile after full ones in the same CTA (test_gemm_cases_sit_where_they_say).
_GEMM_PERSIST = [_gc(3400, 1032, 392, i, splits=3, alpha=0.125, persist=True, gpu=True) if GEMM_KINDS[i].get("a_mn")
                 else _gc(10200, 1032, 72, i, alpha=0.125, persist=True, gpu=True) for i in range(10)]
# GPU-sized shapes at the epilogue settings the fused layers use (bf16: alpha 0.5 with bias and column sums, and alpha 1
# without either; act and dact at alpha 0.125; fp32 with bias): M and N across the 128 / 256 tile boundaries with K
# tails for every operand layout, several tiles per CTA, and (_GEMM_WIDE) every instantiation at M and N one 8-row /
# 8-column step either side of a 256 multiple (an MN-major A keeps M a multiple of 8).
_LEGACY_EPI = {"bf16": {"alpha": 0.5}, "act": {"alpha": 0.125}, "dact": {"alpha": 0.125}, "f32": {}}


def _legacy(M, N, K, a_mn, b_mn, epi, act, splits):
    kind = {"epi": ["bf16", "act", "dact", "f32"][epi], "a_mn": a_mn, "b_mn": b_mn}
    if epi in (1, 2):
        kind["act"] = act
    if epi == 3:
        kind["splits"] = splits
    return {"M": M, "N": N, "K": K, **kind, **_LEGACY_EPI[kind["epi"]], "gpu": True}


_GEMM_PARITY = [
    # M, N, K, a_mn, b_mn, epi, act, splits   (epi: 0 bf16, 1 bf16 + act (two outputs), 2 bf16 x act'(aux), 3 fp32)
    (128, 256, 64, 0, 0, 3, 0, 1), (1000, 768, 200, 0, 0, 3, 0, 1), (1000, 768, 328, 0, 0, 0, 0, 1),
    (512, 1024, 256, 0, 0, 1, 0, 1), (1000, 712, 264, 0, 0, 1, 1, 1),
    (1000, 768, 264, 0, 1, 0, 0, 1), (640, 512, 512, 0, 1, 2, 0, 1), (1000, 776, 192, 0, 1, 2, 1, 1),
    (768, 768, 4096, 1, 1, 3, 0, 4), (1000, 520, 1000, 1, 1, 3, 0, 3), (520, 768, 1000, 1, 0, 3, 0, 2),
    (300, 4, 512, 0, 0, 3, 0, 1), (8, 512, 768, 0, 1, 3, 0, 1),
    (5000, 2304, 768, 0, 0, 0, 0, 1), (5000, 3072, 768, 0, 0, 1, 0, 1), (5000, 3072, 768, 0, 1, 2, 0, 1),
    (2304, 768, 5000, 1, 1, 3, 0, 5),
    (129, 136, 72, 0, 0, 0, 0, 1), (257, 200, 136, 0, 0, 1, 1, 1), (300, 264, 648, 0, 1, 2, 1, 1),
    (384, 392, 320, 1, 0, 3, 0, 2), (640, 136, 2048, 1, 1, 3, 0, 7), (96, 1160, 64, 0, 1, 0, 0, 1),
    (2000, 4104, 512, 0, 0, 1, 0, 1), (1500, 1032, 256, 0, 1, 2, 0, 1), (16, 8, 16, 0, 0, 3, 0, 1),
]
_GEMM_WIDE = [(M if not k[0] else {255: 248, 257: 264, 4097: 4104}.get(M, M), N, K) + k
                     for M, N, K in [(255, 520, 136), (257, 264, 200), (4097, 776, 72), (1000, 1032, 584)]
                     for k in [(0, 0, 0, 0, 1), (0, 0, 1, 0, 1), (0, 0, 1, 1, 1), (0, 0, 3, 0, 1), (0, 1, 0, 0, 1),
                               (0, 1, 2, 0, 1), (0, 1, 2, 1, 1), (0, 1, 3, 0, 1), (1, 1, 3, 0, 3), (1, 0, 3, 0, 2)]]
# the ViT-B/16 image tower's GEMMs at the benchmark's N and K, M cut from 100 864 tokens to 2048 rows (the FC1 wgrad:
# its contraction over the tokens cut to 8192)
_GEMM_TOWER = [
    (2048, 2304, 768, 0, 0, 0, 0, 1),    # QKV projection
    (2048, 3072, 768, 0, 0, 1, 0, 1),    # FC1 + QuickGELU
    (2048, 768, 3072, 0, 0, 0, 0, 1),    # FC2
    (2048, 768, 3072, 0, 1, 0, 0, 1),    # FC1 dgrad
    (2048, 3072, 768, 0, 1, 2, 0, 1),    # FC2 dgrad x QuickGELU'
    (768, 3072, 8192, 1, 1, 3, 0, 5),    # FC1 wgrad, split-K
]
_GEMM = (
    [{"M": 128, "N": 256, "K": 192, "epi": "bf16"}, {"M": 64, "N": 128, "K": 128, "epi": "f32"}]
    + _both_modes(_GEMM_EDGES + _GEMM_PERSIST + [_legacy(*c) for c in _GEMM_PARITY + _GEMM_WIDE + _GEMM_TOWER]
                  + [dict(_legacy(*c), alpha=1.0, bias=False, colsum=False) for c in _GEMM_PARITY if c[5] == 0])
    # the automatic choice: 1-CTA tiles below M = 512 or with fewer 256 x 256 tiles than SM pairs, clusters above
    + [_gc(511, 4104, 72, 1, gpu=True), _gc(1024, 4104, 72, 1, gpu=True), _gc(512, 520, 1000, 8, splits=40, gpu=True),
       _gc(1024, 264, 136, 6, alpha=-0.5, pad=8)]
)

# ---- cases -----------------------------------------------------------------------------------------------------------------
_WIDTHS = [128 * nv for nv in range(1, 9)]

CASES = {
    "cast_bf16": [{"n": 1}, {"n": 3}, {"n": 21}, {"n": 1001, "seed": 1}, {"n": 3_000_003, "gpu": True}],
    "cast_f32": [{"n": 1}, {"n": 7}, {"n": 65535}],
    "im2col": [{"B": 1, "H": 32, "W": 48, "ps": 16, "ld": 768}, {"B": 2, "H": 28, "W": 42, "ps": 14, "ld": 592},
               {"B": 2, "H": 224, "W": 224, "ps": 14, "ld": 592, "gpu": True},
               {"B": 64, "H": 224, "W": 224, "ps": 14, "ld": 592, "gpu": True},
               {"B": 64, "H": 224, "W": 224, "ps": 16, "ld": 768, "gpu": True}],
    "add_layernorm_fwd": [{"M": 37, "d": d, "seed": d} for d in _WIDTHS] + [
        {"M": 9, "d": 512, "rpg": 77, "gather": "idx"},           # ln_final at the EOT rows (CLIP text)
        {"M": 5, "d": 768, "rpg": 50, "gather": "zero"},          # ln_post at the CLS rows (CLIP vision)
        {"M": 40, "d": 256, "y": False}, {"M": 40, "d": 384, "x": False},
        {"M": 17000, "d": 128, "gpu": True}, {"M": 17000, "d": 1024, "gpu": True},
        {"M": 300, "d": 768, "rpg": 77, "gather": "idx", "gpu": True}],
    "layernorm_bwd": [{"M": 37, "d": d, "seed": d} for d in _WIDTHS] + [
        {"M": 23, "d": 768, "dy": "bf16", "alias": True},          # the encoder layers' (..., G, G, Gb, ...) call
        {"M": 9, "d": 512, "rpg": 77, "gather": "idx"},
        {"M": 6, "d": 768, "rpg": 50, "gather": "zero", "gin": False},
        {"M": 31, "d": 256, "g_bf16": False, "gsum": False},
        {"M": 4000, "d": 128, "dy": "bf16", "alias": True, "gpu": True},     # above num_sms * 24 rows
        {"M": 1000, "d": 1024, "dy": "bf16", "alias": True, "gpu": True},    # above num_sms * 6 rows
        {"M": 3, "d": 1024, "gpu": True},
        {"M": 640, "d": 512, "rpg": 77, "gather": "idx", "gpu": True}],
    "vit_embed_ln_fwd": [{"B": 3, "S": 5, "d": d, "seed": d} for d in _WIDTHS] + [
        {"B": 64, "S": 197, "d": 768, "gpu": True}, {"B": 70, "S": 257, "d": 1024, "gpu": True}],
    "vit_embed_ln_bwd": [{"B": 3, "S": 5, "d": d, "seed": d} for d in _WIDTHS] + [
        {"B": 64, "S": 197, "d": 768, "gpu": True}, {"B": 16, "S": 257, "d": 1024, "gpu": True}],
    "batch_sum": [{"Bn": 7, "n": 512, "ld": 520}, {"Bn": ("chunks", 0), "n": 512, "ld": 512},
                  {"Bn": ("chunks", 1), "n": 512, "ld": 512}, {"Bn": 2000, "n": 512, "ld": 516},
                  {"Bn": 5, "n": 12, "ld": 3 * 12}, {"Bn": 33, "n": 64, "ld": 77 * 64},
                  {"Bn": 64, "n": 197 * 768, "ld": 197 * 768, "gpu": True}],
    "colsum_bf16": [{"M": 37, "N": 264, "ld": 264}, {"M": 1001, "N": 776, "ld": 784}, {"M": 1, "N": 8, "ld": 8},
                    {"M": 31, "N": 2056, "ld": 2064}, {"M": 4096, "N": 3072, "ld": 3072, "gpu": True},
                    {"M": 12608, "N": 768, "ld": 768, "gpu": True}],
    "sum_scale": [{"n": 1, "scale": 0.5, "accumulate": False}, {"n": 300, "scale": -1.5, "accumulate": True},
                  {"n": 5000, "scale": 1 / 3, "accumulate": False}, {"n": 2, "scale": 2.0, "accumulate": True}],
    "matmul_f32": [{"M": 3, "N": 5, "K": 7, "ta": False, "tb": False, "acc": False, "alpha": 1.0},
                   {"M": 33, "N": 17, "K": 65, "ta": True, "tb": True, "acc": True, "alpha": -0.5},
                   {"M": 40, "N": 9, "K": 3, "ta": False, "tb": True, "acc": False, "alpha": 2.0}],
    "text_embed_fwd": [{"B": 3, "S": 7, "d": 64, "V": 100}, {"B": 33, "S": 77, "d": 512, "V": 49408, "gpu": True}],
    "text_embed_bwd": [{"B": 4, "S": 16, "d": 64, "V": 50}, {"B": 3, "S": 9, "d": 12, "V": 1000},
                       {"B": 64, "S": 77, "d": 512, "V": 49408, "keep": 0.3, "gpu": True},
                       {"B": 256, "S": 77, "d": 768, "V": 1024, "gpu": True}],
    "argmax_tokens": [{"B": 3, "S": 77}, {"B": 13, "S": 5}, {"B": 70, "S": 100, "gpu": True}],
    "coca_text_embed_fwd": [{"B": 2, "S": 6, "d": 64, "V": 40, "cls": True},
                            {"B": 3, "S": 5, "d": 32, "V": 40, "cls": False}],
    "bert_embed_ln_fwd": [{"B": 2, "S": 9, "d": 128, "V": 30}, {"B": 3, "S": 5, "d": 768, "V": 30, "types": False},
                          {"B": 16, "S": 512, "d": 768, "V": 30522, "gpu": True}],
    "bert_embed_ln_bwd": [{"B": 2, "S": 9, "d": 128, "V": 30}, {"B": 3, "S": 5, "d": 768, "V": 30, "types": False},
                          {"B": 16, "S": 128, "d": 768, "V": 1000, "gpu": True}],
    "l2norm_fwd": [{"B": 5, "E": 512, "zero_row": 1}, {"B": 9, "E": 77}, {"B": 3, "E": 1},
                   {"B": 1000, "E": 768, "zero_row": 999, "gpu": True}],
    "l2norm_bwd": [{"B": 5, "E": 512}, {"B": 9, "E": 77}, {"B": 1000, "E": 768, "gpu": True}],
    "act_fwd": [{"n": 8, "kind": 0}, {"n": 8, "kind": 1}, {"n": 1001, "kind": 0}, {"n": 1001, "kind": 1},
                {"n": 1_000_001, "kind": 1, "gpu": True}],
    "tanh_": [{"n": 9}, {"n": 1001}],
    "tanh_bwd": [{"n": 9}, {"n": 1001}],
    "act_bwd": [{"n": 9, "kind": 0}, {"n": 9, "kind": 1}, {"n": 4001, "kind": 0}, {"n": 4001, "kind": 1},
                {"n": 1_000_001, "kind": 0, "gpu": True}, {"n": 1_000_001, "kind": 1, "gpu": True}],
    "gather_rows_cast": [{"B": 3, "rpg": 5, "row": 0, "d": 64}, {"B": 4, "rpg": 7, "row": 6, "d": 12}],
    "gather_rows_idx_cast": [{"R": 50, "ld": 72, "d": 64, "n": 13}, {"R": 9, "ld": 12, "d": 12, "n": 1},
                             {"R": 5000, "ld": 772, "d": 768, "n": 3000, "gpu": True}],
    "scatter_rows_add": [{"B": 3, "rpg": 5, "row": 0, "d": 64}, {"B": 4, "rpg": 7, "row": 6, "d": 12}],
    "scatter_rows_idx_add": [{"R": 50, "ld": 72, "d": 64, "n": 30}, {"R": 9, "ld": 12, "d": 12, "n": 1},
                             {"R": 2000, "ld": 772, "d": 768, "n": 3000, "gpu": True}],
    "concat_tokens": [{"B": 2, "Sa": 3, "Sb": 4, "d": 16, "cls": True}, {"B": 3, "Sa": 5, "Sb": 0, "d": 8, "cls": True},
                      {"B": 2, "Sa": 2, "Sb": 3, "d": 4, "cls": False}],
    "split_tokens_cast": [{"B": 2, "Sa": 3, "Sb": 4, "d": 16, "cls": True}, {"B": 3, "Sa": 5, "Sb": 0, "d": 8, "cls": True},
                          {"B": 2, "Sa": 2, "Sb": 3, "d": 4, "cls": False}],
    "vit_assemble_fwd": [{"B": 2, "S": 5, "d": 16, "cls": True, "mask": True},
                         {"B": 2, "S": 4, "d": 8, "cls": False, "mask": False},
                         {"B": 3, "S": 10, "d": 32, "cls": True, "mask": False}],
    "vit_assemble_bwd": [{"B": 2, "S": 5, "d": 16, "cls": True, "mask": True},
                         {"B": 2, "S": 4, "d": 8, "cls": False, "mask": False},
                         {"B": 64, "S": 197, "d": 768, "cls": True, "mask": True, "gpu": True}],
    "zero_": [{"n": 5}, {"n": 4096}],
    "kv_cache_append": [
        {"B": 2, "H": 3, "Sp": 5, "Sn": 2, "hd": 64, "past": F32, "out": F32, "out_bf16": True},
        {"B": 2, "H": 2, "Sp": 4, "Sn": 1, "hd": 96, "past": BF, "out": BF, "out_bf16": False},
        {"B": 1, "H": 2, "Sp": 0, "Sn": 3, "hd": 128, "past": F32, "out": F32, "out_bf16": True},
        {"B": 3, "H": 1, "Sp": 7, "Sn": 5, "hd": 64, "past": F32, "out": None, "out_bf16": True},
        {"B": 4, "H": 12, "Sp": 300, "Sn": 1, "hd": 64, "past": BF, "out": BF, "out_bf16": False, "gpu": True}],
    "ce_labels": [{"M": 6, "V": 49408, "stride": 2, "n_ignored": 2}, {"M": 5, "V": 97, "stride": 1},
                  {"M": 4, "V": 49408, "stride": 3, "n_ignored": 4},              # every row ignored
                  {"M": 300, "V": 49408, "stride": 2, "n_ignored": 50, "gpu": True}],
    "ce_labels_bwd": [{"M": 6, "V": 49408, "stride": 2, "n_ignored": 2, "gscale": True}, {"M": 5, "V": 97, "stride": 1},
                      {"M": 4, "V": 49408, "stride": 3, "n_ignored": 4},
                      {"M": 300, "V": 49408, "stride": 2, "n_ignored": 50, "gpu": True}],
    "gemm": _GEMM,
    "attention_fwd": _PACKED,
    "attention_fwd_kmask": _KMASKED,
    "attention_bwd": _PACKED,
    "attention_bwd_kmask": _KMASKED,
    "attention_probs": _PROBS,
    "attention_fwd_generic": _GENERIC,
    "attention_bwd_generic": _GENERIC,
    "attention_fwd_decode": _DECODE,
    "contrastive_ce_stats": _CONTRASTIVE_STATS,
    "contrastive_ce_grad": _CONTRASTIVE_GRAD,
    "gemm_ce_stats": _GEMM_CE_STATS,
    "ce_stats_reduce": _CE_STATS_REDUCE,
    "gemm_ce_grad": _GEMM_CE_GRAD,
    "linear_cross_entropy": _LINEAR_CE,
}

# Kernels whose results DESIGN.md §4 documents as run-to-run bit-exact (no floating-point atomics).
DETERMINISTIC = ["layernorm_bwd", "vit_embed_ln_bwd", "batch_sum", "colsum_bf16", "text_embed_bwd", "ce_labels",
                 "sum_scale", "contrastive_ce_stats", "contrastive_ce_grad", "gemm_ce_stats", "ce_stats_reduce",
                 "gemm_ce_grad", "linear_cross_entropy", "gemm"]
# The ops on the GEMM kernel, whose two variants (one CTA per 128 x 256 tile, 2-CTA clusters) run the same wgmma
# sequence per 128-row block and differ only in the tile origin and the B multicast: bit-identical results.
GEMM_FAMILY = ["gemm", "gemm_ce_stats", "gemm_ce_grad", "linear_cross_entropy"]

CHECKS = {op: globals()["check_" + op] for op in CASES}


def case_id(case):
    return ",".join(f"{k}={getattr(v, '__name__', None) or (str(v).replace('torch.', ''))}"
                    for k, v in case.items() if k != "gpu")


def emulation():
    """The CPU emulation of every kernel (tests/emu_ops.py + tests/emu_decode_ops.py) as one `impl`."""
    import types

    import emu_decode_ops
    import emu_ops

    ns = {n: getattr(emu_ops, n) for n in emu_ops.NAMES}
    ns.update(attention_fwd_decode=emu_decode_ops.attention_fwd_decode, kv_cache_append=emu_decode_ops.kv_cache_append)
    return types.SimpleNamespace(**ns)
