"""Per-element error bounds (or bit-exact checks) for the row-wise, sampler and pre/post-processing kernels, in both libraries.

The checker and the error model are those of tests/test_kernel_bounds_gpu.py: every output element must satisfy

    |got - y| <= u |y| + (1 + u) E + floor

against a float64 reference built from plain torch ops, where E is derived from the kernel's arithmetic.  Every intermediate
storage-type rounding (fp16 / bf16) counts as one u of that value, carried to the output by the slope of what follows it.
Kernels that perform exactly the reference's roundings (the copies, the external row gate, cfg_x0) are held to torch.equal.

CPU tests: test_every_entry_point_has_a_bound_test parses include/star_sm100.h and requires every compute entry point to map,
in COVERAGE below, to existing bound or exact tests, and every op the CogVideoX path calls to have a bf16 one;
test_checkers_catch_injected_faults feeds each new checker a simulated output and one injected fault per family.
"""
import glob
import importlib
import math
import os
import re

import pytest
import torch
import torch.nn.functional as F

from tests.test_kernel_bounds_gpu import (BoundCheck, check_bound, _finish, U_OUT, FLOOR, U32, ERR_EX2, _silu_step,
                                          NORM_FP32_ROUND, _offset_input, _group_stats, _norm_bound, _rnd, _g,
                                          run_gemm_case, plan, tap_epilogue, _contract, layernorm_instance)
from tests.util import assert_close

HALF, BF16, F64, F32 = torch.float16, torch.bfloat16, torch.float64, torch.float32
DTYPES = [pytest.param(HALF, id="fp16"), pytest.param(BF16, id="bf16")]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# ---- error model additions: one place, one reason each -------------------------------------------------------------------
ERR_FDIV = 2.0 ** -22          # fast-math fp32 division x / y (__fdividef) and 1 / y: 2 ulp (CUDA C++ Programming Guide, intrinsics)
ERR_LG2 = 2.0 ** -22           # __log2f (lg2.approx) outside [0.5, 2]: 2 ulp (CUDA C++ Programming Guide, intrinsics)
ERR_SINCOS = 2.0 ** -20.5      # sin.approx.f32 / cos.approx.f32: max absolute error 2^-20.5 in -100 pi .. 100 pi (PTX ISA).
#                                Beyond that range (test_sinusoidal_bound reaches 999 rad) no error is documented: the bound
#                                assumes the same error on the reduced argument, with RANGE_RED below as the whole growth
RANGE_RED = 3                  # __sinf / __cosf reduce x as x * (1 / 2 pi) in fp32: product rounded toward zero (2 U32 relative)
#                                and the rounded constant (U32): a phase error of 3 U32 |x| radians, growing with the argument
#                                (a model of the reduction, not a documented figure)
ERR_RSQRT = 2.0 ** -22.9       # rsqrt.approx.f32: max relative error 2^-22.9 (PTX ISA)
QK_SUM_ROUND = 11              # per-head sums of qk_ln_rope: 8 sequential fp32 adds per lane, then 3 shuffle levels
VAE_HEAD_ROUND = 19            # vae_head: 9 fp32 products and 9 adds onto the bias, each rounded once
INTERP_ROUND = 8               # bilinear: hx a, lx b, their sum, hy (..), the same for the second row, the final sum (6 roundings
#                                on values <= the largest corner) and 1 - lx, 1 - ly (one rounding of a weight each)
WARP_TREE = 5                  # a 32-lane shuffle reduction adds 5 levels of fp32 rounding to a sum
BLOCK_TREE = 8                 # softmax_rows: the 8 warp partials are added in fp32 by every thread


def _st(t, dtype):
    """round an fp64 tensor to the storage type and back"""
    return t.to(dtype).to(F64)


def _sigmoid_gate(lin, dlin, dtype):
    """gate = fl(sigmoid_f(fl(lin))) known to within the returned error: the slope 1/4 carries dlin, sigmoid_f is
    1 / (1 + __expf(-x)) (ex2.approx with its argument scaled in fp32, fast division), then one storage rounding"""
    g = torch.sigmoid(lin)
    u, fl = U_OUT[dtype], FLOOR[dtype]
    dg = 0.25 * (dlin + u * lin.abs() + fl) + g * ((1 - g) * (ERR_EX2 + 3 * U32 * lin.abs()) + ERR_FDIV + U32)
    return g, dg + u * g + fl


def _temporal_gate(x64, w0, w1, n_lane, dtype):
    """fp64 temporal LIEM gate sigmoid(w0 max_c + w1 mean_c) per row and its error: the fp32 row sum (n_lane terms per lane and
    the warp tree), the fast division by C, the storage roundings of the mean and of the linear term"""
    u, fl = U_OUT[dtype], FLOOR[dtype]
    mean, mx = x64.mean(1, keepdim=True), x64.amax(1, keepdim=True)
    dmean = U32 * (n_lane + WARP_TREE) * x64.abs().mean(1, keepdim=True) + (ERR_FDIV + U32) * mean.abs()
    dmean = dmean + u * mean.abs() + fl
    lin = w0 * mx + w1 * mean
    dlin = abs(w1) * dmean + 2 * U32 * ((w0 * mx).abs() + (w1 * mean).abs())
    return _sigmoid_gate(lin, dlin, dtype)


# ---- coverage: every compute entry point of include/star_sm100.h -> its bound / exact tests ----------------------------------
B = "tests.test_kernel_bounds_gpu::"
S = "tests.test_spatial_tiles_gpu::"
R = "tests.test_rowops_bounds_gpu::"
N = "tests.test_banded_bounds_gpu::"
COVERAGE = {
    "star_linear": [(B + "test_tapgemm_bound", "fp16,bf16")],
    "star_linear_ex": [(B + "test_tapgemm_bound", "fp16,bf16")],
    "star_conv2d_3x3": [(B + "test_tapgemm_bound", "fp16,bf16"), (N + "test_conv2d_3x3_rows_bound", "fp16,bf16"),
                        (N + "test_conv2d_3x3_rows_past_2_32_elements", "fp16")],
    "star_conv2d_3x3_s2": [(R + "test_conv2d_s2_bound", "fp16")],
    "star_conv2d_3x3_s2p": [(B + "test_tapgemm_bound", "fp16"), (R + "test_vae_convs_bf16_bound", "bf16")],
    "star_conv_t3": [(B + "test_tapgemm_bound", "fp16"), (N + "test_conv_t3_band_bound", "fp16,bf16"),
                     (N + "test_conv_t3_band_past_2_31_elements", "fp16")],
    "star_conv2d_3x3_c4": [(R + "test_conv2d_c4_bound", "fp16")],
    "star_attention": [(B + "test_attention_bound", "fp16,bf16")],
    "star_attention_causal": [(B + "test_attention_causal_bound", "fp16")],
    "star_temporal_attention": [(B + "test_temporal_attention_bound", "fp16")],
    "star_conv3d_causal": [(B + "test_tapgemm_bound", "fp16"), (R + "test_vae_convs_bf16_bound", "bf16")],
    "star_groupnorm": [(B + "test_groupnorm_offset_bound", "fp16"), (R + "test_groupnorm_bf16_bound", "bf16"),
                       (N + "test_groupnorm_bands_bound", "fp16,bf16"), (N + "test_groupnorm_bands_refuses_C_above_2048", "fp16"),
                       (N + "test_groupnorm_past_2_32_elements", "fp16")],
    "star_groupnorm_mod": [(B + "test_groupnorm_mod_offset_bound", "fp16"), (R + "test_groupnorm_mod_bf16_bound", "bf16"),
                           (N + "test_groupnorm_mod_geometry_bound", "fp16,bf16")],
    "star_layernorm": [(B + "test_layernorm_offset_bound", "fp16"), (R + "test_layernorm_gate_bound", "fp16"),
                       (R + "test_layernorm_bf16_bound", "bf16")],
    "star_liem_spatial_gate": [(R + "test_liem_spatial_gate_bound", "fp16,bf16")],
    "star_row_gate": [(R + "test_row_gate_external_exact", "fp16,bf16"), (R + "test_row_gate_temporal_bound", "fp16,bf16")],
    "star_qk_ln_rope": [(R + "test_qk_ln_rope_bound", "fp16,bf16")],
    "star_concat_add": [(R + "test_concat_add_exact", "fp16")],
    "star_add": [(R + "test_add_exact", "fp16")],
    "star_upsample2x_crop": [(R + "test_upsample2x_exact", "fp16,bf16")],
    "star_time_avgpool2": [(R + "test_time_avgpool2_bound", "fp16,bf16")],
    "star_upsample2x": [(R + "test_upsample2x_exact", "fp16,bf16"), (N + "test_upsample2x_past_2_32_elements", "fp16")],
    "star_softmax_rows": [(R + "test_softmax_rows_bound", "fp16"), (R + "test_softmax_rows_refuses_102401_columns", "fp16")],
    "star_vae_head": [(R + "test_vae_head_bound", "fp16"), (N + "test_vae_head_and_tokens_to_nchw5_past_2_32_elements", "fp16")],
    "star_nchw5_to_tokens": [(R + "test_layout_conversions_exact", "fp16,bf16")],
    "star_tokens_to_nchw5": [(R + "test_layout_conversions_exact", "fp16,bf16"),
                             (N + "test_vae_head_and_tokens_to_nchw5_past_2_32_elements", "fp16")],
    "star_bilinear_pad": [(R + "test_bilinear_pad_bound", "fp32")],
    "star_adain_color_fix": [(R + "test_adain_color_fix_bound", "fp32,uint8"), (R + "test_adain_refuses_too_many_planes", "fp32"),
                             (N + "test_adain_color_fix_past_2_31_elements", "uint8")],
    "star_cfg_x0": [(R + "test_cfg_x0_exact", "fp16")],
    "star_cfg_x0_blend": [(S + "test_blend_unit_weights_bit_exact", "fp16")],
    "star_sinusoidal": [(R + "test_sinusoidal_bound", "fp16,bf16")],
    "star_silu": [(R + "test_silu_bound", "fp16,bf16")],
}


def _header_entry_points():
    src = open(os.path.join(ROOT, "include", "star_sm100.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(name for name, args in re.findall(r"\bint\s+(star_\w+)\s*\(([^;]*?)\)\s*;", src, flags=re.S)
                  if args.replace(" ", "").endswith("void*stream"))


def _cogvideox_ops():
    ops = set()
    for path in glob.glob(os.path.join(ROOT, "star_b200", "cogvideox", "*.py")):
        ops |= set(re.findall(r"\bops\.(\w+)\(", open(path).read()))
    return sorted(ops)


def test_every_entry_point_has_a_bound_test():
    entries = _header_entry_points()
    assert len(entries) >= 30, f"parsed only {entries}"
    missing = [e for e in entries if not COVERAGE.get(e)]
    assert not missing, f"entry points without a per-element bound or exact test: {missing}"
    stale = sorted(set(COVERAGE) - set(entries))
    assert not stale, f"coverage entries for entry points the header no longer declares: {stale}"
    for entry, tests in COVERAGE.items():
        for test_id, dtypes in tests:
            mod, name = test_id.split("::")
            assert callable(getattr(importlib.import_module(mod), name, None)), f"{entry}: {test_id} does not exist"
            assert dtypes and set(dtypes.split(",")) <= {"fp16", "bf16", "fp32", "uint8"}, f"{entry}: dtypes {dtypes!r}"
    ops = _cogvideox_ops()
    assert "layernorm" in ops and "qk_ln_rope" in ops, f"parsed only {ops}"
    no_bf16 = [op for op in ops if not any("bf16" in d.split(",") for _, d in COVERAGE.get("star_" + op, []))]
    assert not no_bf16, f"ops of the CogVideoX path (bf16 library) without a bf16 bound test: {no_bf16}"


# ---- references and bounds (device-agnostic: the self-test runs them on the CPU) -------------------------------------------
def softmax_ref(s, cols):
    """fp64 softmax over the first cols columns of fp16 logits and its bound.  Kernel: the row max (exact), e = __expf(x - max)
    (the fp32 difference and its scaling by log2 e each round: 3 U32 |x - max|, then ex2.approx), a per-thread fp32 sum of
    ceil(cols / 256) terms plus the warp and block trees, one fast reciprocal and the product."""
    x = s[:, :cols].to(F64)
    z = x - x.amax(1, keepdim=True)
    e = torch.exp(z)
    tot = e.sum(1, keepdim=True)
    p = e / tot
    term = ERR_EX2 + 3 * U32 * z.abs()
    sum_rel = (e * term).sum(1, keepdim=True) / tot + U32 * (math.ceil(cols / 256) + WARP_TREE + BLOCK_TREE)
    return p, _finish(p, (term + sum_rel + ERR_FDIV + U32) * p, HALF)


def cfg_scale(y, u, g, r):
    """the reference's fp16 rescale factor per sample, from exact statistics: std(y), std(out) (unbiased), each rounded to
    fp16, out std + 1e-12, the ratio, r * ratio and + (1 - r), each rounded to fp16 after fp32 arithmetic"""
    h = lambda t: t.to(F32).to(HALF).to(F64)                                   # noqa: E731
    o = cfg_combine(y, u, g)
    n = y[0].numel()
    scales = []
    for b in range(y.shape[0]):
        sdy = h(torch.tensor(y[b].to(F64).std().item()))
        sdo = h(torch.tensor(o[b].std().item()))
        den = h(sdo + float(torch.tensor(1e-12, dtype=F32)))
        ratio = h(sdy / den)
        rr = float(torch.tensor(r, dtype=F32))
        a = h(rr * ratio)
        scales.append(h(a + float(torch.tensor(1.0, dtype=F32) - torch.tensor(rr, dtype=F32))))
    assert n > 1
    return scales


def cfg_combine(y, u, g):
    """out = u + g (y - u) with the reference's fp16 roundings (fp32 arithmetic, then fp16), as fp64"""
    h = lambda t: t.to(F32).to(HALF).to(F64)                                   # noqa: E731
    y64, u64 = y.to(F64), u.to(F64)
    d = h(y64 - u64)
    gd = h(d * float(torch.tensor(g, dtype=F32)))
    return h(u64 + gd)


def _fp16_neighbours(v):
    bits = torch.tensor([v], dtype=HALF).view(torch.int16)
    return [(bits + k).view(HALF).item() for k in (-1, 0, 1)]


def check_cfg_exact(y, u, xt, al, sg, g, r, guided, x0):
    """guided must equal the fp16 op sequence for one rescale factor per sample, the reference's factor or one of its fp16
    neighbours; x0 must equal fl(fl(alpha xt) - fl(sigma guided)) bit for bit"""
    o = cfg_combine(y, u, g)
    scales = cfg_scale(y, u, g, r) if r is not None else [None] * y.shape[0]
    for b in range(y.shape[0]):
        if scales[b] is None:
            want = [o[b].to(HALF)]
        else:
            want = [(o[b] * s).to(F32).to(HALF) for s in _fp16_neighbours(scales[b])]
        hits = [torch.equal(guided[b], w) for w in want]
        if not any(hits):
            nbad = min(int((guided[b] != w).sum()) for w in want)
            raise AssertionError(f"cfg_x0 sample {b}: guided output matches no rescale factor in "
                                 f"{[] if scales[b] is None else _fp16_neighbours(scales[b])} ({nbad} elements differ at best)")
    a32, s32 = al.reshape(-1).to(F32), sg.reshape(-1).to(F32)
    shape = (-1,) + (1,) * (xt.dim() - 1)
    want_x0 = a32.view(shape) * xt.to(F32) - s32.view(shape) * guided.to(F32)
    if not torch.equal(x0, want_x0):
        bad = (x0 != want_x0).nonzero()[:5].tolist()
        raise AssertionError(f"cfg_x0: x0 differs from fl(fl(alpha xt) - fl(sigma out)) at {bad}")


def gated_layernorm_ref(x, gamma, beta, eps, mode, gate, w0, w1, dtype):
    """fp64 LayerNorm(x * g) gamma + beta and its bound.

    Mode 1 (external gate): x and g are storage values, so x g is exact in fp32 and the kernel's product is fl(x g), which
    the reference restates exactly.  Mode 2 (temporal gate, see _temporal_gate): a relative gate error delta scales the whole
    row, which LayerNorm removes except through eps, |d yn| <= |yn| (1 - f) delta with f = var / (var + eps); each product
    is rounded to the storage type (u |v| + floor per element dv), moving yn by at most rstd (|dv_i| + mean |dv| +
    |yn_i| rms(dv)).  Statistics in fp32, one warp (or sub-warp) per row: n_sum = the values per lane plus the shuffle tree,
    so the sum is off by n_sum U32 sum |v|; the mean multiplies by 1 / C from a fast division; the variance accumulates the
    rounded differences by fma (n_sum + 2 roundings of var, the mean's error entering squared), is scaled the same way, eps
    is added, and rsqrt.approx follows.  The apply rounds NORM_FP32_ROUND times."""
    u, fl = U_OUT[dtype], FLOOR[dtype]
    x64 = x.to(F64)
    C = x.shape[1]
    n_sum = (40 if C in (320, 640) else 8 * math.ceil(C / 8 / 32)) + WARP_TREE
    if mode == 1:
        g = gate.to(F64)[:, None]
        v = _st(x64 * g, dtype)
        dg = torch.zeros_like(g)
    else:
        g, dg = _temporal_gate(x64, w0, w1, n_sum - WARP_TREE, dtype)
        v = x64 * g
    m = v.mean(1, keepdim=True)
    var = ((v - m) ** 2).mean(1, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + eps)
    yn = (v - m) * rstd
    f = var / (var + eps)
    if mode == 1:
        d_prod = torch.zeros_like(yn)
    else:
        dv = u * v.abs() + fl
        d_prod = rstd * (dv + dv.mean(1, keepdim=True) + yn.abs() * (dv ** 2).mean(1, keepdim=True).sqrt())
    d_gate = yn.abs() * (1 - f) * torch.where(g > 0, dg / g, torch.where(dg > 0, float("inf"), 0.0))
    dm = n_sum * U32 * v.abs().mean(1, keepdim=True) + (ERR_FDIV + U32) * m.abs()
    dvar = ((n_sum + 3) * U32 + ERR_FDIV) * var + dm ** 2        # fma sums, d^2 of a rounded d (2), the scaling (1 + 1 / C)
    rel_rstd = 0.5 * (dvar + U32 * (var + eps)) / (var + eps) + ERR_RSQRT
    d_stat = yn.abs() * rel_rstd + dm * rstd + U32 * yn.abs()
    g64, b64 = gamma.to(F64), beta.to(F64)
    y = yn * g64 + b64
    err = g64.abs() * (d_prod + d_gate + d_stat) + NORM_FP32_ROUND * U32 * (v.abs() * rstd * g64.abs() + b64.abs())
    return y, _finish(y, err, dtype)


def liem_ref(x, w98, BT, H, W, dtype, drop_tap=False):
    """fp64 spatial LIEM gate sigmoid(conv7x7([max_c, mean_c])) and its bound.  Kernel: the fp32 channel sum (per lane and
    the warp tree) over C with a fast division, max / mean rounded to the storage type, 98 fp32 fmas over the clipped window
    (zero padding = skipped taps), the conv output rounded to the storage type, sigmoid_f, the gate rounded.
    drop_tap: the self-test's fault, the top-left tap dropped from every window clipped at the top-left corner."""
    u, fl = U_OUT[dtype], FLOOR[dtype]
    x64 = x.to(F64)
    C = x.shape[1]
    mx, mean = x64.amax(1), x64.mean(1)
    n_lane = 8 * math.ceil(C / 8 / 32)
    dmean = U32 * (n_lane + WARP_TREE) * x64.abs().mean(1) + (ERR_FDIV + U32) * mean.abs() + u * mean.abs() + fl
    mm = torch.stack([mx, mean], 1).view(BT, H, W, 2).permute(0, 3, 1, 2)
    dmm = torch.stack([torch.zeros_like(dmean), dmean], 1).view(BT, H, W, 2).permute(0, 3, 1, 2)
    w = w98.to(F64).view(1, 2, 7, 7)
    z = F.conv2d(mm, w, padding=3)
    if drop_tap:
        mm0 = mm.clone()
        mm0[:, :, 0, 0] = 0
        z = torch.where((torch.arange(H, device=x.device)[:, None] < 3) & (torch.arange(W, device=x.device)[None, :] < 3),
                        F.conv2d(mm0, w, padding=3), z)
    dz = F.conv2d(dmm, w.abs(), padding=3) + 98 * U32 * F.conv2d(mm.abs(), w.abs(), padding=3)
    gate, dg = _sigmoid_gate(z, dz, dtype)
    gate, dg = gate.reshape(-1, 1), dg.reshape(-1, 1)
    return gate, _finish(gate, dg, dtype)


def adain_ref(video, source):
    """fp64 adain_color_fix of video (1, C, F, H, W) to source (F, C, h, w), as (F * H * W, C) on the 0..255 scale, and its
    bound.  Kernel: v = clamp(fma(x, .5, .5)) (one fp32 rounding), per-plane sums of v and v^2 accumulated in fp32 per thread
    (ceil(n / (grid * 256)) terms, then the warp tree; the block and grid sums are fp64), statistics in fp64 from those sums,
    scale and shift rounded to fp32, one fma, the clamps (1-Lipschitz) and * 255.  The sum errors are carried through the
    variance, sqrt ratio and shift as worst-case intervals."""
    _, C, Fr, H, W = video.shape
    HW, shw = H * W, source.shape[2] * source.shape[3]
    v = ((video[0].to(F64) + 1) / 2).clamp(0, 1).reshape(C, Fr, HW)
    s = ((source.to(F64) + 1) / 2).reshape(Fr, C, shw).transpose(0, 1)

    def stats(t, n):
        grid = min(math.ceil(n / 256), 256)
        gam = U32 * (math.ceil(n / (grid * 256)) + WARP_TREE + 1)
        S1, Q = t.sum(-1, keepdim=True), (t * t).sum(-1, keepdim=True)
        dS, dQ = gam * t.abs().sum(-1, keepdim=True), gam * Q
        mean = S1 / n
        var = ((t - mean) ** 2).sum(-1, keepdim=True) / (n - 1) + 1e-5
        dvar = (dQ + 2 * S1.abs() / n * dS + dS ** 2 / n) / (n - 1)
        return mean, dS / n, var, dvar

    tm, dtm, tv, dtv = stats(v, HW)
    sm, dsm, sv, dsv = stats(s, shw)
    k = torch.sqrt(sv / tv)
    k_hi = torch.sqrt((sv + dsv) / (tv - dtv).clamp_min(1e-300))
    k_lo = torch.sqrt((sv - dsv).clamp_min(0) / (tv + dtv))
    dk = torch.maximum(k_hi - k, k - k_lo)
    dk = torch.where(tv - dtv > 0, dk, torch.full_like(dk, float("inf")))
    shift = sm - tm * k
    pre = shift + v * k
    dev = (v - tm).abs()
    e_pre = dsm + k * dtm + torch.where(dev > 0, dev * dk, torch.zeros_like(dev)) + dk * dtm \
        + U32 * (2 * v * k + shift.abs() + pre.abs())
    y = pre.clamp(0, 1) * 255
    err = 255 * e_pre
    to_out = lambda t: t.permute(1, 2, 0).reshape(Fr * HW, C)                  # noqa: E731  (c, f, hw) -> (f hw, c)
    y, err = to_out(y), to_out(err)
    return y, U32 * y + (1 + U32) * err + 2.0 ** -149


def check_adain_u8(got8, y, bound, what):
    """the uint8 output is the round-to-nearest of a value within bound of y: it must lie in [rn(y - b), rn(y + b)], which is
    round(y) itself wherever y is not within its bound of a .5 boundary"""
    lo = torch.ceil(y - bound - 0.5).clamp(0, 255)
    hi = torch.floor(y + bound + 0.5).clamp(0, 255)
    g = got8.to(F64)
    bad = (g < lo) | (g > hi)
    exact = (lo == hi).float().mean().item()
    print(f"[bounds] adain-u8          {what}: {exact * 100:.2f} % of elements must equal round(y)")
    if bad.any():
        idx = bad.nonzero()[:5].tolist()
        raise AssertionError(f"{what}: {int(bad.sum())} uint8 outputs outside [rn(y - b), rn(y + b)], first at "
                             f"{[(r, c, int(got8[r, c]), y[r, c].item()) for r, c in idx]}")


# ---- CPU self-test of the new checkers -----------------------------------------------------------------------------------
def test_checkers_catch_injected_faults():
    """Simulated kernel outputs (the fp64 reference rounded to the output type) pass each checker; one injected fault per
    family fails it.  The printed list shows which faults the rel-L2 / max-abs check of tests/util.py lets through.

    LayerNorm is invariant to a common scale of its row except through eps, so a gate one ulp off can only be seen on a row
    whose variance after the gate is comparable to eps; the gated-LayerNorm fault is injected on such a row."""
    gen = torch.Generator().manual_seed(0)
    missed = []

    def fault(name, check, got, ref):
        with pytest.raises(AssertionError):
            check(got)
        try:
            assert_close(got, ref, what=name)
            missed.append(name)
        except AssertionError:
            pass

    # cfg_x0: a rescale factor two fp16 ulps off on sample 1
    y = torch.randn(2, 4, 3, 10, 8, generator=gen).half()
    u = (y.float() + 0.3 * torch.randn(y.shape, generator=gen)).half()
    xt = torch.randn(y.shape, generator=gen)
    al, sg = torch.tensor([0.6, 0.7]), torch.tensor([0.8, 0.5])
    o = cfg_combine(y, u, 7.5)
    scales = cfg_scale(y, u, 7.5, 0.2)
    guided = torch.stack([(o[b] * scales[b]).to(F32).to(HALF) for b in range(2)])
    x0 = al.view(-1, 1, 1, 1, 1) * xt - sg.view(-1, 1, 1, 1, 1) * guided.float()
    check_cfg_exact(y, u, xt, al, sg, 7.5, 0.2, guided, x0)
    bad = guided.clone()
    off = (torch.tensor([scales[1]], dtype=HALF).view(torch.int16) + 2).view(HALF).item()
    bad[1] = (o[1] * off).to(F32).to(HALF)
    bad_x0 = al.view(-1, 1, 1, 1, 1) * xt - sg.view(-1, 1, 1, 1, 1) * bad.float()
    fault("cfg_x0 rescale factor 2 ulps off on one sample", lambda g: check_cfg_exact(y, u, xt, al, sg, 7.5, 0.2, g, bad_x0),
          bad, guided)

    # softmax: one row normalised over cols - 1
    cols = 300
    s = (3 * torch.randn(6, cols, generator=gen)).half()
    p, b = softmax_ref(s, cols)
    check_bound(p.half(), p, b, "clean softmax")
    e = torch.exp(s.double() - s.double().amax(1, keepdim=True))
    g = p.half()
    g[3] = (e[3] / e[3, :cols - 1].sum()).half()
    fault("softmax row normalised over cols - 1", lambda t: check_bound(t, p, b, "softmax fault"), g, p.half())

    # external row gate: one row using a gate one fp16 ulp off (exact check)
    x = torch.randn(40, 320, generator=gen).half()
    gate = torch.rand(40, generator=gen).half()
    want = (x.double() * gate.double()[:, None]).half()
    g1 = gate.clone()
    g1[17] = (g1[17:18].view(torch.int16) + 1).view(HALF)[0]
    got = (x.double() * g1.double()[:, None]).half()
    fault("row gate one fp16 ulp off on one row", lambda t: _assert_equal(t, want, "row gate"), got, want)

    # AdaIN: one plane's scale 0.5 % off
    video = (0.8 * torch.randn(1, 3, 2, 24, 32, generator=gen))
    src = torch.rand(2, 3, 6, 8, generator=gen) * 2 - 1
    ya, ba = adain_ref(video, src)
    check_bound(ya.float(), ya, ba, "clean adain")
    v = ((video[0].double() + 1) / 2).clamp(0, 1).reshape(3, 2, -1)
    sv = ((src.double() + 1) / 2).reshape(2, 3, -1)
    c, f = 1, 0
    k = torch.sqrt((sv[f, c].var() + 1e-5) / (v[c, f].var() + 1e-5)) * 1.005
    yf = ((v[c, f] - v[c, f].mean()) * k + sv[f, c].mean()).clamp(0, 1) * 255
    g = ya.float().clone()
    g.view(2, -1, 3)[f, :, c] = yf.float()
    fault("adain plane scale 0.5 % off", lambda t: check_bound(t, ya, ba, "adain fault"), g, ya.float())

    # spatial LIEM gate: one clipped tap dropped
    xl = torch.randn(2 * 6 * 5, 64, generator=gen).half()
    w98 = (0.2 * torch.randn(98, generator=gen)).half()
    gl, bl = liem_ref(xl, w98, 2, 6, 5, HALF)
    check_bound(gl.half(), gl, bl, "clean liem")
    gf, _ = liem_ref(xl, w98, 2, 6, 5, HALF, drop_tap=True)
    fault("liem gate with one clipped tap dropped", lambda t: check_bound(t, gl, bl, "liem fault"), gf.half(), gl.half())

    # gated LayerNorm: the simulated output passes (mode 2, rows not a multiple of 4)
    xg = (torch.randn(37, 320, generator=gen) + 16).half()
    gam, bet = (1 + 0.1 * torch.randn(320, generator=gen)).half(), (0.1 * torch.randn(320, generator=gen)).half()
    yl, bl = gated_layernorm_ref(xg, gam, bet, 1e-5, 2, None, 0.03125, -0.015625, HALF)
    check_bound(yl.half(), yl, bl, "clean gated layernorm")
    # ... and one row using a gate one fp16 ulp off (mode 1), on rows whose gated variance is about eps / 4
    xe = (torch.sqrt(torch.tensor(1e-5)) * torch.randn(37, 320, generator=gen)).half()
    ge = (0.5 + 0.1 * torch.rand(37, generator=gen)).half()
    yl, bl = gated_layernorm_ref(xe, gam, bet, 1e-5, 1, ge, 0, 0, HALF)
    check_bound(yl.half(), yl, bl, "clean gated layernorm, var ~ eps")
    ge1 = ge.clone()
    ge1[5] = (ge1[5:6].view(torch.int16) + 1).view(HALF)[0]
    g = yl.half()
    g[5] = gated_layernorm_ref(xe, gam, bet, 1e-5, 1, ge1, 0, 0, HALF)[0][5].half()
    fault("gated layernorm gate one fp16 ulp off on one row", lambda t: check_bound(t, yl, bl, "gated layernorm fault"),
          g, yl.half())

    print("[bounds] faults assert_close lets pass:", missed)
    assert missed, "every injected fault is also caught by assert_close"


def _assert_equal(got, want, what):
    if not torch.equal(got, want):
        bad = (got != want).nonzero()[:5].tolist()
        raise AssertionError(f"{what}: {int((got != want).sum())} elements differ from the exact result, first at {bad}")


# ---- GPU -----------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ops():
    from star_b200 import ops as O
    torch.cuda.reset_peak_memory_stats()
    yield O
    print(f"[bounds] rowops: peak device memory {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")


def _rnd_dt(shape, seed, dtype, scale=1.0):
    return _rnd(shape, seed, scale, F32).to(dtype)


# exact: copies and conversions
@pytest.mark.gpu
@pytest.mark.parametrize("Ca,Cb", [(8, 8), (320, 640), (264, 136)])
def test_concat_add_exact(ops, Ca, Cb):
    rows = 1001
    a, b, c = _rnd((rows, Ca), 1), _rnd((rows, Cb), 2), _rnd((rows, Cb), 3)
    _assert_equal(ops.concat_add(a, b, c), torch.cat([a, (b.to(F64) + c.to(F64)).half()], 1), f"concat_add {Ca}|{Cb} + c")
    _assert_equal(ops.concat_add(a, b), torch.cat([a, b], 1), f"concat_add {Ca}|{Cb}")


@pytest.mark.gpu
@pytest.mark.parametrize("n", [8, 1000, 8 * 100003])
def test_add_exact(ops, n):
    a, b = _rnd((n,), 1, 100.0), _rnd((n,), 2, 0.01)
    _assert_equal(ops.add(a, b), (a.to(F64) + b.to(F64)).half(), f"add n={n}")


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("BT,H,W,C", [(2, 9, 4, 8), (3, 5, 7, 264), (1, 17, 27, 1280)])
def test_upsample2x_exact(ops, dtype, BT, H, W, C):
    x = _rnd_dt((BT * H * W, C), 1, dtype)
    up = x.view(BT, H, W, C).repeat_interleave(2, 1).repeat_interleave(2, 2)
    _assert_equal(ops.upsample2x(x, BT, H, W), up.reshape(-1, C), "upsample2x")
    _assert_equal(ops.upsample2x_crop(x, BT, H, W), up[:, 1:-1].reshape(-1, C), "upsample2x_crop")


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("B,C,Fr,H,W", [(2, 8, 3, 10, 8), (1, 3, 1, 7, 9), (1, 264, 2, 5, 6)])
def test_layout_conversions_exact(ops, dtype, B, C, Fr, H, W):
    x5 = torch.randn(B, C, Fr, H, W, device="cuda") * 100
    tok = ops.nchw5_to_tokens(x5, dtype=dtype)
    _assert_equal(tok, x5.permute(0, 2, 3, 4, 1).reshape(-1, C).to(dtype), "nchw5_to_tokens")
    wide = torch.cat([tok, _rnd_dt((tok.shape[0], 8), 2, dtype)], 1)              # ldx = C + 8 > C
    _assert_equal(ops.tokens_to_nchw5(wide[:, :C], B, C, Fr, H, W), x5.to(dtype), "tokens_to_nchw5")


# cfg_x0: exact up to the choice of one fp16 rescale factor per sample
@pytest.mark.gpu
@pytest.mark.parametrize("B,shape,rescale", [(1, (4, 32, 122, 216), 0.2), (2, (4, 5, 18, 16), 0.2), (3, (4, 3, 10, 8), 0.7),
                                             (2, (4, 3, 10, 8), None)])
def test_cfg_x0_exact(ops, B, shape, rescale):
    g = torch.Generator(device="cuda").manual_seed(1)
    y = torch.randn(B, *shape, generator=g, device="cuda").half()
    u = (y.float() + 0.3 * torch.randn(y.shape, generator=g, device="cuda")).half()
    xt = torch.randn(y.shape, generator=g, device="cuda")
    al = torch.linspace(0.6, 0.9, B, device="cuda").view(B, 1, 1, 1, 1)
    sg = torch.linspace(0.8, 0.4, B, device="cuda").view(B, 1, 1, 1, 1)
    x0, guided = ops.cfg_x0(y, u, xt, al, sg, 7.5, rescale, return_guided=True)
    torch.cuda.synchronize()
    check_cfg_exact(y, u, xt, al, sg, 7.5, rescale, guided, x0)


# softmax_rows
SOFTMAX_COLS = (1, 7, 8, 9, 3294, 26352, 102400)


@pytest.mark.gpu
@pytest.mark.parametrize("cols", SOFTMAX_COLS)
def test_softmax_rows_bound(ops, cols):
    rows = 6 if cols > 30000 else 40
    ld = (cols + 8) // 8 * 8 + 8                                                   # ld > cols, a multiple of 8
    s = _rnd((rows, ld), 4, 3.0)
    s[0, cols - 1] = 20                                         # maximum in the last column (the scalar tail when cols % 8)
    s[1, 0] = 20                                                # maximum in the first element
    s[2, :cols] = (0.1 * s[2, :cols].float()).half()
    s[2, cols // 2] = 12                                        # one dominant logit: the others' weights are fp16 subnormals
    s[3, :cols] = -3                                            # a constant row
    p, b = softmax_ref(s, cols)
    got = ops.softmax_rows(s, cols)
    torch.cuda.synchronize()
    assert (got[:, cols:] == 0).all(), "columns cols..ld are not zeroed"
    check_bound(got[:, :cols], p, b, f"softmax_rows {rows}x{cols} ld {ld}", "softmax",
                lambda r, c: f"[row kind {['max in last column', 'max first', 'dominant logit', 'constant'][r] if r < 4 else 'random'}]")


@pytest.mark.gpu
def test_softmax_rows_refuses_102401_columns(ops):
    from star_b200.lib import StarError
    s = torch.zeros(2, 102408, dtype=HALF, device="cuda")
    n0 = ops.launch_count()
    with pytest.raises(StarError, match="do not fit in shared memory"):
        ops.softmax_rows(s, 102401)
    assert ops.launch_count() == n0, "the refused call launched a kernel"
    assert (s == 0).all()


# LayerNorm with the fused LIEM gates, row gates, spatial LIEM gate
@pytest.mark.gpu
@pytest.mark.parametrize("ratio", [0, 64])
@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("C", [320, 640, 512, 768, 1280, 3072])
def test_layernorm_gate_bound(ops, C, mode, ratio):
    """Rows 0..299 are scaled by 1e-3 .. 3e-2 (mean and spread alike): their variance after the gate runs from far below eps
    to far above it, where the output depends on the gate (elsewhere LayerNorm cancels it)."""
    rows = 999                                                   # not a multiple of the 4 / 2 rows a sub-kernel warp packs
    x = _offset_input(rows, C, ratio, seed=3, per="row")
    s = torch.ones(rows, device="cuda")
    s[:300] = torch.logspace(-3, -1.5, 300, device="cuda")
    x = (x.float() * s[:, None]).half()
    gamma = (1 + 0.1 * torch.randn(C, device="cuda")).half()
    beta = (0.1 * torch.randn(C, device="cuda")).half()
    gate = torch.rand(rows, device="cuda").half() if mode == 1 else None
    w0, w1 = 0.03125, -0.015625
    got = ops.layernorm(x, gamma, beta, mode, gate, w0, w1, eps=1e-5)
    torch.cuda.synchronize()
    y, b = gated_layernorm_ref(x, gamma, beta, 1e-5, mode, gate, w0, w1, HALF)
    check_bound(got, y, b, f"layernorm<{layernorm_instance(C)}> C{C} gate_mode {mode} |mean|/std {ratio}", "layernorm-gate")


@pytest.mark.gpu
@pytest.mark.parametrize("ratio", [16, 64])
@pytest.mark.parametrize("C", [320, 3072])
def test_layernorm_bf16_bound(ops, C, ratio):
    """gate_mode 0, as the CogVideoX blocks call it: the bound of the fp16 test_layernorm_offset_bound in bf16"""
    x = _offset_input(333, C, ratio, seed=4, per="row", dtype=BF16)
    gamma = (1 + 0.1 * torch.randn(C, device="cuda")).to(BF16)
    beta = (0.1 * torch.randn(C, device="cuda")).to(BF16)
    got = ops.layernorm(x, gamma, beta, eps=1e-6)
    torch.cuda.synchronize()
    x64 = x.to(F64)
    mean = x64.mean(1, keepdim=True)
    rstd = 1.0 / torch.sqrt(((x64 - mean) ** 2).mean(1, keepdim=True) + 1e-6)
    y, b = _norm_bound(x64, mean, rstd, gamma.to(F64), beta.to(F64), dtype=BF16)
    check_bound(got, y, b, f"bf16 layernorm<{layernorm_instance(C)}> C{C} |mean|/std {ratio}", "layernorm-bf16")


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("C", [8, 320, 3072])
def test_row_gate_external_exact(ops, dtype, C):
    x = _offset_input(555, C, 4, seed=5, per="row", dtype=dtype)
    gate = torch.rand(555, device="cuda").to(dtype)
    _assert_equal(ops.row_gate(x, 1, gate), (x.to(F64) * gate.to(F64)[:, None]).to(dtype), f"row_gate mode 1 C{C}")


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("C", [8, 320, 3072])
def test_row_gate_temporal_bound(ops, dtype, C):
    x = _offset_input(555, C, 4, seed=6, per="row", dtype=dtype)
    w0, w1 = 0.40625, -0.296875
    got = ops.row_gate(x, 2, None, w0, w1)
    torch.cuda.synchronize()
    x64 = x.to(F64)
    g, dg = _temporal_gate(x64, w0, w1, 8 * math.ceil(C / 8 / 32), dtype)
    y = x64 * g
    check_bound(got, y, _finish(y, x64.abs() * dg, dtype), f"row_gate mode 2 C{C} {dtype}", "row-gate")


LIEM_HW = [(1, 1), (1, 9), (3, 3), (6, 7), (7, 6), (7, 7), (3, 20), (17, 27)]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("H,W", LIEM_HW)
def test_liem_spatial_gate_bound(ops, dtype, H, W):
    BT, C = 3, 320
    x = _rnd_dt((BT * H * W, C), 1, dtype)
    w98 = _rnd_dt((98,), 2, dtype, 0.2)
    got = ops.liem_spatial_gate(x, w98, BT, H, W)
    torch.cuda.synchronize()
    y, b = liem_ref(x, w98, BT, H, W, dtype)
    check_bound(got.view(-1, 1), y, b, f"liem {BT}x{H}x{W} {dtype}", "liem",
                lambda r, c: f"[frame {r // (H * W)}, pixel ({r % (H * W) // W}, {r % W})]")


# qk LayerNorm + 3-D RoPE
def qk_ln_rope_ref(qkv, heads, koff, qg, qb, kg, kb, cos, sin, seq, text_len, eps, dtype):
    """fp64 value and bound of the q and k column blocks after star_qk_ln_rope.  LayerNorm(64) statistics in fp32: sums of
    QK_SUM_ROUND roundings, the variance from the rounded mean (its error enters squared), rsqrt.approx; the apply rounds
    NORM_FP32_ROUND times; the LayerNorm output is rounded to the storage type (one u, carried through the rotation's |cos|,
    |sin| <= 1); the rotation's two products and difference round in fp32."""
    u, fl = U_OUT[dtype], FLOOR[dtype]
    rows = qkv.shape[0]
    outs = []
    for off, gm, bt in ((0, qg, qb), (koff, kg, kb)):
        x = qkv[:, off:off + heads * 64].to(F64).reshape(rows, heads, 64)
        m = x.mean(-1, keepdim=True)
        var = ((x - m) ** 2).mean(-1, keepdim=True)
        rstd = 1 / torch.sqrt(var + eps)
        dm = QK_SUM_ROUND * U32 * x.abs().mean(-1, keepdim=True)
        dvar = (QK_SUM_ROUND + 2) * U32 * var + dm ** 2
        rel_rstd = 0.5 * dvar / (var + eps) + ERR_RSQRT + U32
        yn = (x - m) * rstd
        dyn = yn.abs() * rel_rstd + dm * rstd + U32 * yn.abs()
        g64, b64 = gm.to(F64), bt.to(F64)
        ln = yn * g64 + b64
        e_ln = g64.abs() * dyn + NORM_FP32_ROUND * U32 * ((yn * g64).abs() + b64.abs())
        tok = torch.arange(rows, device=qkv.device) % seq
        img = (tok >= text_len)[:, None, None]
        y, err = ln.clone(), e_ln.clone()
        if img.any():
            idx = (tok - text_len).clamp_min(0)
            c, s = cos.to(F64)[idx][:, None, :], sin.to(F64)[idx][:, None, :]
            e_in = e_ln + u * ln.abs() + fl                                     # the stored LayerNorm output
            x1, x2, e1, e2 = ln[..., 0::2], ln[..., 1::2], e_in[..., 0::2], e_in[..., 1::2]
            r = torch.empty_like(ln)
            er = torch.empty_like(ln)
            r[..., 0::2] = x1 * c[..., 0::2] - x2 * s[..., 0::2]
            r[..., 1::2] = x2 * c[..., 1::2] + x1 * s[..., 1::2]
            er[..., 0::2] = c[..., 0::2].abs() * e1 + s[..., 0::2].abs() * e2 + 2 * U32 * ((x1 * c[..., 0::2]).abs() + (x2 * s[..., 0::2]).abs())
            er[..., 1::2] = c[..., 1::2].abs() * e2 + s[..., 1::2].abs() * e1 + 2 * U32 * ((x2 * c[..., 1::2]).abs() + (x1 * s[..., 1::2]).abs())
            y, err = torch.where(img, r, y), torch.where(img, er, err)
        outs.append((y.reshape(rows, -1), _finish(y, err, dtype).reshape(rows, -1)))
    return outs


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("text_len", [0, 13, 40])
def test_qk_ln_rope_bound(ops, dtype, text_len):
    heads, seq, nseq = 3, 40, 3                                 # rows span three sequences
    ld, koff = 3 * heads * 64 + 64, heads * 64 + 64             # ld > 3 heads 64, koff != heads 64
    qkv = _offset_input(nseq * seq, ld, 0, seed=7, per="row", dtype=dtype)
    qkv[:, :heads * 64] += torch.linspace(-8, 8, heads * 64, device="cuda").to(dtype)    # per-head offsets in q
    before = qkv.clone()
    qg, qb, kg, kb = ((_rnd_dt((64,), s, dtype, 0.5).to(F32) + (1 if s % 2 == 0 else 0)).to(dtype) for s in (10, 11, 12, 13))
    ang = torch.rand(seq - text_len, 64, device="cuda", generator=torch.Generator(device="cuda").manual_seed(14)) * 6.28
    ang = ang * torch.linspace(1, 150, 64, device="cuda")                       # angles up to ~940 rad
    cos, sin = ang.cos().contiguous(), ang.sin().contiguous()
    ops.qk_ln_rope(qkv, heads, koff, qg, qb, kg, kb, cos, sin, seq, text_len, 1e-6)
    torch.cuda.synchronize()
    (yq, bq), (yk, bk) = qk_ln_rope_ref(before, heads, koff, qg, qb, kg, kb, cos, sin, seq, text_len, 1e-6, dtype)
    loc = lambda r, c: f"[sequence {r // seq}, token {r % seq} ({'text' if r % seq < text_len else 'image'}), head {c // 64}]"  # noqa: E731
    check_bound(qkv[:, :heads * 64], yq, bq, f"qk_ln_rope q text_len {text_len} {dtype}", "qk-ln-rope", loc)
    check_bound(qkv[:, koff:koff + heads * 64], yk, bk, f"qk_ln_rope k text_len {text_len} {dtype}", "qk-ln-rope", loc)
    untouched = torch.ones(ld, dtype=torch.bool, device="cuda")
    untouched[:heads * 64] = False
    untouched[koff:koff + heads * 64] = False
    _assert_equal(qkv[:, untouched], before[:, untouched], "qk_ln_rope columns outside q and k")


# elementwise
@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("n", [1, 777, 70001])
def test_silu_bound(ops, dtype, n):
    x = _rnd_dt((n,), 1, dtype, 8.0)
    if n > 100:
        x[:8] = torch.tensor([20.5, -20.5, 30, -30, 60, -60, 1000, -1000], device="cuda").to(dtype)
    got = ops.silu(x)
    torch.cuda.synchronize()
    y, err = _silu_step(x.to(F64), torch.zeros(n, dtype=F64, device="cuda"))
    check_bound(got.view(1, -1), y.view(1, -1), _finish(y, err, dtype).view(1, -1), f"silu n={n} {dtype}", "silu")


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("T", [2, 3, 8, 9])
def test_time_avgpool2_bound(ops, dtype, T):
    HW, C = 37, 264
    x = _rnd_dt((T * HW, C), 1, dtype, 30.0)
    got = ops.time_avgpool2(x, T, HW)
    torch.cuda.synchronize()
    f = x.to(F64).view(T, HW, C)
    y = torch.cat([f[:1], (f[1::2] + f[2::2]) / 2]) if T % 2 else (f[0::2] + f[1::2]) / 2
    y = y.reshape(-1, C)
    check_bound(got, y, _finish(y, U32 * y.abs(), dtype), f"time_avgpool2 T{T} {dtype}", "avgpool",
                lambda r, c: f"[output frame {r // HW}]")


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("dim", [320, 1280, 3072])
def test_sinusoidal_bound(ops, dtype, dim):
    """cos || sin of t * 10000^(-k / half) for t = 0..999.  Kernel: fast division -k / half, powf as ex2.approx(y lg2.approx
    10000) (the exponent's relative error times its size, ln 2 per unit of exponent), the fp32 product t * freq, and
    __cosf / __sinf with their range reduction."""
    t = torch.arange(1000, device="cuda")
    got = ops.sinusoidal(t, dim, dtype=dtype)
    torch.cuda.synchronize()
    half = dim // 2
    k = torch.arange(half, device="cuda", dtype=F64)
    ex = -k / half * math.log2(10000.0)
    freq = torch.exp2(ex)
    a = t.to(F64)[:, None] * freq[None, :]
    a_rel = ERR_EX2 + math.log(2) * ex.abs() * (ERR_FDIV + ERR_LG2 + U32) + U32
    err = a.abs() * (a_rel + RANGE_RED * U32) + ERR_SINCOS
    y = torch.cat([torch.cos(a), torch.sin(a)], 1)
    err = torch.cat([err, err], 1)
    check_bound(got, y, _finish(y, err, dtype), f"sinusoidal dim {dim} {dtype}", "sinusoidal",
                lambda r, c: f"[t {r}, {'cos' if c < half else 'sin'} k {c % half}]")


# temporal VAE pieces
@pytest.mark.gpu
@pytest.mark.parametrize("B,T,H,W,ldx", [(2, 1, 10, 12, 8), (1, 4, 7, 9, 5), (2, 3, 5, 6, 3)])
def test_vae_head_bound(ops, B, T, H, W, ldx):
    HW = H * W
    x = _rnd((B * T * HW, ldx), 1)
    w27, b3 = _rnd((27,), 2, 0.3), _rnd((3,), 3, 0.1)
    got = ops.vae_head(x, w27, b3, B, T, H, W)
    torch.cuda.synchronize()
    xs = F.pad(x.to(F64)[:, :3].view(B, T, HW, 3), (0, 0, 0, 0, 1, 1))                   # zero frames at both ends
    w = w27.to(F64).view(3, 3, 3)                                                        # [co][ci][dt]
    y = b3.to(F64).view(1, 1, 1, 3).expand(B, T, HW, 3).clone()
    mag = y.abs()
    for dt in range(3):
        y = y + xs[:, dt:dt + T] @ w[:, :, dt].t()
        mag = mag + xs[:, dt:dt + T].abs() @ w[:, :, dt].abs().t()
    y, mag = (t.permute(0, 1, 3, 2).reshape(B * T * 3, HW) for t in (y, mag))
    check_bound(got.view(B * T * 3, HW), y, _finish(y, VAE_HEAD_ROUND * U32 * mag, HALF), f"vae_head B{B} T{T} ldx {ldx}",
                "vae-head", lambda r, c: f"[frame {r // 3}, channel {r % 3}]")


def bilinear_ref(x, H, W):
    """fp64 bilinear resize (align_corners False) of fp32 x (NC, h, w) and its bound.  Kernel: source positions from the fp32
    scale h / H (its rounding error known exactly) with one fma, so a position error dpos moves the value by dpos times the
    largest step between the neighbouring rows (columns) of either sampled column (row); INTERP_ROUND fp32 roundings of the
    interpolation itself on values <= the largest corner."""
    nc, h, w = x.shape
    x64 = x.to(F64)
    dev = x.device

    def axis(n_out, n_in):
        scale = n_in / n_out
        s32 = float(torch.tensor(n_in, dtype=F32) / torch.tensor(n_out, dtype=F32))
        d = torch.arange(n_out, device=dev, dtype=F64) + 0.5
        pos = (d * scale - 0.5).clamp_min(0)
        i0 = pos.floor().long().clamp(max=n_in - 1)
        i1 = (i0 + 1).clamp(max=n_in - 1)
        lam = pos - i0
        dpos = d * abs(s32 - scale) + U32 * (d * s32 - 0.5).abs() + U32       # scale error, the fma, 1 - lambda
        return i0, i1, lam, dpos

    y0, y1, ly, dy = axis(H, h)
    x0, x1, lx, dx = axis(W, w)
    g = lambda yi, xi: x64[:, yi][:, :, xi]                                    # noqa: E731
    a, b, c, d = g(y0, x0), g(y0, x1), g(y1, x0), g(y1, x1)
    ly, lx = ly[None, :, None], lx[None, None, :]
    y = (1 - ly) * ((1 - lx) * a + lx * b) + ly * ((1 - lx) * c + lx * d)
    m = torch.stack([a.abs(), b.abs(), c.abs(), d.abs()]).amax(0)
    # steps adjacent to each row / column: Dr[r] = max(|x[r] - x[r-1]|, |x[r+1] - x[r]|)
    dr = F.pad((x64[:, 1:] - x64[:, :-1]).abs(), (0, 0, 1, 1))
    dr = torch.maximum(dr[:, :-1], dr[:, 1:])
    dc = F.pad((x64[:, :, 1:] - x64[:, :, :-1]).abs(), (1, 1))
    dc = torch.maximum(dc[:, :, :-1], dc[:, :, 1:])
    slope_y = torch.stack([dr[:, yi][:, :, xi] for yi in (y0, y1) for xi in (x0, x1)]).amax(0)
    slope_x = torch.stack([dc[:, yi][:, :, xi] for yi in (y0, y1) for xi in (x0, x1)]).amax(0)
    err = INTERP_ROUND * U32 * m + slope_y * dy[None, :, None] + slope_x * dx[None, None, :]
    return y, U32 * y.abs() + (1 + U32) * err + 2.0 ** -149


@pytest.mark.gpu
@pytest.mark.parametrize("shape,H,W,pad", [((4, 3, 24, 40), 96, 160, (5, 6, 3, 2)),        # upscaling
                                           ((1, 3, 240, 426), 120, 213, (0, 0, 0, 0)),     # downscaling
                                           ((2, 3, 17, 9), 17, 9, (1, 2, 3, 0)),           # identity size
                                           ((1, 3, 1, 20), 5, 50, (0, 1, 1, 0)),           # h = 1
                                           ((1, 3, 20, 1), 50, 5, (2, 0, 0, 1)),           # w = 1
                                           ((2, 3, 17, 9), 50, 31, (1, 2, 3, 0))])
def test_bilinear_pad_bound(ops, shape, H, W, pad):
    x = torch.rand(*shape, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1)) * 2 - 1
    pl, pr, pt, pb = pad
    got = ops.bilinear_pad(x, H, W, pad, 1.0)
    torch.cuda.synchronize()
    nc = math.prod(shape[:-2])
    y, b = bilinear_ref(x.view(nc, *shape[-2:]), H, W)
    ref_torch = F.interpolate(x.to(F64), size=(H, W), mode="bilinear", align_corners=False).view(nc, H, W)
    assert (ref_torch - y).abs().max().item() < 1e-12, "the fp64 restatement disagrees with F.interpolate"
    g = got.view(nc, H + pt + pb, W + pl + pr)
    inner = g[:, pt:pt + H, pl:pl + W]
    check_bound(inner.reshape(-1, W), y.reshape(-1, W), b.reshape(-1, W), f"bilinear {shape} -> {H}x{W}", "bilinear",
                lambda r, c: f"[plane {r // H}, output ({r % H}, {c})]")
    border = torch.ones_like(g, dtype=torch.bool)
    border[:, pt:pt + H, pl:pl + W] = False
    assert (g[border] == 1.0).all(), "padding is not exactly the pad value"
    if shape[-2:] == (H, W):
        _assert_equal(inner, x.view(nc, H, W), "bilinear at the identity size")


# AdaIN colour fix
ADAIN_CASES = [  # C, F, H, W, source h, w, kind
    (1, 3, 96, 128, 24, 32, "random"), (2, 2, 96, 128, 24, 32, "random"), (3, 4, 96, 128, 24, 32, "near-flat"),
    (4, 2, 60, 100, 15, 25, "constant"), (3, 1, 2880, 5120, 720, 1280, "random"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("C,Fr,H,W,h,w,kind", ADAIN_CASES)
def test_adain_color_fix_bound(ops, C, Fr, H, W, h, w, kind):
    g = torch.Generator(device="cuda").manual_seed(2)
    video = torch.randn(1, C, Fr, H, W, generator=g, device="cuda") * 0.8
    if kind == "near-flat":                   # spread 2e-3: the variance is below the 1e-5 epsilon
        video = 0.1 + 2e-3 * video
    elif kind == "constant":
        video = torch.full_like(video, 0.3)
    src = torch.rand(Fr, C, h, w, generator=g, device="cuda") * 2 - 1
    got = ops.adain_color_fix(video, src)
    got8 = ops.adain_color_fix(video, src, uint8=True)
    torch.cuda.synchronize()
    y, b = adain_ref(video, src)
    what = f"adain C{C} F{Fr} {H}x{W} from {h}x{w} ({kind})"
    check_bound(got.view(-1, C), y, b, what, "adain", lambda r, c: f"[frame {r // (H * W)}, channel {c}]")
    check_adain_u8(got8.view(-1, C), y, b, what)


@pytest.mark.gpu
def test_adain_refuses_too_many_planes(ops):
    """C * F planes are one grid row each in the statistics launch: 4 x 16400 = 65600 planes exceed 65535 and are refused on
    the host before anything is launched"""
    from star_b200.lib import StarError
    video = torch.zeros(1, 4, 16400, 1, 2, device="cuda")
    src = torch.zeros(16400, 4, 1, 2, device="cuda")
    n0 = ops.launch_count()
    with pytest.raises(StarError, match="65535 grid rows"):
        ops.adain_color_fix(video, src)
    assert ops.launch_count() == n0


# tap-GEMM entry points without a case in test_kernel_bounds_gpu.py
C4_CASES = [(2, 1, 50, 320, ""), (2, 40, 1, 320, "res"), (1, 3, 129, 320, "res"), (2, 122, 216, 320, "res")]


@pytest.mark.gpu
@pytest.mark.parametrize("BT,H,W,Cout,extras", C4_CASES)
def test_conv2d_c4_bound(ops, BT, H, W, Cout, extras):
    """im2col to K = 64 (36 taps x channels, zero padded) and one 64-wide tap-GEMM K chunk"""
    x = _rnd((BT, H, W, 4), 1)
    w9 = _rnd((Cout, 3, 3, 4), 2, 1 / 6)
    bias = _rnd((Cout,), 3, 0.1)
    res = _rnd((BT * H * W, Cout), 4) if "res" in extras else None
    got = ops.conv2d_3x3_c4(x, w9, bias, res)
    torch.cuda.synchronize()
    x64, w64 = x.to(F64), w9.to(F64)
    acc, mag = _contract("conv2d_3x3", {}, x64, w64), _contract("conv2d_3x3", {}, x64.abs(), w64.abs())
    y, b = tap_epilogue(acc, mag, 4, HALF, bias.to(F64), residual=None if res is None else res.to(F64))
    check_bound(got, y, b, f"conv2d_3x3_c4 {BT}x{H}x{W} -> {Cout} {extras}", "conv-c4",
                lambda r, c: f"[frame {r // (H * W)}, pixel ({r % (H * W) // W}, {r % W})]")


@pytest.mark.gpu
@pytest.mark.parametrize("BT,H,W,Cin,Cout", [(2, 9, 11, 64, 128), (1, 1, 17, 72, 320), (2, 18, 16, 320, 320)])
def test_conv2d_s2_bound(ops, BT, H, W, Cin, Cout):
    """the UNet downsample: stride 2, padding (2, 1) -- the stride-2 path with pad (top 2, bottom 2, left 1, right 1)"""
    x = _rnd((BT, H, W, Cin), 1)
    w9 = _rnd((Cout, 3, 3, Cin), 2, (9 * Cin) ** -0.5)
    bias = _rnd((Cout,), 3, 0.1)
    got, Ho, Wo = ops.conv2d_3x3_s2(x, w9, bias)
    torch.cuda.synchronize()
    d = {"pad": (2, 2, 1, 1)}
    x64, w64 = x.to(F64), w9.to(F64)
    acc, mag = _contract("conv2d_3x3_s2p", d, x64, w64), _contract("conv2d_3x3_s2p", d, x64.abs(), w64.abs())
    assert acc.shape[0] == BT * Ho * Wo
    y, b = tap_epilogue(acc, mag, 9 * math.ceil(Cin / 64) * 4, HALF, bias.to(F64))
    check_bound(got, y, b, f"conv2d_3x3_s2 {BT}x{H}x{W} {Cin}->{Cout}", "conv-s2")


VAE_BF16_CASES = [
    _g("bf16-c3d-K24", "conv3d_causal", "bias,res", T=3, H=5, W=7, Cin=24, Cout=300, dtype=BF16),
    _g("bf16-c3d-K128", "conv3d_causal", "bias", T=2, H=6, W=6, Cin=128, Cout=128, dtype=BF16),
    _g("bf16-s2p-K24-odd", "conv2d_3x3_s2p", "bias", BT=2, H=9, W=11, Cin=24, Cout=64, pad=(0, 1, 0, 1), dtype=BF16),
    _g("bf16-s2p-K128-even", "conv2d_3x3_s2p", "bias", BT=1, H=10, W=12, Cin=128, Cout=256, pad=(0, 1, 0, 1), dtype=BF16),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", VAE_BF16_CASES, ids=[c.id for c in VAE_BF16_CASES])
def test_vae_convs_bf16_bound(ops, case):
    got, y, bound, locate, untouched = run_gemm_case(ops, case)
    pl = plan(case)
    check_bound(got, y, bound, f"{case.id} (BN {pl.bn}, {pl.tiles} tiles)", "tapgemm-bf16", locate)
    assert untouched(), f"{case.id}: wrote outside the output view"


# GroupNorm on the bf16 library (the CogVideoX 3-D VAE)
@pytest.mark.gpu
@pytest.mark.parametrize("ns,rps,C,silu,ratio", [(2, 999, 128, 1, 16), (1, 2000, 512, 0, 64), (2, 300, 2560, 1, 64)])
def test_groupnorm_bf16_bound(ops, ns, rps, C, silu, ratio):
    x = _offset_input(ns * rps, C, ratio, seed=1, dtype=BF16)
    gamma = (1 + 0.1 * torch.randn(C, device="cuda")).to(BF16)
    beta = (0.1 * torch.randn(C, device="cuda")).to(BF16)
    got = ops.groupnorm(x, gamma, beta, ns, 1e-6, silu)
    torch.cuda.synchronize()
    mean, rstd = _group_stats(x, ns, C, 1e-6)
    chk = BoundCheck(f"bf16 groupnorm ns{ns} rows/sample {rps} C{C} silu{silu} |mean|/std {ratio}", "groupnorm-bf16",
                     lambda r, c: f"[sample {r // rps}, group {c // (C // 32)}]")
    for sample in range(ns):
        rows = slice(sample * rps, (sample + 1) * rps)
        y, b = _norm_bound(x[rows].to(F64), mean[sample], rstd[sample], gamma.to(F64), beta.to(F64), silu=bool(silu), dtype=BF16)
        chk.add(got[rows], y, b, row0=sample * rps)
    chk.done()


@pytest.mark.gpu
@pytest.mark.parametrize("ratio", [16, 64])
def test_groupnorm_mod_bf16_bound(ops, ratio):
    T, H, W, Tl, Hl, Wl, C = 5, 8, 12, 3, 4, 6, 256
    x = _offset_input(T * H * W, C, ratio, seed=2, dtype=BF16)
    gamma = (1 + 0.1 * torch.randn(C, device="cuda")).to(BF16)
    beta = (0.1 * torch.randn(C, device="cuda")).to(BF16)
    mod = _rnd_dt((Tl * Hl * Wl, 2 * C), 3, BF16)
    ymod, bmod = mod[:, :C], mod[:, C:]
    got = ops.groupnorm_mod(x, gamma, beta, ymod, bmod, T, H, W, Tl, Hl, Wl, 1e-6, True)
    torch.cuda.synchronize()
    mean, rstd = _group_stats(x, 1, C, 1e-6)
    t = torch.arange(T, device="cuda")
    ts = torch.where(t == 0, 0, 1 + (t - 1) * (Tl - 1) // (T - 1))
    src = ((ts[:, None, None] * Hl + (torch.arange(H, device="cuda") * Hl // H)[None, :, None]) * Wl
           + (torch.arange(W, device="cuda") * Wl // W)[None, None, :]).reshape(-1)
    y, b = _norm_bound(x.to(F64), mean[0], rstd[0], gamma.to(F64), beta.to(F64), ymod.to(F64)[src], bmod.to(F64)[src], True,
                       dtype=BF16)
    check_bound(got, y, b, f"bf16 groupnorm_mod T{T} {H}x{W} C{C} |mean|/std {ratio}", "groupnorm-bf16",
                lambda r, c: f"[frame {r // (H * W)}, group {c // (C // 32)}]")
