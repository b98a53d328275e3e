"""Per-element error bounds for the tap-GEMM, flash-attention, temporal-attention and norm kernels, on every dispatch path.

Each case is compared against a float64 reference built from plain torch ops (matmul, F.conv2d / F.conv3d, an explicit
softmax), and every output element must satisfy

    |got - y| <= u |y| + (1 + u) E + floor

u is the unit roundoff of the output type (the final rounding), E bounds everything the kernel does before that rounding
(fp32 accumulation, approximate intrinsics, statistics) and floor is half the output type's smallest subnormal.  E of a
linear op is proportional to M, the same fp64 reference evaluated on absolute values (sum |a w| + |bias| + ...).  The
constants are derived in the block below, one reason each; none is fitted to observed errors.

tests/util.py::assert_close bounds rel-L2 and max|err| / max|ref| and lets a wrong bias on one column, a single element a few
ulps off or one mis-masked attention key pass; test_checker_catches_injected_faults shows which.  The case tables follow the
host-side dispatch rules of star_abi.cu (tile width and box shape as tools/gemm_roofline.py restates them, temporal template)
and test_case_tables_cover_every_path checks, on the CPU, that every tile width x {full, partial last column tile} x {plain,
GEGLU}, every K-tail entry point and every temporal-attention template has a case.  Failures name the violating (row, col) positions, their tile and the worst
error / bound ratio; passing cases print their worst ratio (pytest -s).
"""
import math
from collections import namedtuple

import pytest
import torch
import torch.nn.functional as F

from tests.util import assert_close
from tools.gemm_roofline import geometry, tile_width

HALF, BF16, F64 = torch.float16, torch.bfloat16, torch.float64

# ---- error model: one place, one reason each ---------------------------------------------------------------------------------
U_OUT = {HALF: 2.0 ** -11, BF16: 2.0 ** -8}      # output rounding to nearest: half an ulp, relative
FLOOR = {HALF: 2.0 ** -25, BF16: 2.0 ** -134}    # half the smallest subnormal: absolute rounding error next to zero
U32 = 2.0 ** -24                                 # fp32 unit roundoff: accumulators, epilogue and statistics arithmetic
ROUND_PER_K16 = 4         # per k16 MMA step: tensor cores align and add the 16 exact products truncating (2^-23), then add the accumulator (2^-23)
EPILOGUE_ROUND = 8        # fp32 roundings after the accumulator: bias, rowvec, colscale and residual adds, activation arithmetic
SLOPE_GELU = 1.13         # max |gelu'(x)| (erf and tanh forms): carries the accumulator error through the activation
SLOPE_SILU = 1.1          # max |silu'(x)|
ERR_ERF_AS = 1.5e-7 + 2.0 ** -22     # erf_as: Abramowitz-Stegun 7.1.26 (|err| <= 1.5e-7) times its ex2.approx factor
ERR_TANH_APPROX = 2.0 ** -10.9       # tanh.approx.f32: about 2^-11 relative (PTX ISA), |tanh| <= 1 so also absolute
ERR_EX2 = 2.0 ** -22                 # ex2.approx.ftz.f32: relative error (PTX ISA: 2^-22.5 and better); also __expf's core
SUBNORMAL_P = 2.0 ** -25  # fp16 P: weights below 2^-14 round with absolute error up to half the smallest subnormal
# Which weights can be subnormal: the kernel rounds p = 2^(s log2e - m) against its running maximum m, which never exceeds the
# final one, so p >= e (1 - d) where e = exp(s - max s) is the reference weight and d <= K_SCORE / 2 U32 scale |q||k| + ERR_EX2
# its relative error (the score term below, and ex2.approx).  Only keys with e < 2^-14 / (1 - d) can round as subnormals, and
# 1 / (1 - d) <= 1 + 2 d for d <= 1/2, so the term sums |v| over e < 2^-14 (1 + SUBNORMAL_MARGIN d).  Their absolute errors
# sit in the unnormalised accumulator (rescaled by alpha <= 1 afterwards) and are divided by l >= 1 like the rest of it.
SUBNORMAL_MARGIN = 2
# Score error: 4 k16 steps over head_dim 64 at ROUND_PER_K16 each, plus the fp32 scale*log2e multiply and the fmaf against the
# running max (relative to |s|, itself <= |q||k|); a relative error e of every softmax weight moves the output by <= 2 e (P|V|).
K_SCORE = 2 * (4 * ROUND_PER_K16 + 6)
# Norm statistics may cost at most one more output rounding: u relative in rstd and u * std in the mean,
# i.e. |dy| <= u |gamma| (|x - mean| rstd + 1).
K_STAT = 1.0
NORM_FP32_ROUND = 4       # a = gamma rstd and b = beta - mean a rounded to fp32, the fmaf x a + b, the gamma/beta (LayerNorm) steps

NUM_SMS = 132             # H100 SXM; a case with more tiles than this runs more than one tile per persistent CTA


def _ceil(a, b):
    return -(-a // b)


# ---- the checker ---------------------------------------------------------------------------------------------------------
WORST = {}


class BoundCheck:
    """Accumulates |got - y| / bound over one or more row chunks; done() raises on any violation."""

    def __init__(self, what, family, locate=None, nshow=5):
        self.what, self.family, self.locate, self.nshow = what, family, locate, nshow
        self.worst, self.worst_at, self.nbad, self.shown, self.n = 0.0, None, 0, [], 0

    def add(self, got, y, bound, row0=0, rows=None, col0=0):
        """rows (optional): the global row index of every local row, for chunks that are not a contiguous row range"""
        assert got.shape == y.shape == bound.shape, f"{self.what}: shapes {tuple(got.shape)} {tuple(y.shape)} {tuple(bound.shape)}"
        at = lambda r, c: (int(rows[r]) if rows is not None else r + row0, c + col0)       # noqa: E731
        g = got.to(F64)
        if not torch.isfinite(g).all():
            bad = (~torch.isfinite(g)).nonzero()[: self.nshow].tolist()
            raise AssertionError(f"{self.what}: non-finite output at (row, col) {[at(r, c) for r, c in bad]}")
        ratio = (g - y).abs() / bound
        self.n += ratio.numel()
        w = ratio.max().item()
        if w > self.worst:
            flat = int(ratio.argmax().item())
            self.worst, self.worst_at = w, at(flat // ratio.shape[1], flat % ratio.shape[1])
        badmask = ratio > 1.0
        nb = int(badmask.sum().item())
        if nb:
            self.nbad += nb
            for r, c in badmask.nonzero()[: max(0, self.nshow - len(self.shown))].tolist():
                self.shown.append((*at(r, c), g[r, c].item(), y[r, c].item(), bound[r, c].item()))
        return self

    def done(self):
        WORST[self.family] = max(WORST.get(self.family, 0.0), self.worst)
        print(f"[bounds] {self.family:16s} {self.what}: worst |err|/bound {self.worst:.3f} over {self.n} elements")
        if self.nbad:
            loc = self.locate or (lambda r, c: "")
            lines = [f"  ({r}, {c}) {loc(r, c)}: got {gv:.6g} ref {yv:.6g} |err| {abs(gv - yv):.3g} bound {bv:.3g}"
                     for r, c, gv, yv, bv in self.shown]
            wr, wc = self.worst_at
            raise AssertionError(f"{self.what}: {self.nbad} of {self.n} elements exceed the bound; worst |err|/bound "
                                 f"{self.worst:.2f} at ({wr}, {wc}) {loc(wr, wc)}; first violations:\n" + "\n".join(lines))
        return self.worst


def check_bound(got, y, bound, what, family="selftest", locate=None):
    return BoundCheck(what, family, locate).add(got, y, bound).done()


def _finish(y, err, dtype):
    """bound of the final rounding of a value known to within err"""
    u = U_OUT[dtype]
    return u * y.abs() + (1 + u) * err + FLOOR[dtype]


def _gelu_erf(x):
    return 0.5 * x * (1 + torch.erf(x / math.sqrt(2.0)))


def _gelu_tanh(x):
    return 0.5 * x * (1 + torch.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * x ** 3)))


def _silu_step(z, err):
    """silu of a value z known to within err; kernels: x / (1 + __expf(-x)) with fast-math division"""
    y = z * torch.sigmoid(z)
    return y, SLOPE_SILU * err + 0.25 * z.abs() * (ERR_EX2 + z.abs() * U32) + 2 * ERR_EX2 * y.abs()


def tap_epilogue(acc, mag, k16_steps, dtype, bias=None, geglu=False, act=None, colscale=None, rowvec=None, residual=None,
                 silu=False):
    """fp64 value and bound of the tap-GEMM epilogue (tapgemm.cuh order: bias, GEGLU / GELU, colscale, rowvec, residual,
    SiLU).  acc / mag: the contraction on values / on absolute values; rowvec already gathered per output row."""
    unit = U32 * (ROUND_PER_K16 * k16_steps + EPILOGUE_ROUND)
    if bias is not None:
        acc, mag = acc + bias, mag + bias.abs()
    if geglu:
        n = acc.shape[1] // 2
        v, g, mv, mg = acc[:, :n], acc[:, n:], mag[:, :n], mag[:, n:]
        gg = _gelu_erf(g)
        y = v * gg
        ev, eg = unit * mv, unit * mg
        err = gg.abs() * ev + (v.abs() + ev) * (SLOPE_GELU * eg + 0.5 * g.abs() * ERR_ERF_AS)
    else:
        y, err = acc, unit * mag
        if act == "erf":
            y, err = _gelu_erf(acc), SLOPE_GELU * err + 0.5 * acc.abs() * ERR_ERF_AS
        elif act == "tanh":
            y, err = _gelu_tanh(acc), SLOPE_GELU * err + 0.5 * acc.abs() * ERR_TANH_APPROX
    if colscale is not None:
        y, err = y * colscale, err * colscale.abs() + U32 * (y * colscale).abs()
    for add in (rowvec, residual):
        if add is not None:
            err = err + 2 * U32 * (y.abs() + add.abs())
            y = y + add
    if silu:
        y, err = _silu_step(y, err)
    return y, _finish(y, err, dtype)


def attention_core(q, k, v, scale, dtype, causal=False, q0=0):
    """fp64 softmax(q k^T scale) v over [..., N, 64] and its bound.  Kernel error: the scores (K_SCORE), ex2.approx of every
    weight, P rounded to the storage type before the P V MMA while l sums the unrounded weights (2 u_p), the fp32 P V and l
    accumulations, fp16 P subnormals; all relative to P|V| except the last.  q0: sequence index of the first query row (a
    row chunk of a causal problem)."""
    s = (q @ k.transpose(-1, -2)).mul_(scale)
    nq, nk = s.shape[-2], s.shape[-1]
    if causal:
        qidx = q0 + torch.arange(nq, device=s.device)
        s.masked_fill_(torch.arange(nk, device=s.device)[None, :] > qidx[:, None], float("-inf"))
    e = s.sub_(s.amax(-1, keepdim=True)).exp_()
    l = e.sum(-1, keepdim=True)
    va = v.abs()
    qk = q.norm(dim=-1, keepdim=True) * k.norm(dim=-1).amax(-1, keepdim=True).unsqueeze(-1)
    score = K_SCORE * U32 * scale * qk
    sub = None
    if dtype == HALF:
        sub = ((e < 2.0 ** -14 * (1 + SUBNORMAL_MARGIN * (score / 2 + ERR_EX2))).to(F64) @ va) / l
    p = e.div_(l)
    y = p @ v
    pv = p @ va
    del s, e, p
    u_p = U_OUT[dtype]
    rel = 2 * u_p + 2 * ERR_EX2 + U32 * (ROUND_PER_K16 * _ceil(nk, 16) + _ceil(nk, 4) + 8) + score
    err = rel * pv if sub is None else rel * pv + SUBNORMAL_P * sub
    return y, _finish(y, err, dtype)


def attention_ref(q, k, v, batch, heads, nq, nk, div, scale, dtype, causal=False):
    """[batch * nq, heads * 64] fp64 value and bound of star_attention / star_attention_causal"""
    d = 64
    kvb = _ceil(batch, div)
    qf = q.to(F64)[:, :heads * d].reshape(batch, nq, heads, d).transpose(1, 2)
    kf = k.to(F64)[:, :heads * d].reshape(kvb, nk, heads, d).transpose(1, 2)
    vf = v.to(F64)[:, :heads * d].reshape(kvb, nk, heads, d).transpose(1, 2)
    idx = torch.arange(batch, device=q.device) // div
    y, b = attention_core(qf, kf[idx], vf[idx], scale, dtype, causal)
    back = lambda t: t.transpose(1, 2).reshape(batch * nq, heads * d)          # noqa: E731
    return back(y), back(b)


# ---- tap-GEMM dispatch (tile width and geometry: tools/gemm_roofline.py) ---------------------------------------------------
def stages(bn):
    """TapGemmSmem<BN>::STAGES: (A 128x64 + W BNx64) fp16 stages in 227 KB, at most 8"""
    return min((232448 - 1024 - 256) // (128 * 64 * 2 + bn * 64 * 2), 8)


Plan = namedtuple("Plan", "bn npt n_tiles m_tiles tiles iters stages k16 on box")


def plan(case):
    on, box, taps, K, N, _ = geometry(case.op, case.d)
    geglu = bool(case.flags & 1)
    bn = tile_width(N, geglu)
    npt = bn // 2 if geglu else bn
    m_tiles = math.prod(_ceil(o, b) for o, b in zip(on, box))
    n_tiles = _ceil(N, npt)
    chunks = _ceil(K, 64)
    return Plan(bn, npt, n_tiles, m_tiles, m_tiles * n_tiles, taps * chunks, stages(bn), taps * chunks * 4, on, box)


def tile_locator(pl):
    def locate(r, c):
        g, rr = [], r
        for o in pl.on:
            g.append(rr % o)
            rr //= o
        bc = [gi // bi for gi, bi in zip(g, pl.box)]
        m, mul = 0, 1
        for b, o, bx in zip(bc, pl.on, pl.box):
            m += b * mul
            mul *= _ceil(o, bx)
        return f"[m-tile {m}, n-tile {c // pl.npt}, box {tuple(bc)} of {tuple(pl.box)}, tile-local ({r}, {c % pl.npt})]"
    return locate


# ---- the tap-GEMM case table ---------------------------------------------------------------------------------------------
# extras: bias, res, rowvec (+ its divisor / row pitch), cs (colscale), oddldo / oddldres (odd row pitch), outoff / resoff
# (view offset by one element: 2-byte aligned, scalar store / load path).  flags: 1 GEGLU, 2 SiLU, 4 GELU erf, 8 GELU tanh.
G = namedtuple("G", "id op d extras flags bn dtype")


def _g(id, op, extras="", flags=0, bn=None, dtype=HALF, **d):
    return G(id, op, d, extras, flags, bn, dtype)


GEMM_CASES = [
    # tile width x {full, partial} x {one tile per CTA, several}; K chunks fewer / more than the 7 / 6 / 4 ring stages
    _g("bn160-partial", "linear", "bias", rows=300, K=320, N=300, bn=160),
    _g("bn160-full-multi", "linear", "bias,res", rows=4500, K=640, N=640, bn=160),
    _g("bn160-partial-multi-1chunk", "linear", "bias", rows=9000, K=64, N=300, bn=160),
    _g("bn256-partial-multi", "linear", "bias,res", rows=4500, K=640, N=1000, bn=256),
    _g("bn256-full", "linear", "bias", rows=300, K=320, N=256, bn=256),
    _g("bn256-full-multi-2chunks", "linear", "", rows=4500, K=128, N=1024, bn=256),
    _g("bn128-partial-multi", "linear", "bias", rows=2000, K=640, N=1150, bn=128),
    _g("bn128-partial-multi-3chunks-rowvec", "linear", "bias,rowvec,res", rows=2000, K=192, N=1150, bn=128, rv_div=7),
    _g("bn128-full", "linear", "bias", rows=200, K=320, N=128, bn=128),
    # GEGLU on both of its tile widths
    _g("geglu-bn128-full", "linear", "bias", 1, rows=300, K=320, N=320, bn=128),
    _g("geglu-bn128-partial", "linear", "bias", 1, rows=300, K=320, N=300, bn=128),
    _g("geglu-bn256-full", "linear", "bias", 1, rows=300, K=320, N=1280, bn=256),
    _g("geglu-bn256-partial-multi", "linear", "bias", 1, rows=4500, K=320, N=1000, bn=256),
    # K tails (K % 64 != 0): the last W box of tap t reaches into tap t+1, A is zero-filled past K
    _g("linear-K8", "linear", "bias", rows=300, K=8, N=300, bn=160),
    _g("linear-K24", "linear", "bias,res", rows=300, K=24, N=1000, bn=256),
    _g("linear-K72", "linear", "bias", rows=300, K=72, N=1150, bn=128),
    _g("linear-K136-geglu", "linear", "bias", 1, rows=300, K=136, N=300, bn=128),
    # epilogues
    _g("bias-rowvec-res-silu", "linear", "bias,rowvec,res", 2, rows=300, K=320, N=320, bn=160, rv_div=7),
    _g("gelu-erf", "linear", "bias", 4, rows=300, K=320, N=1000, bn=256),
    _g("linear_ex-colscale-res-gelu-tanh", "linear_ex", "bias,cs,res", 8, rows=300, K=320, N=1150, bn=128),
    # odd N, odd row pitches, 2-byte-aligned views: scalar store / load paths
    _g("N3", "linear", "bias,res", rows=300, K=64, N=3, bn=128),
    _g("N127-silu", "linear", "bias,res", 2, rows=300, K=64, N=127, bn=128),
    _g("odd-ldo", "linear", "bias,oddldo", rows=300, K=320, N=300, bn=160),
    _g("odd-ldres", "linear", "bias,res,oddldres", rows=300, K=320, N=256, bn=256),
    _g("out-offset-1", "linear", "bias,res,outoff", rows=300, K=320, N=300, bn=160),
    _g("res-offset-1", "linear", "bias,res,resoff", rows=300, K=64, N=1150, bn=128),
    # conv2d 3x3: W > 128, H = 1, W = 1, several frames per box with a ragged last box, K tails
    _g("conv-W129", "conv2d_3x3", "bias,res", BT=1, H=3, W=129, Cin=64, Cout=128, bn=128),
    _g("conv-W200-K72", "conv2d_3x3", "bias", BT=2, H=2, W=200, Cin=72, Cout=300, bn=160),
    _g("conv-H1-rowvec", "conv2d_3x3", "bias,rowvec,res", BT=3, H=1, W=50, Cin=64, Cout=256, bn=256, rv_div=50),
    _g("conv-W1", "conv2d_3x3", "bias", BT=2, H=40, W=1, Cin=64, Cout=160, bn=160),
    _g("conv-BT11-4x4-rowvec", "conv2d_3x3", "bias,rowvec,res", BT=11, H=4, W=4, Cin=64, Cout=320, bn=160, rv_div=48),
    _g("conv-K8", "conv2d_3x3", "bias", BT=2, H=6, W=10, Cin=8, Cout=64, bn=128),
    _g("conv-K24", "conv2d_3x3", "bias,res", BT=3, H=5, W=9, Cin=24, Cout=1000, bn=256),
    _g("conv-K136", "conv2d_3x3", "bias", BT=2, H=7, W=12, Cin=136, Cout=300, bn=160),
    # stride-2 conv with explicit padding: odd / even H, W, H = 1, K tails
    _g("s2p-K8-odd", "conv2d_3x3_s2p", "bias", BT=2, H=9, W=11, Cin=8, Cout=64, pad=(0, 1, 0, 1), bn=128),
    _g("s2p-K24-even", "conv2d_3x3_s2p", "bias", BT=2, H=10, W=12, Cin=24, Cout=300, pad=(2, 2, 1, 1), bn=160),
    _g("s2p-K72-H1", "conv2d_3x3_s2p", "bias", BT=3, H=1, W=17, Cin=72, Cout=256, pad=(1, 1, 1, 1), bn=256),
    _g("s2p-K136", "conv2d_3x3_s2p", "bias", BT=1, H=8, W=7, Cin=136, Cout=128, pad=(0, 1, 0, 1), bn=128),
    # temporal conv: HW < 128 packs several frames per box (ragged last box), two clips that must not bleed into each other
    _g("t3-HW1-K8", "conv_t3", "bias,res", B=2, T=130, HW=1, Cin=8, Cout=64, bn=128),
    _g("t3-HW50-K24", "conv_t3", "bias", B=2, T=5, HW=50, Cin=24, Cout=300, bn=160),
    _g("t3-HW127-K72", "conv_t3", "bias,res", B=2, T=3, HW=127, Cin=72, Cout=256, bn=256),
    _g("t3-HW129-K136", "conv_t3", "bias", B=2, T=3, HW=129, Cin=136, Cout=128, bn=128),
    # causal Conv3d 3x3x3 (27 taps)
    _g("c3d-K8", "conv3d_causal", "bias", T=3, H=5, W=7, Cin=8, Cout=64, bn=128),
    _g("c3d-K24", "conv3d_causal", "bias,res", T=2, H=4, W=4, Cin=24, Cout=300, bn=160),
    _g("c3d-K72", "conv3d_causal", "bias", T=5, H=3, W=9, Cin=72, Cout=1000, bn=256),
    _g("c3d-K136", "conv3d_causal", "bias,res", T=2, H=6, W=6, Cin=136, Cout=128, bn=128),
    # bf16 library (CogVideoX DiT)
    _g("bf16-bn160-partial", "linear", "bias,res", rows=300, K=320, N=300, bn=160, dtype=BF16),
    _g("bf16-bn256-partial-multi", "linear", "bias", rows=4500, K=640, N=1000, bn=256, dtype=BF16),
    _g("bf16-bn128-K72", "linear", "bias,res", rows=300, K=72, N=1150, bn=128, dtype=BF16),
    _g("bf16-linear_ex-tanh", "linear_ex", "bias,cs,res", 8, rows=300, K=320, N=640, bn=160, dtype=BF16),
    _g("bf16-geglu-partial", "linear", "bias", 1, rows=300, K=320, N=300, bn=128, dtype=BF16),
    _g("bf16-conv-K24", "conv2d_3x3", "bias,res", BT=3, H=5, W=9, Cin=24, Cout=300, bn=160, dtype=BF16),
]

K_TAIL_OPS = ("linear", "conv2d_3x3", "conv_t3", "conv3d_causal", "conv2d_3x3_s2p")
K_TAILS = (8, 24, 72, 136)


def _contract(op, d, x, w):
    """fp64 contraction of one entry point on (x, w) as [rows, Cout]"""
    if op in ("linear", "linear_ex"):
        return x @ w.t()
    if op == "conv2d_3x3":
        y = F.conv2d(x.permute(0, 3, 1, 2), w.permute(0, 3, 1, 2), padding=1)
        return y.permute(0, 2, 3, 1).reshape(-1, w.shape[0])
    if op == "conv2d_3x3_s2p":
        pt, pb, pl, pr = d["pad"]
        y = F.conv2d(F.pad(x.permute(0, 3, 1, 2), (pl, pr, pt, pb)), w.permute(0, 3, 1, 2), stride=2)
        return y.permute(0, 2, 3, 1).reshape(-1, w.shape[0])
    if op == "conv_t3":
        xb = x.reshape(d["B"], d["T"], d["HW"], -1).permute(0, 3, 1, 2)
        y = F.conv2d(xb, w.permute(0, 2, 1).unsqueeze(-1), padding=(1, 0))
        return y.permute(0, 2, 3, 1).reshape(-1, w.shape[0])
    if op == "conv3d_causal":
        x5 = x.reshape(1, d["T"] + 2, d["H"], d["W"], -1).permute(0, 4, 1, 2, 3)
        y = F.conv3d(x5, w.permute(0, 4, 1, 2, 3), padding=(0, 1, 1))
        return y.permute(0, 2, 3, 4, 1).reshape(-1, w.shape[0])
    raise ValueError(op)


def _rnd(shape, seed, scale=1.0, dtype=HALF, device="cuda"):
    g = torch.Generator(device=device).manual_seed(seed)
    return (torch.randn(*shape, generator=g, device=device) * scale).to(dtype)


def _view(rows, n, ld, offset, dtype, fill=None, seed=None):
    """[rows, n] view of a fresh buffer with row pitch ld whose first element sits `offset` elements into the allocation"""
    if seed is not None:
        flat = _rnd((offset + rows * ld,), seed, dtype=dtype)
    else:
        flat = torch.full((offset + rows * ld,), fill, dtype=dtype, device="cuda")
    return flat, flat[offset:].view(rows, ld)[:, :n]


SENTINEL = -1024.0          # exact in fp16 and bf16


def run_gemm_case(O, case):
    """launch one case; returns (got, fp64 value, bound, locator, untouched-region check or None)"""
    d, op, dt, ex = case.d, case.op, case.dtype, case.extras
    pl = plan(case)
    on, box, taps, K, N, _ = geometry(op, d)
    geglu = bool(case.flags & 1)
    wrows = 2 * N if geglu else N
    if op in ("linear", "linear_ex"):
        x = _rnd((d["rows"], K), 1, dtype=dt)
        w = _rnd((wrows, K), 2, K ** -0.5, dt)
    elif op == "conv2d_3x3" or op == "conv2d_3x3_s2p":
        x = _rnd((d["BT"], d["H"], d["W"], K), 1, dtype=dt)
        w = _rnd((N, 3, 3, K), 2, (9 * K) ** -0.5, dt)
    elif op == "conv_t3":
        x = _rnd((d["B"] * d["T"] * d["HW"], K), 1, dtype=dt)
        w = _rnd((N, 3, K), 2, (3 * K) ** -0.5, dt)
    else:
        x = _rnd(((d["T"] + 2) * d["H"] * d["W"], K), 1, dtype=dt)
        w = _rnd((N, 3, 3, 3, K), 2, (27 * K) ** -0.5, dt)
    rows = math.prod(on)
    bias = _rnd((wrows,), 3, 0.1, dt) if "bias" in ex else None
    cs = _rnd((N,), 4, dtype=dt) if "cs" in ex else None
    res = rv = rv_idx = None
    if "res" in ex:
        ldr = N + 1 if "oddldres" in ex else N
        _, res = _view(rows, N, ldr, 1 if "resoff" in ex else 0, dt, seed=5)
    if "rowvec" in ex:
        div = d["rv_div"]
        nrv = _ceil(rows, div)
        if op == "conv2d_3x3":                                           # a column slice of a wider matrix: ldrowvec > N
            rv = _rnd((nrv, N + 40), 6, dtype=dt)[:, 8:8 + N]
        else:
            rv = _rnd((nrv, N), 6, dtype=dt)
        rv_idx = torch.arange(rows, device="cuda") // div
    ldo = N + 1 if "oddldo" in ex else (N + 8 if "outoff" in ex else N)
    outflat, out = _view(rows, N, ldo, 1 if "outoff" in ex else 0, dt, fill=SENTINEL)

    if op == "linear":
        O.linear(x, w, bias, res, rv, d.get("rv_div", 1), case.flags, out=out)
    elif op == "linear_ex":
        O.linear_ex(x, w, bias, cs, res, case.flags, out=out)
    elif op == "conv2d_3x3":
        O.conv2d_3x3(x, w, bias, rv, d.get("rv_div", 1), res, out=out)
    elif op == "conv2d_3x3_s2p":
        got, _, _ = O.conv2d_3x3_s2p(x, w, bias, d["pad"])
        out.copy_(got)
    elif op == "conv_t3":
        O.conv_t3(x, w, bias, res, d["B"], d["T"], d["HW"], out=out)
    else:
        O.conv3d_causal(x, w, d["T"], d["H"], d["W"], bias, res, out=out)
    torch.cuda.synchronize()

    x64, w64 = x.to(F64), w.to(F64)
    acc, mag = _contract(op, d, x64, w64), _contract(op, d, x64.abs(), w64.abs())
    f64 = lambda t: None if t is None else t.to(F64)                    # noqa: E731
    y, bound = tap_epilogue(acc, mag, pl.k16, dt, f64(bias), geglu, {4: "erf", 8: "tanh"}.get(case.flags & 12),
                            f64(cs), None if rv is None else rv.to(F64)[rv_idx], f64(res), bool(case.flags & 2))

    def untouched():
        mask = torch.ones_like(outflat, dtype=torch.bool)
        off = 1 if "outoff" in ex else 0
        mask[off:].view(rows, ldo)[:, :N] = False
        return bool((outflat[mask] == SENTINEL).all())
    return out, y, bound, tile_locator(pl), untouched


# ---- temporal attention and norm tables ----------------------------------------------------------------------------------
def temporal_template(t):
    """star_temporal_attention: T <= 64 runs temporal_attn2_kernel<TP> with TP = T padded to 16, else the long kernel"""
    return "long" if t > 64 else _ceil(t, 16) * 16


TEMPORAL_T = (1, 2, 15, 16, 17, 31, 32, 33, 47, 48, 49, 63, 64, 65)


def layernorm_instance(c):
    """star_layernorm: sub-kernels for C = 320 / 640, else layernorm_kernel<N> with N >= 16-byte groups per lane"""
    if c in (320, 640):
        return f"sub{c}"
    oct_ = _ceil(c // 8, 32)
    return 2 if oct_ <= 2 else 3 if oct_ <= 3 else 5 if oct_ <= 5 else 12


LAYERNORM_C = (512, 768, 1280, 3072, 320, 640)


# ---- CPU tests: the checker and the case tables --------------------------------------------------------------------------
def _cpu_linear(rows, K, N, seed):
    a = _rnd((rows, K), seed, device="cpu")
    w = _rnd((N, K), seed + 1, K ** -0.5, device="cpu")
    bias = _rnd((N,), seed + 2, 0.1, device="cpu")
    a64, w64 = a.double(), w.double()
    return tap_epilogue(a64 @ w64.t(), a64.abs() @ w64.abs().t(), 4 * _ceil(K, 64), HALF, bias.double())


def test_checker_catches_injected_faults():
    """A simulated kernel output (the fp64 reference rounded to fp16) passes the per-element checker; each injected fault
    fails it.  The table printed shows which faults the rel-L2 / max-abs check of tests/util.py lets through."""
    rows, K, N = 300, 320, 1280                       # a UNet width: one wrong column is 1 / sqrt(N) of the rel-L2
    y, bound = _cpu_linear(rows, K, N, seed=10)
    clean = y.half()
    check_bound(clean, y, bound, "clean fp16 rounding")
    faults = {}

    r, c = [int(i) for i in ((y.abs() >= 1) & (y.abs() < 2)).nonzero()[0]]     # |y| in [1, 2): half an ulp is 2^-11
    g = clean.clone()
    g[r, c] = (g[r, c].double() + 8 * 2.0 ** -11).half()
    faults["one element 8 half-ulps off"] = (g, y, bound)

    g = clean.clone()
    g[:, 1000] = (y[:, 1000] + 0.05).half()
    faults["bias +0.05 on one column"] = (g, y, bound)

    g = clean.clone()
    g[290] = 0                                          # rows 256..299: the ragged last 128-row tile
    faults["one row of the ragged tile zeroed"] = (g, y, bound)

    nq, nk = 1000, 300
    q, k, v = (_rnd((nq if i == 0 else nk, 64), 20 + i, device="cpu") for i in range(3))
    ya, ba = attention_ref(q, k, v, 1, 1, nq, nk, 1, 0.125, HALF)
    g = ya.half()
    check_bound(g, ya, ba, "clean attention")
    short, _ = attention_ref(q, k[:nk - 1], v[:nk - 1], 1, 1, nq, nk - 1, 1, 0.125, HALF)
    g[7] = short[7].half()
    faults["attention row 7 misses its last key"] = (g, ya, ba)

    missed_by_assert_close = []
    for name, (g, ref, b) in faults.items():
        with pytest.raises(AssertionError):
            check_bound(g, ref, b, name)
        try:
            assert_close(g, ref.half(), what=name)
            missed_by_assert_close.append(name)
        except AssertionError:
            pass
    print("[bounds] faults assert_close lets pass:", missed_by_assert_close)
    assert missed_by_assert_close, "every injected fault is also caught by assert_close"


def test_case_tables_cover_every_path():
    assert {bn: stages(bn) for bn in (128, 160, 256)} == {128: 7, 160: 6, 256: 4}
    cells = set()
    for case in GEMM_CASES:
        pl = plan(case)
        assert pl.bn == case.bn, f"{case.id}: the tile-width rule picks {pl.bn}, the case expects {case.bn}"
        geglu = bool(case.flags & 1)
        N = geometry(case.op, case.d)[4]
        cells.add(("geglu" if geglu else "plain", pl.bn, "partial" if N % pl.npt else "full"))
        if pl.tiles > NUM_SMS:
            cells.add(("multi-tile", pl.bn))
        cells.add(("ring", pl.bn, "fewer" if pl.iters < pl.stages else "more"))
        K = geometry(case.op, case.d)[3]
        if K % 64:
            cells.add(("ktail", case.op.replace("linear_ex", "linear"), K))
        if case.op in ("conv2d_3x3", "conv3d_causal"):
            if case.d["W"] > 128:
                cells.add(("conv", "W>128"))
            if case.d["H"] == 1:
                cells.add(("conv", "H=1"))
            if case.d["W"] == 1:
                cells.add(("conv", "W=1"))
            if pl.box[2] > 1 and pl.on[2] % pl.box[2]:
                cells.add(("conv", "multi-frame ragged box"))
        if case.op == "conv_t3":
            cells.add(("t3", case.d["HW"]))
        if case.op == "conv2d_3x3_s2p":
            cells.add(("s2p", "H=1" if case.d["H"] == 1 else ("odd" if case.d["H"] % 2 else "even")))
        for e in ("oddldo", "oddldres", "outoff", "resoff", "rowvec", "cs"):
            if e in case.extras:
                cells.add(("epi", e))
        if case.flags & 14:
            cells.add(("act", case.flags & 14))
        if N % 2:
            cells.add(("odd N", N))
        if case.dtype == BF16:
            cells.add(("bf16", case.op))
    want = {("plain", bn, fill) for bn in (128, 160, 256) for fill in ("full", "partial")}
    want |= {("geglu", bn, fill) for bn in (128, 256) for fill in ("full", "partial")}
    want |= {("multi-tile", bn) for bn in (128, 160, 256)}
    want |= {("ring", bn, r) for bn in (128, 160, 256) for r in ("fewer", "more")}
    want |= {("ktail", op, k) for op in K_TAIL_OPS for k in K_TAILS}
    want |= {("conv", g) for g in ("W>128", "H=1", "W=1", "multi-frame ragged box")}
    want |= {("t3", hw) for hw in (1, 50, 127, 129)} | {("s2p", g) for g in ("H=1", "odd", "even")}
    want |= {("epi", e) for e in ("oddldo", "oddldres", "outoff", "resoff", "rowvec", "cs")}
    want |= {("act", 2), ("act", 4), ("act", 8), ("odd N", 3), ("odd N", 127), ("bf16", "linear"), ("bf16", "linear_ex")}
    missing = want - cells
    assert not missing, f"dispatch cells without a case: {sorted(map(str, missing))}"

    templates = {temporal_template(t) for t in TEMPORAL_T}
    assert templates == {16, 32, 48, 64, "long"}
    for b in (16, 32, 48, 64):                           # both sides of every template boundary
        assert b in TEMPORAL_T and b + 1 in TEMPORAL_T
    assert 1 in TEMPORAL_T
    assert {layernorm_instance(c) for c in LAYERNORM_C} == {2, 3, 5, 12, "sub320", "sub640"}


# ---- GPU: tap-GEMM -------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ops():
    from star_b200 import ops as O
    yield O
    print(f"[bounds] worst |err|/bound per family: { {k: round(v, 3) for k, v in sorted(WORST.items())} }; "
          f"peak device memory {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")


@pytest.mark.gpu
@pytest.mark.parametrize("case", GEMM_CASES, ids=[c.id for c in GEMM_CASES])
def test_tapgemm_bound(ops, case):
    got, y, bound, locate, untouched = run_gemm_case(ops, case)
    fam = "tapgemm" + ("-bf16" if case.dtype == BF16 else "")
    pl = plan(case)
    check_bound(got, y, bound, f"{case.id} (BN {pl.bn}, {pl.tiles} tiles, {pl.iters} K chunks)", fam, locate)
    assert untouched(), f"{case.id}: wrote outside the output view"


# ---- GPU: flash attention ------------------------------------------------------------------------------------------------
ATTN_CASES = [(nq, 300, 0.125 if i % 2 else 1.0) for i, nq in enumerate((1, 5, 64, 65, 127, 129))] + \
             [(65, nk, 0.125 if i % 2 == 0 else 1.0) for i, nk in enumerate((1, 8, 127, 128, 129, 300))]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [HALF, BF16], ids=["fp16", "bf16"])
@pytest.mark.parametrize("nq,nk,scale", ATTN_CASES)
def test_attention_bound(ops, nq, nk, scale, dtype):
    """batch 5 over 3 kv batches (kv_batch_div 2 does not divide it), 2 heads"""
    batch, heads, div = 5, 2, 2
    C = heads * 64
    q = _rnd((batch * nq, C), 1, dtype=dtype)
    kv = _rnd((_ceil(batch, div) * nk, 2 * C), 2, dtype=dtype)
    k, v = kv[:, :C], kv[:, C:]
    got = ops.attention(q, k, v, batch, heads, nq, nk, div, scale)
    torch.cuda.synchronize()
    y, b = attention_ref(q, k, v, batch, heads, nq, nk, div, scale, dtype)
    fam = "attention" + ("-bf16" if dtype == BF16 else "")
    check_bound(got, y, b, f"b{batch} h{heads} {nq}x{nk} div{div} scale {scale}", fam,
                lambda r, c: f"[batch {r // nq}, q-tile {r % nq // 128}, query {r % nq}, head {c // 64}]")


@pytest.mark.gpu
def test_attention_strided_views_bound(ops):
    """Q / K / V column views of one buffer with ld > 3 heads 64, O a column view of a wider buffer"""
    batch, heads, n = 3, 2, 200
    C = heads * 64
    buf = _rnd((batch * n, 3 * C + 64), 1)
    q, k, v = buf[:, 8:8 + C], buf[:, 8 + C + 16:8 + 2 * C + 16], buf[:, 3 * C + 56 - C:3 * C + 56]
    obuf = torch.full((batch * n, C + 72), SENTINEL, dtype=HALF, device="cuda")
    out = obuf[:, 32:32 + C]
    ops.attention(q, k, v, batch, heads, n, n, 1, 0.125, out=out)
    torch.cuda.synchronize()
    y, b = attention_ref(q, k, v, batch, heads, n, n, 1, 0.125, HALF)
    check_bound(out, y, b, "strided q/k/v/out views", "attention",
                lambda r, c: f"[batch {r // n}, q-tile {r % n // 128}, head {c // 64}]")
    assert (obuf[:, :32] == SENTINEL).all() and (obuf[:, 32 + C:] == SENTINEL).all()


@pytest.mark.gpu
def test_attention_peaky_first_and_last_tile_bound(ops):
    """Rows whose logit maximum sits only in the last (partial) key tile, or only in the first: the running maximum appears
    late, or every later tile is rescaled against an early one."""
    nq, nk, heads = 200, 300, 1
    g = torch.Generator(device="cuda").manual_seed(7)
    u = (torch.randint(0, 2, (2, 64), generator=g, device="cuda") * 2 - 1).float()      # +-1 directions, |u|^2 = 64
    k = torch.randn(nk, 64, generator=g, device="cuda") * 0.5
    k[nk - 1], k[0] = 1.25 * u[0], 1.25 * u[1]
    q = torch.randn(nq, 64, generator=g, device="cuda") * 0.3
    q[0::3] = 1.25 * u[0] + 0.05 * q[0::3]            # logit ~ 0.125 * 100 = 12.5 on the last key only
    q[1::3] = 1.25 * u[1] + 0.05 * q[1::3]            # ... on the first key only
    v = torch.randn(nk, 64, generator=g, device="cuda")
    q, k, v = q.half(), k.half(), v.half()
    s = q.float() @ k.float().t()
    assert (s[0::3].argmax(1) == nk - 1).all() and (s[1::3].argmax(1) == 0).all()
    got = ops.attention(q, k, v, 1, heads, nq, nk, 1, 0.125)
    torch.cuda.synchronize()
    y, b = attention_ref(q, k, v, 1, heads, nq, nk, 1, 0.125, HALF)
    check_bound(got, y, b, "peaky rows (max in the first / last key tile)", "attention",
                lambda r, c: f"[q-tile {r // 128}, query {r} (peak in {'last' if r % 3 == 0 else 'first' if r % 3 == 1 else 'no'} tile)]")


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 2, 127, 128, 129, 257])
def test_attention_causal_bound(ops, n):
    batch, heads = 2, 2
    C = heads * 64
    qkv = _rnd((batch * n, 3 * C), 1)
    q, k, v = qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:]
    got = ops.attention_causal(q, k, v, batch, heads, n, 0.125)
    torch.cuda.synchronize()
    y, b = attention_ref(q, k, v, batch, heads, n, n, 1, 0.125, HALF, causal=True)
    check_bound(got, y, b, f"causal b{batch} h{heads} N{n}", "attention-causal",
                lambda r, c: f"[batch {r // n}, q-tile {r % n // 128}, query {r % n}, head {c // 64}]")


# ---- GPU: temporal attention ---------------------------------------------------------------------------------------------
def temporal_ref(qkv, B, T, HW, heads, Ci, scale, dtype):
    d = 64
    x = qkv.to(F64).reshape(B, T, HW, -1)
    split = lambda o: x[..., o:o + heads * d].reshape(B, T, HW, heads, d).permute(0, 2, 3, 1, 4)     # noqa: E731
    y, b = attention_core(split(0), split(Ci), split(2 * Ci), scale, dtype)
    back = lambda t: t.permute(0, 3, 1, 2, 4).reshape(B * T * HW, heads * d)                       # noqa: E731
    return back(y), back(b)


TEMPORAL_CASES = [(1, t, 37, 2, 128, 384) for t in TEMPORAL_T] + [
    (2, 17, 700, 5, 320, 960),          # 7000 items over 2112 warps: every warp runs several items with T % 16 != 0
    (2, 33, 700, 5, 320, 960),
    (1, 49, 40, 3, 256, 832),           # heads * 64 < Ci, ld > 3 Ci
    (1, 65, 40, 3, 256, 832),           # the same on the long kernel
]


@pytest.mark.gpu
@pytest.mark.parametrize("B,T,HW,heads,Ci,ld", TEMPORAL_CASES)
def test_temporal_attention_bound(ops, B, T, HW, heads, Ci, ld):
    buf = _rnd((B * T * HW, ld), 1)
    qkv = buf[:, :3 * Ci] if ld > 3 * Ci else buf
    got = ops.temporal_attention(qkv, B, T, HW, heads, Ci, 0.125)[:, :heads * 64]
    torch.cuda.synchronize()
    y, b = temporal_ref(qkv, B, T, HW, heads, Ci, 0.125, HALF)
    check_bound(got, y, b, f"B{B} T{T} HW{HW} heads{heads} Ci{Ci} ld{ld} ({temporal_template(T)})", "temporal",
                lambda r, c: f"[item (b {r // (T * HW)}, px {r % HW}, head {c // 64}), frame {r // HW % T}]")


# ---- GPU: norm statistics under a mean offset ----------------------------------------------------------------------------
def _offset_input(rows, C, ratio, seed, per="group", dtype=HALF):
    """fp16 (or bf16) rows with unit spread around a per-group (GroupNorm) or per-row (LayerNorm) mean of +-ratio"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    if per == "group":
        mu = (ratio * (torch.randint(0, 2, (32,), generator=g, device="cuda") * 2 - 1)).repeat_interleave(C // 32)
    else:
        mu = (ratio * (torch.randint(0, 2, (rows, 1), generator=g, device="cuda") * 2 - 1))
    x = torch.empty(rows, C, dtype=dtype, device="cuda")
    step = 1 << 16
    for r0 in range(0, rows, step):
        r1 = min(rows, r0 + step)
        x[r0:r1] = (torch.randn(r1 - r0, C, generator=g, device="cuda") + (mu if per == "group" else mu[r0:r1])).to(dtype)
    return x


def _norm_bound(x64, mean, rstd, gamma, beta, ymod=None, bmod=None, silu=False, dtype=HALF):
    """fp64 value and bound of y = (x - mean) rstd gamma + beta (* ymod + bmod) (SiLU)"""
    yn = (x64 - mean) * rstd
    y = yn * gamma + beta
    err = K_STAT * U_OUT[dtype] * gamma.abs() * (yn.abs() + 1) + NORM_FP32_ROUND * U32 * (x64.abs() * rstd * gamma.abs() + beta.abs())
    if ymod is not None:
        err = err * ymod.abs() + 2 * U32 * ((y * ymod).abs() + bmod.abs())
        y = y * ymod + bmod
    if silu:
        y, err = _silu_step(y, err)
    return y, _finish(y, err, dtype)


def _group_stats(x, ns, C, eps, step=1 << 16):
    """fp64 per (sample, channel) mean / rstd of GroupNorm(32), two passes over row chunks"""
    rps = x.shape[0] // ns
    cg = C // 32
    xs = x.view(ns, rps, C)
    s = torch.zeros(ns, C, dtype=F64, device=x.device)
    for r0 in range(0, rps, step):
        s += xs[:, r0:r0 + step].to(F64).sum(1)
    mean = (s.view(ns, 32, cg).sum(-1) / (rps * cg)).repeat_interleave(cg, dim=1)
    q = torch.zeros(ns, C, dtype=F64, device=x.device)
    for r0 in range(0, rps, step):
        q += ((xs[:, r0:r0 + step].to(F64) - mean[:, None]) ** 2).sum(1)
    var = (q.view(ns, 32, cg).sum(-1) / (rps * cg)).repeat_interleave(cg, dim=1)
    return mean, 1.0 / torch.sqrt(var + eps)


GN_CASES = [  # ns, rows per sample, C, silu, |mean| / std
    (2, 999, 320, 1, 16), (2, 999, 320, 0, 64), (1, 2000, 1280, 1, 64), (3, 300, 2048, 0, 64),    # gn_stats2 (C <= 2048)
    (2, 300, 2560, 0, 16), (2, 300, 2560, 1, 64),                                                # gn_stats (first generation)
    (1, 32 * 26352, 320, 1, 64),                        # the level-0 clip: 32 frames of 122 x 216, longest per-thread sums
]


@pytest.mark.gpu
@pytest.mark.parametrize("ns,rps,C,silu,ratio", GN_CASES)
def test_groupnorm_offset_bound(ops, ns, rps, C, silu, ratio):
    x = _offset_input(ns * rps, C, ratio, seed=1)
    gamma = (1 + 0.1 * torch.randn(C, device="cuda")).half()
    beta = (0.1 * torch.randn(C, device="cuda")).half()
    eps = 1e-5
    got = ops.groupnorm(x, gamma, beta, ns, eps, silu)
    torch.cuda.synchronize()
    mean, rstd = _group_stats(x, ns, C, eps)
    chk = BoundCheck(f"groupnorm ns{ns} rows/sample {rps} C{C} silu{silu} |mean|/std {ratio}", "groupnorm",
                     lambda r, c: f"[sample {r // rps}, group {c // (C // 32)}]")
    g64, b64 = gamma.to(F64), beta.to(F64)
    step = 1 << 16
    for sample in range(ns):
        for r0 in range(0, rps, step):
            r1 = min(rps, r0 + step)
            rows = slice(sample * rps + r0, sample * rps + r1)
            y, b = _norm_bound(x[rows].to(F64), mean[sample], rstd[sample], g64, b64, silu=bool(silu))
            chk.add(got[rows], y, b, row0=sample * rps + r0)
            del y, b
    chk.done()


@pytest.mark.gpu
@pytest.mark.parametrize("ratio", [16, 64])
def test_groupnorm_mod_offset_bound(ops, ratio):
    T, H, W, Tl, Hl, Wl, C = 5, 8, 12, 3, 4, 6, 256          # odd T: the first frame maps to latent frame 0 alone
    rows = T * H * W
    x = _offset_input(rows, C, ratio, seed=2)
    gamma = (1 + 0.1 * torch.randn(C, device="cuda")).half()
    beta = (0.1 * torch.randn(C, device="cuda")).half()
    mod = _rnd((Tl * Hl * Wl, 2 * C), 3)
    ymod, bmod = mod[:, :C], mod[:, C:]
    got = ops.groupnorm_mod(x, gamma, beta, ymod, bmod, T, H, W, Tl, Hl, Wl, 1e-6, True)
    torch.cuda.synchronize()
    mean, rstd = _group_stats(x, 1, C, 1e-6)
    t = torch.arange(T, device="cuda")
    ts = torch.where(t == 0, 0, 1 + (t - 1) * (Tl - 1) // (T - 1))
    src = ((ts[:, None, None] * Hl + (torch.arange(H, device="cuda") * Hl // H)[None, :, None]) * Wl
           + (torch.arange(W, device="cuda") * Wl // W)[None, None, :]).reshape(-1)
    y, b = _norm_bound(x.to(F64), mean[0], rstd[0], gamma.to(F64), beta.to(F64), ymod.to(F64)[src], bmod.to(F64)[src], True)
    check_bound(got, y, b, f"groupnorm_mod T{T} {H}x{W} C{C} |mean|/std {ratio}", "groupnorm",
                lambda r, c: f"[frame {r // (H * W)}, group {c // (C // 32)}]")


@pytest.mark.gpu
@pytest.mark.parametrize("ratio", [16, 64])
@pytest.mark.parametrize("C", LAYERNORM_C)
def test_layernorm_offset_bound(ops, C, ratio):
    rows = 999
    x = _offset_input(rows, C, ratio, seed=3, per="row")
    gamma = (1 + 0.1 * torch.randn(C, device="cuda")).half()
    beta = (0.1 * torch.randn(C, device="cuda")).half()
    got = ops.layernorm(x, gamma, beta, eps=1e-5)
    torch.cuda.synchronize()
    x64 = x.to(F64)
    mean = x64.mean(1, keepdim=True)
    rstd = 1.0 / torch.sqrt(((x64 - mean) ** 2).mean(1, keepdim=True) + 1e-5)
    y, b = _norm_bound(x64, mean, rstd, gamma.to(F64), beta.to(F64))
    check_bound(got, y, b, f"layernorm<{layernorm_instance(C)}> C{C} |mean|/std {ratio}", "layernorm")
