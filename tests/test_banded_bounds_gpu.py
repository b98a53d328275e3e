"""Per-element fp64 bounds for the call forms the temporal-VAE decode uses beyond whole tensors: row bands of the 3x3 conv,
pixel bands of the (3,1,1) temporal conv, residual-in-place epilogues, banded GroupNorm applies, the SpatialNorm3D gather
geometry, and tensors whose element offsets pass 2^31 and 2^32.

The checker, the error model and the helpers are those of tests/test_kernel_bounds_gpu.py; no bound here adds a constant.
  - conv2d_3x3(rows=(row0, n)): the fp64 conv of the whole frame, sliced to the band's rows, at the top (zero-padded halo),
    bottom and interior, n = 1 / under one box / over several boxes, several frames per tile, every tile width with a partial
    last column tile, bias / residual / rowvec (ldrowvec > N), out a row slice of a larger allocation on both epilogue paths
    (the direct one forced by moving the views one element into their allocations).  Everything outside the view keeps its
    sentinel.
  - conv_t3(band=(p0, p1)): the fp64 whole-clip temporal conv restricted to the band's pixels, p0 = 0, p1 = HW, bands under
    128 pixels (several frames per tile), T = 1, B > 1; out-of-place and residual-is-out (the VAE's in-place call), whose
    bound is the out-of-place one on the residual's original values.
  - groupnorm(bands=): every band torch.equal to those rows of the whole-clip apply (same statistics, same arithmetic); the
    whole-clip apply held to _norm_bound; C > 2048 refused before any launch.
  - groupnorm_mod: the gather built with F.interpolate(mode="nearest") on the latent tables with the first-frame split of
    cp_enc_dec.py's SpatialNorm3D, not with the kernel's index formula.
  - offsets past 2^31 / 2^32 elements: one test per kernel of the 1080p -> 4x window, checked on sampled rows (the first rows,
    the rows straddling the 2^31 and 2^32 element offsets, the last rows), each within about 12 GiB of device memory.

CPU: test_case_table_covers_the_band_forms requires a case for every cell above; test_checkers_catch_band_faults shows how
each checker catches a halo row from the neighbouring band, a residual read after its store, a gather from latent frame
ts + 1 and one element written at its offset mod 2^32.  Passing cases print their worst |err| / bound (pytest -s); the
large-offset tests print their runtime and peak device memory.
"""
import math
import time
from collections import namedtuple

import pytest
import torch
import torch.nn.functional as F

from tests.test_kernel_bounds_gpu import (BF16, F64, HALF, WORST, BoundCheck, U32, _contract, _finish, _g, _group_stats,
                                          _norm_bound, _offset_input, _rnd, check_bound, plan, tap_epilogue, tile_locator)
from tests.test_rowops_bounds_gpu import VAE_HEAD_ROUND, adain_ref, check_adain_u8
from tools import gemm_roofline as R

GiB = 2 ** 30
SENTINEL = -1024.0                  # exact in fp16 and bf16
MARKS = (2 ** 31, 2 ** 32)          # element offsets where a 32-bit index wraps (signed, unsigned)
LARGE_CAP = 12 * GiB                # device memory one large-offset test may hold


def _ld(n):
    """a row pitch wider than the view that TMA can address (n a multiple of 8)"""
    return n + 8


def _f64(t):
    return None if t is None else t.to(F64)


# ---- 1. conv2d_3x3(rows=) ------------------------------------------------------------------------------------------------
# extras: bias, res (a separate residual), inplace (residual is out), rowvec (a column slice: ldrowvec > N)
CONV_ROWS_CASES = [
    _g("top-n1-multiframe", "conv2d_3x3", "bias", BT=2, H=9, W=40, Cin=64, Cout=296, rows=(0, 1), bn=160),
    _g("bottom-n5-res", "conv2d_3x3", "bias,res", BT=2, H=20, W=36, Cin=64, Cout=1144, rows=(15, 5), bn=128),
    _g("interior-n3-multiframe-rowvec", "conv2d_3x3", "bias,rowvec,res", BT=5, H=12, W=10, Cin=72, Cout=1000, rows=(4, 3),
       rv_div=7, bn=256),
    _g("interior-W130-several-boxes", "conv2d_3x3", "bias,res", BT=1, H=40, W=130, Cin=64, Cout=296, rows=(7, 20), bn=160),
    _g("interior-under-one-box", "conv2d_3x3", "bias", BT=3, H=30, W=24, Cin=64, Cout=1144, rows=(11, 4), bn=128),
    _g("bottom-n1-inplace", "conv2d_3x3", "bias,inplace", BT=2, H=7, W=50, Cin=64, Cout=1000, rows=(6, 1), bn=256),
    _g("interior-inplace-rowvec", "conv2d_3x3", "bias,rowvec,inplace", BT=2, H=16, W=24, Cin=128, Cout=296, rows=(5, 6),
       rv_div=24, bn=160),
    _g("whole-height-rows", "conv2d_3x3", "bias,res", BT=2, H=6, W=20, Cin=64, Cout=1144, rows=(0, 6), bn=128),
    _g("bf16-interior-res", "conv2d_3x3", "bias,res", BT=2, H=14, W=36, Cin=128, Cout=296, rows=(3, 8), bn=160, dtype=BF16),
    _g("bf16-top-inplace", "conv2d_3x3", "bias,inplace", BT=3, H=10, W=16, Cin=64, Cout=1000, rows=(0, 2), bn=256, dtype=BF16),
]

# ---- 2. conv_t3(band=) ---------------------------------------------------------------------------------------------------
CONV_T3_BAND_CASES = [
    _g("t3-p0-0", "conv_t3", "bias", B=1, T=5, HW=300, band=(0, 200), Cin=64, Cout=296, bn=160),
    _g("t3-p1-HW-res", "conv_t3", "bias,res", B=2, T=3, HW=300, band=(170, 300), Cin=64, Cout=1144, bn=128),
    _g("t3-band50-multiframe-res", "conv_t3", "bias,res", B=2, T=7, HW=500, band=(211, 261), Cin=72, Cout=1000, bn=256),
    _g("t3-T1-res", "conv_t3", "bias,res", B=3, T=1, HW=200, band=(50, 150), Cin=64, Cout=296, bn=160),
    _g("t3-band1-inplace", "conv_t3", "bias,inplace", B=2, T=4, HW=90, band=(89, 90), Cin=64, Cout=296, bn=160),
    _g("t3-interior-inplace", "conv_t3", "bias,inplace", B=2, T=5, HW=700, band=(128, 400), Cin=128, Cout=1144, bn=128),
    _g("t3-whole-inplace", "conv_t3", "bias,inplace", B=2, T=3, HW=100, band=(0, 100), Cin=64, Cout=1000, bn=256),
    _g("t3-T1-inplace", "conv_t3", "bias,inplace", B=2, T=1, HW=300, band=(20, 70), Cin=64, Cout=1000, bn=256),
    _g("bf16-t3-band-inplace", "conv_t3", "bias,inplace", B=2, T=3, HW=260, band=(30, 90), Cin=64, Cout=296, bn=160,
       dtype=BF16),
    _g("bf16-t3-p0-res", "conv_t3", "bias,res", B=1, T=4, HW=200, band=(0, 120), Cin=128, Cout=1144, bn=128, dtype=BF16),
]

PATHS = ["staged", "direct"]


def _k16(case):
    return plan(case).k16


def _out_buffer(rows, N, off, dt, pre=0, post=1):
    """[rows, N] view with row pitch _ld(N) that starts `pre` rows and `off` elements into a sentinel-filled allocation"""
    ld = _ld(N)
    flat = torch.full((off + (pre + rows + post) * ld,), SENTINEL, dtype=dt, device="cuda")
    return flat, flat[off:].view(pre + rows + post, ld)[pre:pre + rows, :N]


def _rows_mask(flat, off, pre, rows, N, ld, sel=None):
    """bool mask of flat: True at the elements of view rows `sel` (all rows when None)"""
    mask = torch.zeros_like(flat, dtype=torch.bool)
    grid = mask[off:].view(-1, ld)[pre:pre + rows, :N]
    if sel is None:
        grid[:] = True
    else:
        grid[sel] = True
    return mask


def run_conv_rows_case(O, case, path):
    """launch one conv2d_3x3(rows=) case; returns (got, fp64 value, bound, locator, ok outside the written rows)"""
    d, dt, ex = case.d, case.dtype, case.extras
    on, box, taps, K, N, _ = R.geometry("conv2d_3x3", d)
    BT, H, W = d["BT"], d["H"], d["W"]
    row0, n = d["rows"]
    rows = BT * n * W
    off = 0 if path == "staged" else 1
    pre = 3
    x = _rnd((BT, H, W, K), 1, dtype=dt)
    w = _rnd((N, 3, 3, K), 2, (9 * K) ** -0.5, dt)
    bias = _rnd((N,), 3, 0.1, dt) if "bias" in ex else None
    flat, out = _out_buffer(rows, N, off, dt, pre=pre)
    res = resv = None
    if "inplace" in ex:
        resv = _rnd((rows, N), 5, dtype=dt)
        out.copy_(resv)
        res = out
    elif "res" in ex:
        _, res = _out_buffer(rows, N, off, dt, pre=1)
        res.copy_(_rnd((rows, N), 5, dtype=dt))
        resv = res.clone()
    rv = rv_idx = None
    div = d.get("rv_div", 1)
    if "rowvec" in ex:
        rv = _rnd((-(-rows // div), N + 40), 6, dtype=dt)[:, 8:8 + N]
        rv_idx = torch.arange(rows, device="cuda") // div
    ld = _ld(N)
    staged = R.staged_epilogue(N, (pre * ld + off) * 2, ld, None if res is None else (ld + off) * 2 if res is not out else
                               (pre * ld + off) * 2, None if res is None else ld)
    assert staged == (path == "staged"), f"{case.id}: the views take the {'staged' if staged else 'direct'} epilogue"
    O.conv2d_3x3(x, w, bias, rv, div, res, out=out, rows=(row0, n))
    torch.cuda.synchronize()

    x64, w64 = x.to(F64), w.to(F64)
    band = lambda t: t.view(BT, H, W, N)[:, row0:row0 + n].reshape(-1, N)         # noqa: E731
    acc, mag = band(_contract("conv2d_3x3", d, x64, w64)), band(_contract("conv2d_3x3", d, x64.abs(), w64.abs()))
    y, bound = tap_epilogue(acc, mag, _k16(case), dt, _f64(bias), rowvec=None if rv is None else rv.to(F64)[rv_idx],
                            residual=_f64(resv))
    mask = _rows_mask(flat, off, pre, rows, N, ld)
    ok = bool((flat[~mask] == SENTINEL).all())
    loc = tile_locator(plan(case))
    return out, y, bound, lambda r, c: f"[frame {r // (n * W)}, image row {row0 + r // W % n}] {loc(r, c)}", ok


@pytest.fixture(scope="module")
def ops():
    from star_b200 import ops as O
    torch.cuda.reset_peak_memory_stats()
    yield O
    worst = {k: round(v, 3) for k, v in sorted(WORST.items()) if k != "selftest"}      # selftest: the CPU fault injections
    print(f"[bounds] worst |err|/bound per family: {worst}; "
          f"peak device memory {torch.cuda.max_memory_allocated() / GiB:.2f} GiB")


def _family(base, dt):
    return base + ("-bf16" if dt == BF16 else "")


@pytest.mark.gpu
@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("case", CONV_ROWS_CASES, ids=[c.id for c in CONV_ROWS_CASES])
def test_conv2d_3x3_rows_bound(ops, case, path):
    got, y, bound, locate, ok = run_conv_rows_case(ops, case, path)
    pl = plan(case)
    check_bound(got, y, bound, f"{case.id} {path} (rows {case.d['rows']}, box {pl.box}, {pl.tiles} tiles)",
                _family("conv-rows", case.dtype), locate)
    assert ok, f"{case.id} {path}: wrote outside the band's output rows"


def run_conv_t3_band_case(O, case, path):
    d, dt, ex = case.d, case.dtype, case.extras
    on, box, taps, K, N, _ = R.geometry("conv_t3", d)
    B, T, HW = d["B"], d["T"], d["HW"]
    p0, p1 = d["band"]
    rows = B * T * HW
    off = 0 if path == "staged" else 1
    ld = _ld(N)
    xf = _rnd((rows, K), 1, dtype=dt)
    xb = xf.view(B, T, HW, K)[:, :, p0:p1].contiguous().view(-1, K)
    w = _rnd((N, 3, K), 2, (3 * K) ** -0.5, dt)
    bias = _rnd((N,), 3, 0.1, dt) if "bias" in ex else None
    flat, out = _out_buffer(rows, N, off, dt)
    res = resv = None
    if "inplace" in ex:
        resv = _rnd((rows, N), 5, dtype=dt)
        out.copy_(resv)
        res = out
    elif "res" in ex:
        _, res = _out_buffer(rows, N, off, dt)
        res.copy_(_rnd((rows, N), 5, dtype=dt))
        resv = res.clone()
    before = flat.clone()
    staged = R.staged_epilogue(N, (off + p0 * ld) * 2, ld, None if res is None else (off + p0 * ld) * 2,
                               None if res is None else ld)
    assert staged == (path == "staged"), f"{case.id}: the views take the {'staged' if staged else 'direct'} epilogue"
    O.conv_t3(xb, w, bias, res, B, T, HW, out=out, band=(p0, p1))
    torch.cuda.synchronize()

    idx = (torch.arange(B * T, device="cuda")[:, None] * HW + torch.arange(p0, p1, device="cuda")[None, :]).reshape(-1)
    dd = dict(B=B, T=T, HW=HW)
    x64, w64 = xf.to(F64), w.to(F64)
    acc, mag = _contract("conv_t3", dd, x64, w64)[idx], _contract("conv_t3", dd, x64.abs(), w64.abs())[idx]
    y, bound = tap_epilogue(acc, mag, _k16(case), dt, _f64(bias), residual=None if resv is None else resv.to(F64)[idx])
    mask = _rows_mask(flat, off, 0, rows, N, ld, idx)
    ok = torch.equal(flat[~mask], before[~mask])
    bw = p1 - p0
    return out[idx], y, bound, lambda r, c: f"[clip {r // (T * bw)}, frame {r // bw % T}, pixel {p0 + r % bw}]", ok


@pytest.mark.gpu
@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("case", CONV_T3_BAND_CASES, ids=[c.id for c in CONV_T3_BAND_CASES])
def test_conv_t3_band_bound(ops, case, path):
    got, y, bound, locate, ok = run_conv_t3_band_case(ops, case, path)
    pl = plan(case)
    check_bound(got, y, bound, f"{case.id} {path} (band {case.d['band']}, box {pl.box}, {pl.tiles} tiles)",
                _family("conv-t3-band", case.dtype), locate)
    assert ok, f"{case.id} {path}: wrote outside the band's pixels (or changed an out-of-band residual row)"


# ---- 3. groupnorm(bands=) ------------------------------------------------------------------------------------------------
GN_BAND_CASES = [  # nsamples, frames per sample, pixels per frame, C, band, silu, dtype
    (2, 3, 200, 128, 70, 1, HALF),
    (1, 4, 150, 256, 1, 0, HALF),
    (3, 2, 99, 512, 40, 1, HALF),
    (1, 5, 129, 512, 128, 0, HALF),
    (2, 3, 200, 256, 64, 1, BF16),
    (1, 2, 77, 128, 1, 0, BF16),
]


@pytest.mark.gpu
@pytest.mark.parametrize("ns,T,HW,C,band,silu,dtype", GN_BAND_CASES)
def test_groupnorm_bands_bound(ops, ns, T, HW, C, band, silu, dtype):
    rows = ns * T * HW
    x = _offset_input(rows, C, 16, seed=11, dtype=dtype)
    gamma = (1 + 0.1 * torch.randn(C, device="cuda")).to(dtype)
    beta = (0.1 * torch.randn(C, device="cuda")).to(dtype)
    whole = ops.groupnorm(x, gamma, beta, ns, 1e-5, bool(silu))
    frames = torch.arange(ns * T, device="cuda")[:, None] * HW
    nb = 0
    for (p0, p1), g in ops.groupnorm(x, gamma, beta, ns, 1e-5, bool(silu), bands=(HW, band)):
        assert p0 == nb * band and p1 == min(HW, p0 + band)
        want = whole[(frames + torch.arange(p0, p1, device="cuda")[None, :]).reshape(-1)]
        assert torch.equal(g.view(torch.int16), want.view(torch.int16)), f"band ({p0}, {p1}) differs from the whole-clip apply"
        nb += 1
    assert nb == -(-HW // band)
    torch.cuda.synchronize()
    mean, rstd = _group_stats(x, ns, C, 1e-5)
    rps = T * HW
    chk = BoundCheck(f"groupnorm ns{ns} T{T} HW{HW} C{C} band {band} silu{silu} {dtype}", _family("groupnorm-bands", dtype),
                     lambda r, c: f"[sample {r // rps}, frame {r // HW % T}, pixel {r % HW}, group {c // (C // 32)}]")
    for s in range(ns):
        sl = slice(s * rps, (s + 1) * rps)
        y, b = _norm_bound(x[sl].to(F64), mean[s], rstd[s], gamma.to(F64), beta.to(F64), silu=bool(silu), dtype=dtype)
        chk.add(whole[sl], y, b, row0=s * rps)
    chk.done()


@pytest.mark.gpu
def test_groupnorm_bands_refuses_C_above_2048(ops):
    from star_b200.lib import StarError
    C = 2560
    x = _rnd((2 * 100, C), 1)
    gamma, beta = torch.ones(C, dtype=HALF, device="cuda"), torch.zeros(C, dtype=HALF, device="cuda")
    torch.cuda.synchronize()
    n0 = ops.launch_count()
    with pytest.raises(StarError, match="C > 2048"):
        for _ in ops.groupnorm(x, gamma, beta, 1, 1e-5, True, bands=(100, 30)):
            pass
    assert ops.launch_count() == n0, "the refused banded call launched a kernel"


# ---- 4. groupnorm_mod: the SpatialNorm3D gather --------------------------------------------------------------------------
GnMod = namedtuple("GnMod", "id T H W Tl Hl Wl C")
GN_MOD_CASES = [
    GnMod("cogvideox-T13-r1", 13, 6, 10, 13, 6, 10, 512),
    GnMod("cogvideox-T25-r2", 25, 8, 12, 13, 4, 6, 512),
    GnMod("cogvideox-T49-r4", 49, 16, 8, 13, 4, 2, 256),
    GnMod("cogvideox-T49-r8", 49, 16, 16, 13, 2, 2, 128),
    GnMod("even-T8-no-split", 8, 6, 6, 4, 3, 3, 256),
    GnMod("even-T12-Tl3-no-split", 12, 8, 4, 3, 2, 1, 128),
    GnMod("T-equals-Tl-even", 6, 4, 8, 6, 4, 8, 512),
    GnMod("T1", 1, 16, 16, 1, 2, 2, 256),
    GnMod("ratio3-division", 5, 9, 12, 3, 3, 4, 256),
    GnMod("W1-advance-crosses-frames", 9, 8, 1, 3, 2, 1, 128),
    GnMod("W3-advance-crosses-rows", 7, 4, 3, 4, 2, 3, 256),
    GnMod("ratio41-spatial", 5, 82, 2, 3, 2, 1, 128),
    GnMod("ratio41-temporal-split", 83, 2, 2, 3, 1, 1, 256),
    GnMod("ratio47-temporal-no-split", 94, 1, 3, 2, 1, 3, 128),
]


def gn_mod_split(T):
    """the reference interpolates the first frame alone when T is odd and > 1"""
    return T > 1 and T % 2 == 1


def gn_mod_spatial_path(c):
    """gn_apply_mod_kernel: shifts when H / Hl and W / Wl are powers of two, else the fp32-scale nearest index"""
    pow2 = lambda q: q & (q - 1) == 0                                             # noqa: E731
    return "shift" if pow2(c.H // c.Hl) and pow2(c.W // c.Wl) else "division"


def spatial_norm_gather(tab, T, H, W, Tl, Hl, Wl, shift_frame=None):
    """[Tl*Hl*Wl, C] latent table -> [T*H*W, C] as cp_enc_dec.py's SpatialNorm3D interpolates zq (mode "nearest", the first
    frame alone when T is odd and > 1).  The decoder's zq is bf16 / fp16, whose nearest index uses the fp32 scale n_in / n_out;
    PyTorch's fp64 CPU kernels compute some ranks with an fp64 scale instead (they differ at ratio 41), so the rows are chosen by
    interpolating an fp32 table of latent row numbers (exact below 2^24) and tab is gathered with them.
    shift_frame: simulate a fault that reads latent frame ts + 1 for that output frame."""
    z = torch.arange(Tl * Hl * Wl, dtype=torch.float32).view(1, 1, Tl, Hl, Wl)
    if gn_mod_split(T):
        z = torch.cat([F.interpolate(z[:, :, :1], size=(1, H, W), mode="nearest"),
                       F.interpolate(z[:, :, 1:], size=(T - 1, H, W), mode="nearest")], dim=2)
    else:
        z = F.interpolate(z, size=(T, H, W), mode="nearest")
    src = z.reshape(T, H * W).long().to(tab.device)
    if shift_frame is not None:
        src[shift_frame] = (src[shift_frame] + Hl * Wl).clamp(max=Tl * Hl * Wl - 1)
    return tab[src.reshape(-1)]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [HALF, BF16], ids=["fp16", "bf16"])
@pytest.mark.parametrize("case", GN_MOD_CASES, ids=[c.id for c in GN_MOD_CASES])
def test_groupnorm_mod_geometry_bound(ops, case, dtype):
    T, H, W, Tl, Hl, Wl, C = case.T, case.H, case.W, case.Tl, case.Hl, case.Wl, case.C
    rows = T * H * W
    x = _offset_input(rows, C, 16, seed=12, dtype=dtype)
    gamma = (1 + 0.1 * torch.randn(C, device="cuda")).to(dtype)
    beta = (0.1 * torch.randn(C, device="cuda")).to(dtype)
    mod = _rnd((Tl * Hl * Wl, 2 * C + 8), 13, dtype=dtype)             # column slices of one wider table: ldmod = 2C + 8
    ymod, bmod = mod[:, :C], mod[:, C:2 * C]
    got = ops.groupnorm_mod(x, gamma, beta, ymod, bmod, T, H, W, Tl, Hl, Wl, 1e-6, True)
    torch.cuda.synchronize()
    mean, rstd = _group_stats(x, 1, C, 1e-6)
    ym = spatial_norm_gather(ymod.to(F64), T, H, W, Tl, Hl, Wl)
    bm = spatial_norm_gather(bmod.to(F64), T, H, W, Tl, Hl, Wl)
    y, b = _norm_bound(x.to(F64), mean[0], rstd[0], gamma.to(F64), beta.to(F64), ym, bm, True, dtype=dtype)
    check_bound(got, y, b, f"groupnorm_mod {case.id} T{T} {H}x{W} <- {Tl}x{Hl}x{Wl} C{C} {dtype}",
                _family("groupnorm-mod", dtype), lambda r, c: f"[frame {r // (H * W)}, row {r // W % H}, col {r % W}]")


# ---- 5. offsets past 2^31 and 2^32 elements ------------------------------------------------------------------------------
def sample_rows(nrows, row_elems, marks=MARKS, k=2):
    """the first k rows, the rows around each element offset in marks (the row holding offset m - 1 and the one holding m, and
    their neighbours) and the last k rows of an [nrows, row_elems]-strided tensor"""
    rows = set(range(min(k, nrows))) | set(range(max(0, nrows - k), nrows))
    for m in marks:
        for r in ((m - 1) // row_elems - 1, (m - 1) // row_elems, m // row_elems, m // row_elems + 1):
            if 0 <= r < nrows:
                rows.add(r)
    return torch.tensor(sorted(rows), dtype=torch.long)


class LargeRun:
    """skips when the GPU has too little free memory, records runtime and peak device memory above what was allocated before,
    and frees everything the test allocated before the next one starts"""

    def __init__(self, what, need):
        self.what, self.need = what, need

    def __enter__(self):
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        free, _ = torch.cuda.mem_get_info()
        if free < self.need + GiB:
            msg = f"{self.what}: needs {self.need / GiB:.1f} GiB of device memory, {free / GiB:.1f} GiB free"
            print(f"[bounds] skip {msg}")
            pytest.skip(msg)
        self.base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        self.t0 = time.perf_counter()
        return self

    def __exit__(self, *exc):
        torch.cuda.synchronize()
        dt = time.perf_counter() - self.t0
        peak = torch.cuda.max_memory_allocated() - self.base
        print(f"[bounds] large {self.what}: {dt:.1f} s, peak device memory {peak / GiB:.2f} GiB")
        torch.cuda.empty_cache()
        assert exc[0] is not None or peak <= LARGE_CAP, f"{self.what}: peak {peak / GiB:.2f} GiB above the 12 GiB cap"
        return False


def _rnd_large(rows, cols, seed, step=1 << 20):
    """fp16 [rows, cols] of N(0, 1) values drawn a row chunk at a time: no fp32 copy of the whole tensor"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.empty(rows, cols, dtype=HALF, device="cuda")
    for r0 in range(0, rows, step):
        x[r0:r0 + step] = torch.randn(min(step, rows - r0), cols, generator=g, device="cuda")
    return x


def _assert_rows_equal(got, want, rows, what):
    if not torch.equal(got, want):
        bad = (got != want).any(1).nonzero()[:5].view(-1).tolist()
        raise AssertionError(f"{what}: sampled rows {[int(rows[i]) for i in bad]} differ from the exact result")


@pytest.mark.gpu
def test_groupnorm_past_2_32_elements(ops):
    """one 4368 x 7744 frame at 128 channels (4.33e9 elements): statistics, a band apply of every band, then the whole apply in
    place; sampled rows of both against fp64, and the bands torch.equal the whole apply"""
    C, rows, band = 128, 4368 * 7744, 1 << 21
    with LargeRun("groupnorm 4368x7744x128", rows * C * 2 + 3 * band * C * 2 + GiB):
        x = _offset_input(rows, C, 4, seed=21)
        gamma = (1 + 0.1 * torch.randn(C, device="cuda")).half()
        beta = (0.1 * torch.randn(C, device="cuda")).half()
        sel = sample_rows(rows, C).cuda()
        xs = x[sel].to(F64)
        mean, rstd = _group_stats(x, 1, C, 1e-5)
        got_band = torch.full((len(sel), C), SENTINEL, dtype=HALF, device="cuda")
        for (p0, p1), g in ops.groupnorm(x, gamma, beta, 1, 1e-5, True, bands=(rows, band)):
            inb = (sel >= p0) & (sel < p1)
            got_band[inb] = g[sel[inb] - p0]
            del g
        ops.groupnorm(x, gamma, beta, 1, 1e-5, True, out=x)
        got = x[sel]
        del x
        y, b = _norm_bound(xs, mean[0], rstd[0], gamma.to(F64), beta.to(F64), silu=True)
        BoundCheck("groupnorm whole apply, sampled rows of 4368x7744x128", "groupnorm-large").add(got, y, b, rows=sel).done()
        BoundCheck("groupnorm band apply, sampled rows", "groupnorm-large").add(got_band, y, b, rows=sel).done()
        _assert_rows_equal(got_band, got, sel, "band apply vs whole apply")


def _conv_rows_ref(x, w, hs):
    """fp64 3x3 conv (zero padding) of the image rows hs of x [1, H, W, K]: {h: ([W, N] value, [W, N] on absolute values)}"""
    H = x.shape[1]
    w64 = w.to(F64).permute(0, 3, 1, 2)
    out = {}
    for h in sorted(set(int(v) for v in hs)):
        strip = torch.zeros(1, 3, x.shape[2], x.shape[3], dtype=F64, device=x.device)
        for dr in range(3):
            if 0 <= h + dr - 1 < H:
                strip[0, dr] = x[0, h + dr - 1].to(F64)
        s = strip.permute(0, 3, 1, 2)
        f = lambda a, b: F.conv2d(a, b, padding=(0, 1))[0, :, 0].t()            # noqa: E731
        out[h] = (f(s, w64), f(s.abs(), w64.abs()))
    return out


@pytest.mark.gpu
def test_conv2d_3x3_rows_past_2_32_elements(ops):
    """the last band (4400 rows) of a 4500 x 7744 frame, Cin 8, written by conv2d_3x3(rows=) into a view 64 rows into an
    allocation: the view holds 4.36e9 elements"""
    H, W, K, N, row0, n, pre = 4500, 7744, 8, 128, 100, 4400, 64
    rows = n * W
    with LargeRun("conv2d_3x3 rows=(100, 4400) of 4500x7744, 128 channels out", (pre + rows) * N * 2 + H * W * K * 2 + GiB):
        x = _rnd_large(H * W, K, 1).view(1, H, W, K)
        w = _rnd((N, 3, 3, K), 2, (9 * K) ** -0.5)
        bias = _rnd((N,), 3, 0.1)
        flat = torch.full(((pre + rows) * N,), SENTINEL, dtype=HALF, device="cuda")
        out = flat.view(pre + rows, N)[pre:]
        ops.conv2d_3x3(x, w, bias, out=out, rows=(row0, n))
        torch.cuda.synchronize()
        sel = sample_rows(rows, N)
        got = out[sel.cuda()]
        assert (flat[:pre * N] == SENTINEL).all(), "wrote in front of the output view"
        del flat, out
        ref = _conv_rows_ref(x, w, (row0 + sel // W).tolist())
        acc = torch.stack([ref[row0 + int(r) // W][0][int(r) % W] for r in sel])
        mag = torch.stack([ref[row0 + int(r) // W][1][int(r) % W] for r in sel])
        case = _g("large", "conv2d_3x3", "bias", BT=1, H=H, W=W, Cin=K, Cout=N, rows=(row0, n))
        y, b = tap_epilogue(acc, mag, _k16(case), HALF, bias.to(F64))
        BoundCheck("conv2d_3x3 rows= sampled rows of a 4.36e9-element view", "conv-rows-large").add(got, y, b, rows=sel).done()


@pytest.mark.gpu
def test_conv_t3_band_past_2_31_elements(ops):
    """a 1000-pixel band at p0 = 17e6 of a 2-frame, 17.5e6-pixel clip at 128 channels, residual in place: p0 * C passes 2^31 and
    the second frame's band passes 2^32; every band row against fp64, the rows next to the band untouched"""
    B, T, HW, K, N, p0, p1 = 1, 2, 17_500_000, 64, 128, 17_000_000, 17_001_000
    rows = B * T * HW
    with LargeRun("conv_t3 band (17e6, 17e6 + 1000) of 2 x 17.5e6 pixels, in place", rows * N * 2 + GiB):
        out = torch.full((rows, N), SENTINEL, dtype=HALF, device="cuda")
        idx = (torch.arange(B * T, device="cuda")[:, None] * HW + torch.arange(p0, p1, device="cuda")[None, :]).reshape(-1)
        nb = (torch.arange(B * T, device="cuda")[:, None] * HW + torch.tensor([p0 - 1, p1], device="cuda")[None, :]).reshape(-1)
        resv = _rnd((len(idx), N), 5)
        out[idx] = resv
        xb = _rnd((B * T * (p1 - p0), K), 1)
        w = _rnd((N, 3, K), 2, (3 * K) ** -0.5)
        bias = _rnd((N,), 3, 0.1)
        assert p0 * N > MARKS[0] and (HW + p0) * N > MARKS[1]
        ops.conv_t3(xb, w, bias, out, B, T, HW, out=out, band=(p0, p1))
        torch.cuda.synchronize()
        got, around = out[idx], out[nb]
        del out
        dd = dict(B=B, T=T, HW=p1 - p0)
        x64, w64 = xb.to(F64), w.to(F64)
        case = _g("large", "conv_t3", "bias", B=B, T=T, HW=HW, band=(p0, p1), Cin=K, Cout=N)
        y, b = tap_epilogue(_contract("conv_t3", dd, x64, w64), _contract("conv_t3", dd, x64.abs(), w64.abs()), _k16(case), HALF,
                            bias.to(F64), residual=resv.to(F64))
        BoundCheck("conv_t3 band at p0 * C > 2^31, in place", "conv-t3-large").add(got, y, b, rows=idx.cpu()).done()
        assert (around == SENTINEL).all(), "wrote next to the band"


@pytest.mark.gpu
def test_upsample2x_past_2_32_elements(ops):
    """2184 x 3872 -> 4368 x 7744 at 128 channels (4.33e9 output elements); sampled output rows exact"""
    H, W, C = 2184, 3872, 128
    orows = 4 * H * W
    with LargeRun("upsample2x to 4368x7744x128", (orows + H * W) * C * 2 + GiB):
        x = _rnd_large(H * W, C, 1)
        out = torch.full((orows, C), SENTINEL, dtype=HALF, device="cuda")
        ops.upsample2x(x, 1, H, W, out=out)
        torch.cuda.synchronize()
        sel = sample_rows(orows, C)
        got = out[sel.cuda()]
        del out
        oh, ow = sel // (2 * W), sel % (2 * W)
        _assert_rows_equal(got, x[((oh // 2) * W + ow // 2).cuda()], sel, "upsample2x past 2^32 elements")


@pytest.mark.gpu
def test_vae_head_and_tokens_to_nchw5_past_2_32_elements(ops):
    """x [(b t hw), 128] of 2 frames of 4368 x 3900 (4.36e9 elements): vae_head on its first 3 columns and tokens_to_nchw5 of
    that column view, at sampled token rows"""
    B, T, H, W, ld = 1, 2, 4368, 3900, 128
    HW = H * W
    rows = B * T * HW
    with LargeRun("vae_head / tokens_to_nchw5 over 2 x 4368x3900 tokens, ld 128", rows * ld * 2 + 2 * rows * 3 * 2 + GiB):
        x = _rnd_large(rows, ld, 1)
        w27, b3 = _rnd((27,), 2, 0.3), _rnd((3,), 3, 0.1)
        head = ops.vae_head(x, w27, b3, B, T, H, W).view(B * T, 3, HW)
        nchw = ops.tokens_to_nchw5(x[:, :3], B, 3, T, H, W).view(B, 3, T, HW)
        torch.cuda.synchronize()
        sel = sample_rows(rows, ld)
        bt, hw = sel // HW, sel % HW
        t = bt % T
        got_head = head[bt.cuda(), :, hw.cuda()]
        got_tok = nchw[(bt // T).cuda(), :, t.cuda(), hw.cuda()]
        w = w27.to(F64).view(3, 3, 3)                                      # [co][ci][dt]
        y = b3.to(F64).expand(len(sel), 3).clone()
        mag = y.abs()
        for dt in range(3):
            tt = t + dt - 1
            ok = ((tt >= 0) & (tt < T)).cuda()
            src = (sel + (dt - 1) * HW).clamp(0, rows - 1).cuda()
            xs = x[src, :3].to(F64) * ok[:, None]
            y = y + xs @ w[:, :, dt].t()
            mag = mag + xs.abs() @ w[:, :, dt].abs().t()
        want_tok = x[sel.cuda(), :3]
        del x, head, nchw
        BoundCheck("vae_head, sampled tokens of a 4.36e9-element input", "vae-head-large").add(
            got_head, y, _finish(y, VAE_HEAD_ROUND * U32 * mag, HALF), rows=sel).done()
        _assert_rows_equal(got_tok, want_tok, sel, "tokens_to_nchw5 past 2^32 input elements")


@pytest.mark.gpu
def test_adain_color_fix_past_2_31_elements(ops):
    """350 frames of 1080 x 1920, 3 channels (2.18e9 elements), uint8 output; the frames whose video or output offsets straddle
    2^31, and the first and last, against the fp64 reference of those frames (statistics are per frame and channel)"""
    C, Fr, H, W, h, w = 3, 350, 1080, 1920, 135, 240
    HW = H * W
    need = C * Fr * HW * 4 + Fr * HW * C + Fr * C * h * w * 4 + GiB
    with LargeRun("adain_color_fix 350 x 1080x1920 x 3, uint8 out", need):
        g = torch.Generator(device="cuda").manual_seed(2)
        video = torch.randn(1, C, Fr, H, W, generator=g, device="cuda").mul_(0.8)
        src = torch.rand(Fr, C, h, w, generator=g, device="cuda").mul_(2).sub_(1)
        got8 = ops.adain_color_fix(video, src, uint8=True)
        torch.cuda.synchronize()
        f_out = MARKS[0] // (HW * C)                                   # output (f, hw, c): offset 2^31 in this frame
        f_vid = MARKS[0] // HW - (C - 1) * Fr                          # video (c, f, hw): channel 2's plane at offset 2^31
        assert Fr * HW * C > MARKS[0] and 0 < f_vid < f_out < Fr - 1
        for f in sorted({0, f_vid - 1, f_vid, f_out, f_out + 1, Fr - 1}):
            y, b = adain_ref(video[:, :, f:f + 1], src[f:f + 1])
            check_adain_u8(got8[f].view(-1, C), y, b, f"adain frame {f} of {Fr} x {H}x{W}")
        del video, got8


# ---- 6. CPU: the case table and the checkers -----------------------------------------------------------------------------
LARGE_KERNELS = {"groupnorm": test_groupnorm_past_2_32_elements, "conv2d_3x3 rows=": test_conv2d_3x3_rows_past_2_32_elements,
                 "conv_t3 band=": test_conv_t3_band_past_2_31_elements, "upsample2x": test_upsample2x_past_2_32_elements,
                 "vae_head / tokens_to_nchw5": test_vae_head_and_tokens_to_nchw5_past_2_32_elements,
                 "adain_color_fix": test_adain_color_fix_past_2_31_elements}


def test_case_table_covers_the_band_forms():
    cells = set()
    for case in CONV_ROWS_CASES:
        pl = plan(case)
        d = case.d
        row0, n = d["rows"]
        assert pl.bn == case.bn, f"{case.id}: the tile-width rule picks {pl.bn}, the case expects {case.bn}"
        assert pl.on[1] == n, f"{case.id}: geometry() ignores rows="
        cells.add(("conv rows", "top" if row0 == 0 else "bottom" if row0 + n == d["H"] else "interior"))
        per_frame = -(-pl.on[0] // pl.box[0]) * -(-pl.on[1] // pl.box[1])          # boxes over one frame's band
        cells.add(("conv rows", "n=1" if n == 1 else "one box" if per_frame == 1 else "several boxes"))
        if pl.box[2] > 1:
            cells.add(("conv rows", "several frames per tile"))
        cells.add(("conv rows", "bn", pl.bn, "partial" if d["Cout"] % pl.npt else "full"))
        for e in ("res", "rowvec", "inplace"):
            if e in case.extras:
                cells.add(("conv rows", e))
        if case.dtype == BF16:
            cells.add(("conv rows", "bf16"))
    for case in CONV_T3_BAND_CASES:
        pl = plan(case)
        d = case.d
        p0, p1 = d["band"]
        assert pl.bn == case.bn and pl.on[0] == p1 - p0, f"{case.id}: geometry() ignores band="
        cells.add(("t3 band", "p0=0" if p0 == 0 else "p1=HW" if p1 == d["HW"] else "interior"))
        if pl.box[1] > 1:
            cells.add(("t3 band", "several frames per tile"))
        if d["T"] == 1:
            cells.add(("t3 band", "T=1"))
        if d["B"] > 1:
            cells.add(("t3 band", "B>1"))
        if "inplace" in case.extras:
            cells.add(("t3 band", "inplace"))
        if case.dtype == BF16:
            cells.add(("t3 band", "bf16"))
    for path in PATHS:                                      # every case runs on both epilogue paths
        for op in ("conv rows", "t3 band"):
            cells.add(("inplace", op, path))
    for ns, T, HW, C, band, silu, dtype in GN_BAND_CASES:
        cells |= {("gn bands", "C", C), ("gn bands", "silu", silu)}
        if band == 1:
            cells.add(("gn bands", "band of 1 pixel"))
        if HW % band:
            cells.add(("gn bands", "band does not divide the frame"))
        if ns > 1:
            cells.add(("gn bands", "nsamples>1"))
        if dtype == BF16:
            cells.add(("gn bands", "bf16"))
    lanes = lambda c: 256 // (c // 8)                                             # noqa: E731  GN2_THREADS / (C / 8)
    for c in GN_MOD_CASES:
        cells.add(("gn mod", "split" if gn_mod_split(c.T) else "no split"))
        cells.add(("gn mod", gn_mod_spatial_path(c)))
        cells.add(("gn mod", "C", c.C))
        if c.T == c.Tl:
            cells.add(("gn mod", "T=Tl"))
        if c.T == 1:
            cells.add(("gn mod", "T=1"))
        if c.T % 2 == 0:
            cells.add(("gn mod", "even T"))
        if c.Tl == 13 and c.T in (13, 25, 49):
            cells.add(("gn mod", "cogvideox T", c.T))
        for ratio in {c.H // c.Hl, c.W // c.Wl}:
            cells.add(("gn mod", "ratio", ratio))
        if c.W < lanes(c.C):
            cells.add(("gn mod", "W < lanes"))
        if c.H * c.W < lanes(c.C):
            cells.add(("gn mod", "advance crosses frames"))
        if (c.T * c.H * c.W) % 128:
            cells.add(("gn mod", "rows % GN2_SLAB"))
    for name, fn in LARGE_KERNELS.items():
        if callable(fn):
            cells.add(("large", name))
    want = {("conv rows", p) for p in ("top", "bottom", "interior", "n=1", "one box", "several boxes",
                                        "several frames per tile", "res", "rowvec", "inplace", "bf16")}
    want |= {("conv rows", "bn", bn, "partial") for bn in (128, 160, 256)}
    want |= {("t3 band", p) for p in ("p0=0", "p1=HW", "interior", "several frames per tile", "T=1", "B>1", "inplace", "bf16")}
    want |= {("inplace", op, path) for op in ("conv rows", "t3 band") for path in PATHS}
    want |= {("gn bands", "C", c) for c in (128, 256, 512)} | {("gn bands", "silu", s) for s in (0, 1)}
    want |= {("gn bands", p) for p in ("band of 1 pixel", "band does not divide the frame", "nsamples>1", "bf16")}
    want |= {("gn mod", p) for p in ("split", "no split", "shift", "division", "T=Tl", "T=1", "even T", "W < lanes",
                                      "advance crosses frames", "rows % GN2_SLAB")}
    want |= {("gn mod", "cogvideox T", t) for t in (13, 25, 49)} | {("gn mod", "ratio", r) for r in (1, 2, 3, 4, 8)}
    want |= {("gn mod", "C", c) for c in (128, 256, 512)}
    want |= {("large", k) for k in ("groupnorm", "conv2d_3x3 rows=", "conv_t3 band=", "upsample2x", "vae_head / tokens_to_nchw5",
                                     "adain_color_fix")}
    missing = want - cells
    assert not missing, f"band / in-place / gather / large-offset cells without a case: {sorted(map(str, missing))}"
    # the in-place cases must run on both paths: PATHS parametrizes every conv case
    assert any("inplace" in c.extras for c in CONV_ROWS_CASES) and any("inplace" in c.extras for c in CONV_T3_BAND_CASES)


def test_checkers_catch_band_faults():
    """Simulated kernel outputs (the fp64 reference rounded to fp16) pass each checker; each injected fault fails it."""
    # a halo row taken from the neighbouring band: rows (4, 3) of a 12-row frame read image row 2 in place of row 3
    BT, H, W, K, N, row0, n = 2, 12, 10, 64, 296, 4, 3
    d = dict(BT=BT, H=H, W=W, Cin=K, Cout=N, rows=(row0, n))
    case = _g("cpu", "conv2d_3x3", "bias", **d)
    x = _rnd((BT, H, W, K), 1, device="cpu")
    w = _rnd((N, 3, 3, K), 2, (9 * K) ** -0.5, device="cpu")
    bias = _rnd((N,), 3, 0.1, device="cpu")
    band = lambda t: t.view(BT, H, W, N)[:, row0:row0 + n].reshape(-1, N)         # noqa: E731
    x64, w64 = x.double(), w.double()
    y, b = tap_epilogue(band(_contract("conv2d_3x3", d, x64, w64)), band(_contract("conv2d_3x3", d, x64.abs(), w64.abs())),
                        _k16(case), HALF, bias.double())
    check_bound(y.half(), y, b, "clean banded conv")
    xf = x64.clone()
    xf[:, row0 - 1] = x64[:, row0 - 2]
    yf, _ = tap_epilogue(band(_contract("conv2d_3x3", d, xf, w64)), band(_contract("conv2d_3x3", d, xf.abs(), w64.abs())),
                         _k16(case), HALF, bias.double())
    with pytest.raises(AssertionError):
        check_bound(yf.half(), y, b, "halo row from the neighbouring band")

    # a residual read after its store: one 64-column slab of the first tile adds the stored output instead of the residual
    res = _rnd((BT * n * W, N), 5, device="cpu").double()
    acc = band(_contract("conv2d_3x3", d, x64, w64))
    mag = band(_contract("conv2d_3x3", d, x64.abs(), w64.abs()))
    y, b = tap_epilogue(acc, mag, _k16(case), HALF, bias.double(), residual=res)
    check_bound(y.half(), y, b, "clean in-place residual")
    g = y.half()
    stored = g[:60, :64].double()
    g[:60, :64] = (y[:60, :64] - res[:60, :64] + stored).half()
    with pytest.raises(AssertionError):
        check_bound(g, y, b, "residual read after the store")

    # the SpatialNorm3D gather reading latent frame ts + 1 for one output frame
    T, Hh, Ww, Tl, Hl, Wl, C = 9, 4, 6, 3, 2, 3, 64
    xg = _rnd((T * Hh * Ww, C), 7, device="cpu").double()
    tab_y, tab_b = _rnd((Tl * Hl * Wl, C), 8, device="cpu").double(), _rnd((Tl * Hl * Wl, C), 9, device="cpu").double()
    gamma, beta = torch.ones(C, dtype=F64), torch.zeros(C, dtype=F64)
    mean, rstd = _group_stats(xg, 1, C, 1e-6)
    ym, bm = (spatial_norm_gather(t, T, Hh, Ww, Tl, Hl, Wl) for t in (tab_y, tab_b))
    y, b = _norm_bound(xg, mean[0], rstd[0], gamma, beta, ym, bm, True)
    check_bound(y.half(), y, b, "clean SpatialNorm3D gather")
    ymf, bmf = (spatial_norm_gather(t, T, Hh, Ww, Tl, Hl, Wl, shift_frame=3) for t in (tab_y, tab_b))
    yf, _ = _norm_bound(xg, mean[0], rstd[0], gamma, beta, ymf, bmf, True)
    with pytest.raises(AssertionError):
        check_bound(yf.half(), y, b, "gather from latent frame ts + 1")

    # one element written at its offset mod 2^32: modelled at a modulus of 2^12 on a [rows, 64] output whose rows are sampled
    # at 2^11 and 2^12 elements as the large tests sample them at 2^31 and 2^32
    rows, Cc, mod = 100, 64, 2 ** 12
    yv = (torch.randn(rows, Cc, generator=torch.Generator().manual_seed(3), dtype=F64) * 4)
    bv = _finish(yv, U32 * yv.abs(), HALF)
    sel = sample_rows(rows, Cc, marks=(mod // 2, mod))
    out = yv.half()
    check_bound(out[sel], yv[sel], bv[sel], "clean sampled rows")
    wrapped = out.clone().view(-1)
    o = mod + 5                                               # the first element past the mark lands at o mod 2^12
    wrapped[o % mod], wrapped[o] = wrapped[o], SENTINEL
    wrapped = wrapped.view(rows, Cc)
    assert (o // Cc) in sel.tolist() and (o % mod) // Cc in sel.tolist()
    with pytest.raises(AssertionError):
        check_bound(wrapped[sel], yv[sel], bv[sel], "one element written at its offset mod 2^32")


def test_spatial_norm_gather_is_f_interpolate():
    """spatial_norm_gather's tables against a direct per-row restatement of PyTorch's nearest rule, and the ratios whose fp32
    reciprocal rounds low, where exact integer division picks the next latent row"""
    def nearest(dst, n_out, n_in):                   # upsample_nearest: min(floor(dst * (float) n_in / n_out), n_in - 1)
        s = float(torch.tensor(n_in, dtype=torch.float32) / torch.tensor(n_out, dtype=torch.float32))
        return min(math.floor(float(torch.tensor(dst * s, dtype=torch.float32))), n_in - 1) if n_out != n_in else dst
    from oracle.kernel_ref import spatial_norm_src_index
    for c in GN_MOD_CASES:
        idx = torch.arange(c.Tl * c.Hl * c.Wl, dtype=F64).view(-1, 1)
        got = spatial_norm_gather(idx, c.T, c.H, c.W, c.Tl, c.Hl, c.Wl).view(c.T, c.H, c.W).long()
        assert torch.equal(got.reshape(-1), spatial_norm_src_index(c.T, c.H, c.W, c.Tl, c.Hl, c.Wl, "cpu")), \
            f"{c.id}: oracle/kernel_ref.py's emulated gather differs"
        ts = torch.tensor([(0 if t == 0 else 1 + nearest(t - 1, c.T - 1, c.Tl - 1)) if gn_mod_split(c.T) else
                           nearest(t, c.T, c.Tl) for t in range(c.T)])
        hs = torch.tensor([nearest(h, c.H, c.Hl) for h in range(c.H)])
        ws = torch.tensor([nearest(w, c.W, c.Wl) for w in range(c.W)])
        want = (ts[:, None, None] * c.Hl + hs[None, :, None]) * c.Wl + ws[None, None, :]
        assert torch.equal(got, want), f"{c.id}: first mismatch at {(got != want).nonzero()[0].tolist()}"
    c = next(c for c in GN_MOD_CASES if c.id == "ratio41-spatial")
    assert nearest(41, c.H, c.Hl) == 0 != 41 * c.Hl // c.H
