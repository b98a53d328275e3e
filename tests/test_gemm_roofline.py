"""tools/gemm_roofline.py: the shape enumeration and the byte / FLOP / fill arithmetic (CPU), and the tap-GEMM epilogue's
in-place residual (GPU): the epilogue issues residual loads ahead of the stores of earlier column pairs, which is only
correct because a thread stores to no element whose residual it has not read yet."""
import math

import pytest
import torch

from tests.test_kernel_bounds_gpu import _g, _rnd, plan
from tools import gemm_roofline as R


def test_roofline_restates_the_dispatch():
    cases = [_g("l0-to_out", "linear", rows=32 * 122 * 216, K=320, N=320, bn=160),
             _g("l1-conv", "conv2d_3x3", BT=32, H=62, W=108, Cin=640, Cout=640, bn=160),
             _g("t3", "conv_t3", B=2, T=5, HW=50, Cin=24, Cout=300, bn=160),
             _g("s2p", "conv2d_3x3_s2p", BT=2, H=9, W=11, Cin=8, Cout=64, pad=(0, 1, 0, 1), bn=128),
             _g("c3d", "conv3d_causal", T=5, H=3, W=9, Cin=72, Cout=1000, bn=256),
             _g("geglu", "linear", "bias", 1, rows=300, K=320, N=300, bn=128)]
    for case in cases:
        pl = plan(case)
        shape = R.Shape(case.op, tuple(sorted(case.d.items())), case.flags, ())
        m = R.model(shape)
        assert (m["bn"], m["tiles"], m["iters"]) == (case.bn, pl.tiles, pl.iters), case.id


def test_geometry_of_row_and_pixel_bands():
    """conv2d_3x3(rows=(row0, n)) boxes its n output rows (star_abi.cu: on[1] = H_out, conv_box(H_out, W, BT)); conv_t3(band=
    (p0, p1)) tiles p1 - p0 pixels, box[0] = min(128, band) and several frames per box under 128 (on[0] = band), and reads
    only the band's rows of the clip; hand-computed"""
    conv = dict(BT=2, H=13, W=24, Cin=64, Cout=64)
    assert R.geometry("conv2d_3x3", conv)[:2] == ((24, 13, 2, 1), (24, 5, 1, 1))
    assert R.geometry("conv2d_3x3", dict(conv, rows=(5, 2)))[:2] == ((24, 2, 2, 1), (24, 2, 2, 1))
    assert R.geometry("conv2d_3x3", dict(conv, BT=3, W=40, rows=(0, 1)))[:2] == ((40, 1, 3, 1), (40, 1, 3, 1))
    assert R.geometry("conv2d_3x3", dict(conv, BT=1, H=40, W=300, rows=(10, 4)))[:2] == ((300, 4, 1, 1), (64, 2, 1, 1))
    assert R.geometry("conv2d_3x3", dict(conv, rows=(5, 2)))[5] == 2 * 13 * 24             # the whole frame is read
    t3 = dict(B=2, T=5, HW=50, Cin=64, Cout=64)
    assert R.geometry("conv_t3", t3)[:2] == ((50, 5, 2, 1), (50, 2, 1, 1))
    assert R.geometry("conv_t3", dict(t3, band=(9, 37)))[::5] == ((28, 5, 2, 1), 2 * 5 * 50)   # the clip's rows
    assert R.band_input_rows("conv_t3", dict(t3, band=(9, 37))) == 2 * 5 * 28                 # read compactly
    assert R.band_input_rows("conv_t3", t3) == R.band_input_rows("conv2d_3x3", dict(conv, BT=1, H=10, W=50)) == 500
    assert R.geometry("conv_t3", dict(t3, band=(9, 37)))[1] == (28, 4, 1, 1)
    assert R.geometry("conv_t3", dict(t3, HW=500, T=3, band=(0, 300)))[:2] == ((300, 3, 2, 1), (128, 1, 1, 1))
    assert R.geometry("conv_t3", dict(t3, HW=90, T=3, band=(89, 90)))[:2] == ((1, 3, 2, 1), (1, 3, 1, 1))


def test_roofline_arithmetic():
    conv = R.Shape("conv2d_3x3", tuple(sorted(dict(BT=32, H=122, W=216, Cin=320, Cout=320).items())), 0, ("bias",))
    m = R.model(conv)
    box = R.geometry("conv2d_3x3", dict(conv.dims))[1]
    assert m["bn"] == 160 and m["iters"] == 45 and m["M"] == 32 * 122 * 216
    assert m["flops"] == 2.0 * m["M"] * 9 * 320 * 320
    assert m["hbm_bytes"] == 2.0 * (2 * m["M"] * 320 + 9 * 320 * 320 + 320)
    assert m["fill_bytes"] == m["tiles"] * 45 * (math.prod(box) * 128 + 160 * 128)
    # full 128 x 160 tiles need 57.6 B of operand fill per clock and SM at 2048 FMA per clock and SM, 128 x 256 tiles 48
    lin = lambda n: R.model(R.Shape("linear", (("K", 320), ("N", n), ("rows", 128 * 1000)), 0, ()))     # noqa: E731
    assert abs(lin(320)["fill_needed_b_clk_sm"] - 57.6) < 1e-9 and abs(lin(1280)["fill_needed_b_clk_sm"] - 48.0) < 1e-9
    to_out = R.model(R.Shape("linear", (("K", 320), ("N", 320), ("rows", 843264)), 0, ("bias", "residual")))
    assert to_out["bound"] == "HBM" and abs(to_out["hbm_floor_ms"] - 0.483) < 2e-3 and abs(to_out["mma_floor_ms"] - 0.175) < 2e-3
    ff_in = R.model(R.Shape("linear", (("K", 320), ("N", 1280), ("rows", 843264)), 1, ("bias",)))
    assert ff_in["bn"] == 256 and ff_in["geglu"] and ff_in["bound"] == "MMA" and ff_in["flops"] == 2.0 * 843264 * 320 * 2560


def test_roofline_shape_enumeration():
    from star_b200 import ops as O
    mt = lambda *s: torch.empty(*s, device="meta", dtype=torch.float16)                 # noqa: E731
    calls = [("linear", (mt(500, 320), mt(960, 320)), {}),
             ("linear", (mt(500, 320), mt(2560, 320), mt(2560)), {"flags": 1}),
             ("linear", (mt(500, 320), mt(320, 320), mt(320), mt(500, 320)), {"out": mt(500, 320)}),
             ("linear", (mt(500, 320), mt(320, 320), mt(320)), {"residual": mt(500, 320)}),
             ("conv2d_3x3", (mt(2, 10, 12, 64), mt(128, 3, 3, 64), mt(128)), {"rowvec": mt(2, 128), "rowvec_div": 120}),
             ("conv_t3", (mt(240, 64), mt(64, 3, 64), None, mt(240, 64), 1, 2, 120), {}),
             ("conv2d_3x3_s2", (mt(2, 10, 12, 64), mt(64, 3, 3, 64)), {}),
             ("groupnorm", (mt(500, 320),), {})]
    got = R.enumerate_calls(calls, O)
    assert sum(got.values()) == 7 and len(got) == 6                                     # residual by position or by keyword: one shape
    by = {R.label(s): (s, c) for s, c in got.items()}
    assert by["linear 500x320->320 bias+resi"][1] == 2
    s, _ = by["linear 500x320->1280 bias f1"]
    assert dict(s.dims)["N"] == 1280 and R.model(s)["geglu"]
    assert dict(by["c3x3 2x10x12 64->128 bias+rowv"][0].dims)["rv_div"] == 120
    s, _ = by["conv_t3 1x2x120 64->64 resi"]
    assert R.geometry(s.op, dict(s.dims))[:3] == ((120, 2, 1, 1), (120, 1, 1, 1), 3)
    s, _ = by["c3x3_s2 2x10x12 64->64"]
    assert R.geometry(s.op, dict(s.dims))[0] == (6, 6, 1, 2)


@pytest.mark.gpu
@pytest.mark.parametrize("rows,K,N,flags", [(4500, 320, 320, 0), (300, 64, 300, 2), (700, 320, 1000, 0), (700, 320, 320, 1)])
def test_residual_in_place_matches_out_of_place(rows, K, N, flags):
    from star_b200 import ops as O
    a, w = _rnd((rows, K), 1), _rnd((2 * N if flags & 1 else N, K), 2, K ** -0.5)
    bias, res = _rnd((w.shape[0],), 3, 0.1), _rnd((rows, N), 5)
    want = O.linear(a, w, bias, res, None, 1, flags)
    buf = res.clone()
    O.linear(a, w, bias, buf, None, 1, flags, out=buf)
    torch.cuda.synchronize()
    assert torch.equal(buf.view(torch.int16), want.view(torch.int16))
