"""tap-GEMM staged epilogue: a call whose output and residual TMA can address stores each tile through shared-memory slabs
with TMA (residual slabs loaded with TMA), every other call stores straight from registers.  Both paths apply the same fp32
operations per element, so their outputs must be identical byte for byte (GPU): per epilogue kind and tile width, at
ragged rows and N, several tiles per CTA, conv boxes of fewer than 128 rows, the 32-column tail slab of the 160-wide tile,
in place, and a band of rows written into a larger row space.  The path is chosen from the views alone: the same data one
element further into the allocation takes the direct path.  On the CPU: every tap-GEMM call of a UNet + ControlNet forward
meets the staged path's alignment rule."""
import pytest
import torch

from tests.test_kernel_bounds_gpu import BF16, HALF, _g, _rnd
from tools import gemm_roofline as R

SENTINEL = -1024.0


def _ld(n):
    """a row pitch TMA can address, wider than the view"""
    return (n + 7) // 8 * 8 + 8


def _buf(rows, n, ld, off, dt, seed=None):
    flat = _rnd((off + rows * ld,), seed, dtype=dt) if seed is not None else \
        torch.full((off + rows * ld,), SENTINEL, dtype=dt, device="cuda")
    return flat, flat[off:].view(rows, ld)[:, :n]


def _inputs(case):
    d, dt, ex = case.d, case.dtype, case.extras
    on, box, taps, K, N, rows_in = R.geometry(case.op, d)
    wrows = 2 * N if case.flags & 1 else N
    rows = rows_in if case.op in ("linear", "linear_ex") else None
    if case.op in ("linear", "linear_ex"):
        x, w = _rnd((rows, K), 1, dtype=dt), _rnd((wrows, K), 2, K ** -0.5, dt)
    elif case.op == "conv2d_3x3":
        x, w = _rnd((d["BT"], d["H"], d["W"], K), 1, dtype=dt), _rnd((N, 3, 3, K), 2, (9 * K) ** -0.5, dt)
    elif case.op == "conv_t3":
        x, w = _rnd((rows_in, K), 1, dtype=dt), _rnd((N, 3, K), 2, (3 * K) ** -0.5, dt)
    else:
        x, w = _rnd((rows_in, K), 1, dtype=dt), _rnd((N, 3, 3, 3, K), 2, (27 * K) ** -0.5, dt)
    out_rows = rows_in if case.op in ("linear", "linear_ex", "conv_t3") else on[0] * on[1] * on[2] * on[3]
    bias = _rnd((wrows,), 3, 0.1, dt) if "bias" in ex else None
    cs = _rnd((N,), 4, dtype=dt) if "cs" in ex else None
    res = _buf(out_rows, N, _ld(N), 0, dt, seed=5)[1] if "res" in ex else None
    rv = _rnd((-(-out_rows // d["rv_div"]), N), 6, dtype=dt) if "rowvec" in ex else None
    return x, w, bias, cs, res, rv, out_rows, N


def _call(O, case, x, w, bias, cs, res, rv, out):
    d = case.d
    if case.op == "linear":
        O.linear(x, w, bias, res, rv, d.get("rv_div", 1), case.flags, out=out)
    elif case.op == "linear_ex":
        O.linear_ex(x, w, bias, cs, res, case.flags, out=out)
    elif case.op == "conv2d_3x3":
        O.conv2d_3x3(x, w, bias, rv, d.get("rv_div", 1), res, out=out)
    elif case.op == "conv_t3":
        band = d.get("band")
        if band is not None:
            p0, p1 = band
            x = x.view(d["B"], d["T"], d["HW"], -1)[:, :, p0:p1].contiguous().view(-1, x.shape[1])
        O.conv_t3(x, w, bias, res, d["B"], d["T"], d["HW"], out=out, band=band)
    else:
        O.conv3d_causal(x, w, d["T"], d["H"], d["W"], bias, res, out=out)


def _widths(id, op, extras, flags=0, **d):
    """one case per tile width, N a multiple of 8 with a partial last tile: N = 1144 -> 128, 296 -> 160 (its last tile ends
    in 8 columns of the 32-column tail slab), 1000 -> 256 (GEGLU: N = 296 -> 128, 1000 -> 256)"""
    ns = {128: 296, 256: 1000} if flags & 1 else {128: 1144, 160: 296, 256: 1000}
    return [_g(f"{id}-bn{bn}", op, extras, flags, bn=bn, N=n, **d) for bn, n in ns.items()]


L = dict(rows=300, K=320)
CASES = (
    _widths("none", "linear", "", **L)
    + _widths("bias", "linear", "bias", **L)
    + _widths("bias-res", "linear", "bias,res", **L)
    + _widths("bias-rowvec", "linear", "bias,rowvec", rv_div=7, **L)
    + _widths("geglu", "linear", "bias", 1, **L)
    + _widths("silu", "linear", "bias", 2, **L)
    + _widths("erf", "linear", "bias", 4, **L)
    + _widths("tanh", "linear_ex", "bias", 8, **L)
    + _widths("colscale-res", "linear_ex", "bias,cs,res", **L)
    + _widths("generic-res", "linear", "res", **L)
    + _widths("generic-rowvec-res-silu", "linear", "bias,rowvec,res", 2, rv_div=7, **L)
    + _widths("generic-geglu-nobias", "linear", "", 1, **L)
    + [_g("res-ragged-multi", "linear", "bias,res", rows=20000 + 37, K=136, N=296, bn=160),
       _g("res-N320-tail", "linear", "bias,res", rows=1000, K=320, N=320, bn=160),
       _g("res-N264-two-slab-tile", "linear", "bias,res", rows=1000, K=64, N=264, bn=160),
       _g("res-N1000-multi", "linear", "bias,res", rows=30000 + 11, K=320, N=1000, bn=256),
       _g("geglu-multi-K64", "linear", "bias", 1, rows=9000 + 5, K=64, N=1000, bn=256),
       _g("silu-N120", "linear", "bias", 2, rows=65, K=64, N=120, bn=128),
       # N % 8 != 0: both views take the direct epilogue, and nothing past N is written
       _g("silu-N127-direct", "linear", "bias", 2, rows=65, K=64, N=127, bn=128),
       _g("cs-res-N300-direct", "linear_ex", "bias,cs,res", rows=300, K=320, N=300, bn=160),
       _g("conv-long-ring-res", "conv2d_3x3", "bias,res", BT=2, H=20, W=36, Cin=320, Cout=320, bn=160),
       _g("conv-box90-rowvec", "conv2d_3x3", "bias,rowvec", BT=3, H=5, W=9, Cin=64, Cout=320, rv_div=45, bn=160),
       _g("t3-box100-res", "conv_t3", "bias,res", B=2, T=5, HW=50, Cin=64, Cout=1144, bn=128),
       _g("t3-band-res", "conv_t3", "bias,res", B=2, T=5, HW=50, band=(9, 37), Cin=64, Cout=296, bn=160),
       _g("c3d-bias", "conv3d_causal", "bias", T=2, H=4, W=5, Cin=24, Cout=296, bn=160),
       _g("bf16-colscale-res", "linear_ex", "bias,cs,res", rows=300, K=320, N=640, bn=160, dtype=BF16),
       _g("bf16-gelu-tanh", "linear_ex", "bias", 8, rows=300, K=320, N=1000, bn=256, dtype=BF16),
       _g("bf16-bias", "linear", "bias", rows=300, K=320, N=1144, bn=128, dtype=BF16)]
)


def _run(O, case, off, in_place=False):
    """the output of one call into a view `off` elements into a sentinel-filled allocation (in place: holding the residual);
    (view, whether everything outside it kept its value)"""
    x, w, bias, cs, res, rv, rows, N = _inputs(case)
    ld = _ld(N)
    flat, out = _buf(rows, N, ld, off, case.dtype)
    if in_place:
        out.copy_(res)
        res = out
    before = flat.clone()
    _call(O, case, x, w, bias, cs, res, rv, out)
    torch.cuda.synchronize()
    mask = torch.ones_like(flat, dtype=torch.bool)
    band = case.d.get("band")
    if band is None:
        mask[off:].view(rows, ld)[:, :N] = False
    else:                                                # only the band's pixels of every frame are written
        mask[off:].view(case.d["B"] * case.d["T"], case.d["HW"], ld)[:, band[0]:band[1], :N] = False
    return out.clone(), torch.equal(flat[mask], before[mask])


def _written(case, t):
    """the rows of an output a call writes: all, or the band's pixels of every frame"""
    band = case.d.get("band")
    if band is None:
        return t
    return t.reshape(case.d["B"] * case.d["T"], case.d["HW"], t.shape[1])[:, band[0]:band[1]]


@pytest.fixture(scope="module")
def ops():
    from star_b200 import ops as O
    return O


def test_case_table_covers_the_slab_walks():
    """every tile width and both GEGLU widths, the 160-wide tile's 32-column tail, a tile with fewer slabs than the width
    has, several tiles per CTA, conv boxes under 128 rows and a band write"""
    from tests.test_kernel_bounds_gpu import plan
    cells = set()
    for c in CASES:
        pl = plan(c)
        N = R.geometry(c.op, c.d)[4]
        assert pl.bn == c.bn, c.id
        cells.add(("geglu" if c.flags & 1 else "plain", pl.bn))
        last = N - (pl.n_tiles - 1) * pl.npt                  # columns of the last tile column
        if -(-last // 64) < -(-pl.npt // 64):
            cells.add(("short last tile", pl.bn))
        if pl.bn == 160 and last > 128:
            cells.add("tail slab")
        if pl.tiles > 132:
            cells.add(("multi-tile", pl.bn))
        if pl.box[0] * pl.box[1] * pl.box[2] * pl.box[3] < 128:
            cells.add(("box < 128", c.op))
        if "band" in c.d:
            cells.add("band")
        if c.dtype == BF16:
            cells.add("bf16")
    want = {("plain", 128), ("plain", 160), ("plain", 256), ("geglu", 128), ("geglu", 256), "tail slab", "band", "bf16",
            ("short last tile", 160), ("multi-tile", 160), ("multi-tile", 256), ("box < 128", "conv2d_3x3"),
            ("box < 128", "conv_t3")}
    assert want <= cells, sorted(map(str, want - cells))


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c.id for c in CASES])
def test_staged_matches_direct(ops, case):
    staged, ok_s = _run(ops, case, 0)
    direct, ok_d = _run(ops, case, 1)
    assert ok_s and ok_d, f"{case.id}: wrote outside the output view"
    assert torch.equal(staged.view(torch.int16), direct.view(torch.int16)), f"{case.id}: staged and direct outputs differ"
    assert case.dtype != HALF or not (staged == SENTINEL).all()


@pytest.mark.gpu
@pytest.mark.parametrize("case", [c for c in CASES if "res" in c.extras], ids=[c.id for c in CASES if "res" in c.extras])
def test_staged_in_place(ops, case):
    """out is residual: each slab's residual is loaded before its output is stored over it"""
    staged, ok = _run(ops, case, 0, in_place=True)
    direct, _ = _run(ops, case, 1)
    assert ok
    assert torch.equal(_written(case, staged).view(torch.int16), _written(case, direct).view(torch.int16))


def test_unet_forward_takes_the_staged_epilogue(monkeypatch):
    """Every tap-GEMM call of a (reduced) UNet + ControlNet forward, host graph on the emulated kernels, has an output and
    residual view TMA can address, so none falls back to the direct epilogue.  The model's last conv (4 latent channels) is
    the one exception: its 8-byte output rows are not a whole number of 16-byte units."""
    from oracle import kernel_ref as KR
    from star_b200 import ops
    from star_b200.video_to_video.modules.unet_v2v import ControlledV2VUNet
    from star_b200.utils.synth import synth_state_dict
    from tests.util import SMALL_KW, make_inputs
    calls = []
    for name in dir(KR):
        if not name.startswith("_") and callable(getattr(KR, name)) and hasattr(ops, name):
            fn = getattr(KR, name)
            if name in R.GEMM_OPS:
                def rec(*a, _n=name, _f=fn, **k):
                    calls.append((R.shape_of_call(_n, _f, a, k), R.call_epilogue_views(_n, _f, a, k)))
                    return _f(*a, **k)
                monkeypatch.setattr(ops, name, rec)
            else:
                monkeypatch.setattr(ops, name, fn)
    with torch.device("meta"):
        net = ControlledV2VUNet(**SMALL_KW)
    net.load_state_dict(synth_state_dict({k: tuple(v.shape) for k, v in net.state_dict().items()}, seed=1), assign=True)
    net = net.half().eval()
    x, hint, y = make_inputs(0, 1, 2, 10, 16)
    net(x, torch.tensor([500]), y, hint=hint)
    # The emulated kernels may return transposed results, which the GPU wrappers refuse and the GPU ops never produce;
    # such calls are left out.
    seen = [(s, v) for s, v in calls if v is not None]
    assert len(seen) > 0.9 * len(calls) and any(res is not None for _, (_, _, res) in seen)
    direct = sorted({R.label(s) for s, (n, out, res) in seen if not R.staged_epilogue(n, *out, *(res or (None, None)))})
    assert direct == ["c3x3 2x10x16 320->4 bias"], f"UNet calls on the direct epilogue: {direct}"
