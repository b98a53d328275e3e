"""tap-GEMM epilogue instances: every instance compiled for one epilogue kind, and the generic one, at each tile width it runs
with, held to the per-element bounds of tests/test_kernel_bounds_gpu.py (GPU); the instance list restated in
tools/gemm_roofline.py against the library source, the case table against every (instance, tile width) cell, and the epilogue
kinds one UNet forward issues against the specialised instances (CPU)."""
import os
import re

import pytest
import torch

from tests.test_kernel_bounds_gpu import BF16, _g, _rnd, check_bound, plan, run_gemm_case
from tools import gemm_roofline as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXTRA_EPI = {"bias": "bias", "res": "residual", "rowvec": "rowvec", "cs": "colscale"}


def case_instance(case):
    epi = tuple(EXTRA_EPI[e] for e in case.extras.split(",") if e in EXTRA_EPI)
    return R.epi_instance(case.flags, epi)


def _widths(id, op, extras, flags=0, **d):
    """one case per tile width: N = 1150 -> 128, 300 -> 160, 1000 -> 256 (GEGLU: N = 300 -> 128, 1000 -> 256)"""
    ns = {128: 300, 256: 1000} if flags & 1 else {128: 1150, 160: 300, 256: 1000}
    return [_g(f"{id}-bn{bn}", op, extras, flags, bn=bn, N=n, **d) for bn, n in ns.items()]


L = dict(rows=300, K=320)
EPI_CASES = (
    _widths("none", "linear", "", **L)
    + _widths("bias", "linear", "bias", **L)
    + _widths("bias-res", "linear", "bias,res", **L)
    + _widths("bias-rowvec", "linear", "bias,rowvec", rv_div=7, **L)
    + _widths("geglu", "linear", "bias", 1, **L)
    + _widths("silu", "linear", "bias", 2, **L)
    + _widths("erf", "linear", "bias", 4, **L)
    + _widths("tanh", "linear_ex", "bias", 8, **L)
    + _widths("colscale-res", "linear_ex", "bias,cs,res", **L)
    # the generic instance: kinds with no instance of their own
    + _widths("generic-res", "linear", "res", **L)
    + _widths("generic-rowvec-res-silu", "linear", "bias,rowvec,res", 2, rv_div=7, **L)
    + _widths("generic-geglu-nobias", "linear", "", 1, **L)
    # specialised instances with ragged rows and tails, several tiles per CTA, odd N, scalar store / load paths
    + [_g("bias-res-ragged-multi", "linear", "bias,res", rows=20000 + 37, K=136, N=300, bn=160),
       _g("geglu-multi-K64", "linear", "bias", 1, rows=9000 + 5, K=64, N=1000, bn=256),
       _g("colscale-res-oddldres", "linear_ex", "bias,cs,res,oddldres", rows=301, K=320, N=1150, bn=128),
       _g("bias-res-outoff", "linear", "bias,res,outoff", rows=63, K=320, N=1000, bn=256),
       _g("silu-N127", "linear", "bias", 2, rows=65, K=64, N=127, bn=128),
       _g("conv-bias-rowvec", "conv2d_3x3", "bias,rowvec", BT=3, H=5, W=9, Cin=64, Cout=320, rv_div=45, bn=160),
       _g("conv-bias-res", "conv2d_3x3", "bias,res", BT=3, H=5, W=9, Cin=64, Cout=1000, bn=256),
       _g("t3-bias-res", "conv_t3", "bias,res", B=2, T=5, HW=50, Cin=64, Cout=1150, bn=128),
       _g("c3d-bias", "conv3d_causal", "bias", T=2, H=4, W=5, Cin=24, Cout=300, bn=160),
       # the bf16 library, the way the CogVideoX DiT calls it
       _g("bf16-colscale-res", "linear_ex", "bias,cs,res", rows=300, K=320, N=640, bn=160, dtype=BF16),
       _g("bf16-gelu-tanh", "linear_ex", "bias", 8, rows=300, K=320, N=1000, bn=256, dtype=BF16),
       _g("bf16-bias", "linear", "bias", rows=300, K=320, N=1150, bn=128, dtype=BF16)]
)


def library_instances():
    """TG_EPI_KINDS of tapgemm.cuh, evaluated with the TapGemmEpi values"""
    src = open(os.path.join(ROOT, "star_b200", "csrc", "tapgemm.cuh")).read()
    vals = {m.group(1): int(m.group(2)) for m in re.finditer(r"(TG_EPI_\w+) = (\d+),", src)}
    body = re.search(r"#define TG_EPI_KINDS\(X\)(.*?)\n\n", src, re.S).group(1)
    kinds = []
    for expr in re.findall(r"X\(([^()]*)\)", body):
        k = 0
        for term in expr.split("|"):
            term = term.strip()
            k |= vals[term] if term in vals else int(term)
        kinds.append(k)
    return kinds


def test_epilogue_instances_restate_the_library():
    kinds = library_instances()
    assert kinds[-1] == R.EPI_GENERIC and tuple(kinds[:-1]) == R.EPI_INSTANCES
    src = open(os.path.join(ROOT, "star_b200", "csrc", "tapgemm.cuh")).read()
    for name, bit in R.EPI_BITS.items():
        assert re.search(rf"TG_EPI_{name[:3].upper()}\w* = {bit},", src), name


def test_epilogue_case_table_covers_every_instance():
    cells = set()
    for case in EPI_CASES:
        pl = plan(case)
        assert pl.bn == case.bn, f"{case.id}: the tile-width rule picks {pl.bn}, the case expects {case.bn}"
        k = case_instance(case)
        cells.add((k, pl.bn))
        if k == R.EPI_GENERIC and case.flags & 1:
            cells.add((k, "geglu"))
    want = {(k, bn) for k in R.EPI_INSTANCES + (R.EPI_GENERIC,) for bn in (128, 160, 256) if not (k & 2 and bn == 160)}
    want.add((R.EPI_GENERIC, "geglu"))
    missing = want - cells
    assert not missing, f"epilogue instances without a case: {sorted(map(str, missing))}"


def test_unet_forward_runs_only_specialised_epilogues(monkeypatch):
    """Every tap-GEMM call of a (reduced) UNet + ControlNet forward, host graph on the emulated kernels, maps to an epilogue
    instance of its own kind, not to the generic one.  The reduced model has every block type of the full one."""
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
                    calls.append(R.shape_of_call(_n, _f, a, k))
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
    kinds = {R.epi_kind(s.flags, s.epi) for s in calls}
    assert {"linear", "conv2d_3x3", "conv2d_3x3_s2", "conv_t3"} <= {s.op for s in calls}
    assert {1, 1 | 2, 1 | 16, 1 | 4} <= kinds                     # bias, GEGLU, residual, time-embedding rowvec
    generic = sorted({R.label(s) for s in calls if R.epi_instance(s.flags, s.epi) == R.EPI_GENERIC})
    assert not generic, f"UNet calls on the generic epilogue: {generic}"


@pytest.fixture(scope="module")
def ops():
    from star_b200 import ops as O
    return O


@pytest.mark.gpu
@pytest.mark.parametrize("case", EPI_CASES, ids=[c.id for c in EPI_CASES])
def test_epilogue_instance_bound(ops, case):
    got, y, bound, locate, untouched = run_gemm_case(ops, case)
    pl = plan(case)
    check_bound(got, y, bound, f"{case.id} (epilogue {case_instance(case)}, BN {pl.bn}, {pl.tiles} tiles)",
                "tapgemm-epi" + ("-bf16" if case.dtype == BF16 else ""), locate)
    assert untouched(), f"{case.id}: wrote outside the output view"


@pytest.mark.gpu
@pytest.mark.parametrize("N", [1150, 300, 1000], ids=["bn128", "bn160", "bn256"])
@pytest.mark.parametrize("op", ["linear", "linear_ex"])
def test_specialised_residual_in_place(ops, op, N):
    """out is residual: each thread stores only elements whose residual it has read (bias+res and colscale+res instances)"""
    rows, K = 4500, 320
    a, w = _rnd((rows, K), 1), _rnd((N, K), 2, K ** -0.5)
    bias, cs, res = _rnd((N,), 3, 0.1), _rnd((N,), 4), _rnd((rows, N), 5)
    call = (lambda r, out=None: ops.linear(a, w, bias, r, out=out)) if op == "linear" else \
        (lambda r, out=None: ops.linear_ex(a, w, bias, cs, r, out=out))
    want = call(res)
    buf = res.clone()
    call(buf, out=buf)
    torch.cuda.synchronize()
    assert torch.equal(buf.view(torch.int16), want.view(torch.int16))
