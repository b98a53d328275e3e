"""Temporal VAE at frame sizes past one CTA's shared memory: star_softmax_rows over a cluster of CTAs per row, the VAE's
mid-block attention at 234 576 tokens (a 720p -> 4x frame), whole decode / encode past 102 400 tokens against the fp32
oracle, and enhance_frames on a 720p -> 4x clip with tiled sampling.

The softmax bound is softmax_ref's of tests/test_rowops_bounds_gpu.py with the per-thread term count of one segment and one
more fp32 level in the sum: the n CTA partials are added in rank order.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from tests.test_kernel_bounds_gpu import BoundCheck, _finish, _rnd, U32, ERR_EX2
from tests.test_rowops_bounds_gpu import ERR_FDIV, WARP_TREE, BLOCK_TREE
from tests.util import assert_close, rel_l2

HALF, F64 = torch.float16, torch.float64
SEG_MAX = 102400                 # columns one CTA of star_softmax_rows stages in shared memory


def segment(cols, n):
    """columns per CTA: ceil(cols / n) rounded up to a multiple of 8"""
    return (-(-cols // n) + 7) // 8 * 8


def min_ctas(cols):
    return -(-cols // SEG_MAX)


def softmax_cluster_ref(s, cols, n):
    """fp64 softmax over the first cols columns of fp16 logits and its bound for n CTAs per row: exact max, __expf of the
    fp32 difference, a per-thread sum of ceil(seg / 256) terms, the warp and block trees, n partials, a fast reciprocal and
    the product"""
    x = s[:, :cols].to(F64)
    z = x - x.amax(1, keepdim=True)
    e = torch.exp(z)
    tot = e.sum(1, keepdim=True)
    p = e / tot
    term = ERR_EX2 + 3 * U32 * z.abs()
    levels = math.ceil(segment(cols, n) / 256) + WARP_TREE + BLOCK_TREE + n
    sum_rel = (e * term).sum(1, keepdim=True) / tot + U32 * levels
    return p, _finish(p, (term + sum_rel + ERR_FDIV + U32) * p, HALF)


ROW_KINDS = ["max in last column", "max in first column", "max before a segment boundary", "max after a segment boundary",
             "dominant logit", "constant", "random", "random"]


def softmax_rows_input(cols, n, seed):
    """one row per ROW_KINDS entry, ld > cols"""
    ld = (cols + 8) // 8 * 8 + 8
    s = _rnd((len(ROW_KINDS), ld), seed, 3.0)
    seg = segment(cols, n)
    s[0, cols - 1] = 20
    s[1, 0] = 20
    s[2, min(seg, cols) - 1] = 20
    s[3, min(seg, cols - 1)] = 20
    s[4, :cols] = (0.1 * s[4, :cols].float()).half()
    s[4, cols // 2] = 12
    s[5, :cols] = -3
    return s


def check_softmax_rows(ops, cols, n, seed=7):
    s = softmax_rows_input(cols, n, seed)
    p, b = softmax_cluster_ref(s, cols, n)
    got = ops.softmax_rows(s, cols, n)
    torch.cuda.synchronize()
    assert (got[:, cols:] == 0).all(), f"cols {cols} n {n}: columns cols..ld are not zeroed"
    BoundCheck(f"softmax_rows {s.shape[0]}x{cols} ld {s.shape[1]}, {n} CTAs per row", "softmax",
               lambda r, c: f"[{ROW_KINDS[r]}, segment {c // segment(cols, n)}]").add(got[:, :cols], p, b).done()


@pytest.fixture(scope="module")
def ops():
    from star_b200 import ops as O
    return O


LONG_COLS = [102401, 150000, 234576, 528528, 819200]


@pytest.mark.gpu
@pytest.mark.parametrize("n", ["fit", 8])
@pytest.mark.parametrize("cols", LONG_COLS)
def test_softmax_rows_cluster_bound(ops, cols, n):
    check_softmax_rows(ops, cols, min_ctas(cols) if n == "fit" else n)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [2, 4, 8])
@pytest.mark.parametrize("cols", [8, 3294, 26352])
def test_softmax_rows_cluster_short_rows_bound(ops, cols, n):
    """segments shorter than 8 columns, or empty (8 columns over 8 CTAs leaves 7 empty)"""
    check_softmax_rows(ops, cols, n)


@pytest.mark.gpu
@pytest.mark.parametrize("cols,n,match", [(1000, 0, "ctas_per_row"), (1000, 9, "ctas_per_row"),
                                          (8 * SEG_MAX + 1, 8, "do not fit in shared memory"),
                                          (2 * SEG_MAX + 1, 2, "do not fit in shared memory")])
def test_softmax_rows_cluster_refusals(ops, cols, n, match):
    from star_b200.lib import StarError
    s = torch.zeros(2, (cols + 7) // 8 * 8, dtype=HALF, device="cuda")
    n0 = ops.launch_count()
    with pytest.raises(StarError, match=match):
        ops.softmax_rows(s, cols, n)
    assert ops.launch_count() == n0, "the refused call launched a kernel"
    assert (s == 0).all()


@pytest.mark.gpu
def test_vae_attention_past_one_cta():
    """AutoencoderKLTemporalDecoder._attention at HW = 234 576 (one 2896x5184 frame's mid block, 3 CTAs per row), C = 512:
    512 query rows from the first, a middle and the last row block against an fp32 reference over all keys"""
    from star_b200.video_to_video.modules.temporal_vae import AutoencoderKLTemporalDecoder
    HW, C = 234576, 512
    g = torch.Generator(device="cuda").manual_seed(3)

    def rnd(*shape, scale=1.0):
        return (torch.randn(*shape, generator=g, device="cuda") * scale).half()

    s = C ** -0.5
    a = {"gn": (1 + rnd(C, scale=0.1), rnd(C, scale=0.1)),
         "q": (rnd(C, C, scale=3.0 * s * s), rnd(C, scale=0.1 * s)),          # logits of std ~3: peaked rows
         "k": (rnd(C, C, scale=s), rnd(C, scale=0.1)),
         "v": rnd(C, C, scale=s),
         "o": (rnd(C, C, scale=4 * s), rnd(C, scale=0.1))}
    x = rnd(HW, C)
    out = AutoencoderKLTemporalDecoder._attention(a, x, 1, HW)
    torch.cuda.synchronize()

    f = lambda t: t.float()                                                      # noqa: E731
    xn = F.group_norm(f(x).t().unsqueeze(0), 32, f(a["gn"][0]), f(a["gn"][1]), 1e-6)[0].t()
    k = xn @ f(a["k"][0]).t() + f(a["k"][1])
    v = xn @ f(a["v"]).t()
    # _attention's row blocks are 1 024 rows here: rows of the first block, of the middle one and the last 170 (the final
    # 80-row block and the end of the one before it)
    mid = HW // 2 // 1024 * 1024
    rows = torch.cat([torch.arange(0, 171), torch.arange(mid + 300, mid + 471), torch.arange(HW - 170, HW)]).cuda()
    q = xn[rows] @ f(a["q"][0]).t() + f(a["q"][1])
    attn = torch.softmax(q @ k.t(), dim=-1) @ v @ f(a["o"][0]).t() + f(a["o"][1])
    ref = f(x[rows]) + attn
    assert_close(out[rows], ref, rel=4e-3, what="VAE attention at 234 576 tokens")
    err = rel_l2(f(out[rows]) - f(x[rows]), attn)
    print(f"VAE attention at {HW} tokens: attention term rel-L2 {err:.3e}")
    assert err < 2e-2, f"attention term rel-L2 {err:.3e}"


def _blocked_sdpa(q, k, v, *a, **kw):
    """exact fp32 softmax(q k^T / sqrt(d)) v over blocks of query rows (plain matmuls: no fused kernel)"""
    out = torch.empty(q.shape[:-1] + (v.shape[-1],), dtype=q.dtype, device=q.device)
    scale = q.shape[-1] ** -0.5
    for r in range(0, q.shape[-2], 4096):
        s = torch.matmul(q[..., r:r + 4096, :], k.transpose(-1, -2)) * scale
        out[..., r:r + 4096, :] = torch.matmul(torch.softmax(s, dim=-1), v)
    return out


REDUCED = dict(block_out_channels=(32, 32, 64, 64), layers_per_block=2)


def _reduced_vae():
    from tests.test_vae import _setup
    cfg, sd, vae = _setup(REDUCED, device="cuda")
    return cfg, {k: v.cuda() for k, v in sd.items()}, vae


@pytest.mark.gpu
def test_decode_past_102400_tokens(monkeypatch):
    """one 3-frame window at a 330x330 latent (108 900 tokens per frame: 2 CTAs per softmax row) against the fp32 oracle"""
    from oracle.temporal_vae_ref import decode
    cfg, sdc, vae = _reduced_vae()
    z = torch.randn(3, 4, 330, 330, generator=torch.Generator().manual_seed(1)).cuda()
    got = vae.decode(z, num_frames=3).sample
    torch.cuda.synchronize()
    monkeypatch.setattr(F, "scaled_dot_product_attention", _blocked_sdpa)
    ref = decode(sdc, z, 3, cfg)
    err = rel_l2(got, ref)
    print(f"temporal VAE decode latent 330x330: rel-L2 vs fp32 oracle {err:.3e}")
    assert got.shape == (3, 3, 2640, 2640) and err < 4e-3


@pytest.mark.gpu
def test_encode_past_102400_tokens(monkeypatch):
    """one 2640x2640 frame (a 330x330 latent) against the fp32 oracle"""
    from oracle.temporal_vae_ref import encode_moments
    cfg, sdc, vae = _reduced_vae()
    x = (torch.rand(1, 3, 2640, 2640, generator=torch.Generator().manual_seed(2)) * 2 - 1).cuda()
    got = vae.encode(x).latent_dist.parameters
    torch.cuda.synchronize()
    monkeypatch.setattr(F, "scaled_dot_product_attention", _blocked_sdpa)
    ref = encode_moments(sdc, x, cfg)
    err = rel_l2(got, ref)
    print(f"temporal VAE encode 2640x2640: rel-L2 vs fp32 oracle {err:.3e}")
    assert got.shape == (1, 8, 330, 330) and err < 4e-3


@pytest.mark.gpu
def test_enhance_frames_720p_to_4x_tiled():
    """enhance_frames on an 8-frame 720x1280 clip to 2880x5120: full UNet and temporal VAE (synthetic weights), one solver
    step, tiles of 90x160 latent pixels"""
    from types import SimpleNamespace
    from bench import build_model
    from tools.tiled_bench import synth_vae
    from star_b200.video_to_video.video_to_video_model import VideoToVideo_sr
    dev = torch.device("cuda", 0)
    net, _, _ = build_model(False, dev)
    ny = torch.zeros(1, 77, 1024)
    pipe = VideoToVideo_sr(SimpleNamespace(model_path=None), device=dev, text_encoder=lambda s: ny, vae=synth_vae(dev),
                           generator=net)
    g = torch.Generator().manual_seed(5)
    video = torch.rand(8, 3, 720, 1280, generator=g) * 2 - 1
    y = torch.randn(1, 77, 1024, generator=g)
    torch.cuda.reset_peak_memory_stats(dev)
    frames = pipe.enhance_frames({"video_data": video, "y": y, "target_res": (2880, 5120)}, steps=1, solver_mode="normal",
                                 tile_size=(90, 160), tile_overlap=16)
    peak = torch.cuda.max_memory_allocated(dev)
    print(f"enhance_frames 720x1280 -> 2880x5120, 8 frames, 1 step, tiles 90x160/16: peak {peak / 2 ** 30:.1f} GiB")
    assert frames.shape == (8, 2880, 5120, 3) and frames.dtype == torch.uint8
    assert frames.float().std() > 0
