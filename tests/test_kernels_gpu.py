"""GPU parity tests: every C-ABI entry point (include/star_sm100.h) against its
torch reference in oracle/kernel_ref.py on seeded inputs.  Tolerance: fp16
outputs, fp32 accumulation -> rel-L2 <= 2e-3, max-abs <= 2e-2 * max|ref|
(the north-star's 1e-3 relative fp16 bound is checked end to end on the UNet
output in test_unet_gpu.py; single kernels are held to the fp16 rounding of
their own output)."""
import pytest
import torch

from tests.util import assert_close

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def env():
    from oracle import kernel_ref as R
    from star_b200 import ops as O
    return O, R


def rnd(*shape, seed=0, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, generator=g, device="cuda") * scale).half()


@pytest.mark.parametrize("rows,K,N,flags,extras", [
    (128, 64, 128, 0, ""),
    (300, 320, 320, 0, "bias"),
    (4096, 1280, 1280, 0, "bias,res"),
    (1000, 320, 960, 0, ""),
    (777, 1024, 640, 0, "bias"),
    (513, 320, 4, 0, "bias"),
    (1, 320, 1280, 2, "bias"),
    (2000, 320, 1280, 1, "bias"),
    (640, 512, 2048, 1, "bias"),
    (900, 640, 640, 0, "bias,res,rowvec"),
    (1500, 2560, 320, 0, "bias"),
    (3000, 640, 1280, 0, "bias,res,rowvec"),      # N % 256 == 0: 128x256 tiles, two-pass epilogue, direct residual loads
    (129, 2560, 256, 0, "bias"),
    (5000, 512, 1536, 0, ""),
    (777, 1280, 3840, 2, "bias,res"),
    (1111, 640, 2560, 1, "bias"),                 # GEGLU on 128x256 tiles (128 outputs per tile)
    (600, 1280, 1920, 0, "bias"),                 # padded width 2048
    (900, 640, 960, 0, "bias,res"),
])
def test_linear(env, rows, K, N, flags, extras):
    O, R = env
    a = rnd(rows, K, seed=1)
    w = rnd(N * (2 if flags & 1 else 1), K, seed=2, scale=K ** -0.5)
    bias = rnd(w.shape[0], seed=3, scale=0.1) if "bias" in extras else None
    res = rnd(rows, N, seed=4) if "res" in extras else None
    rowvec = rnd((rows + 299) // 300, N, seed=5) if "rowvec" in extras else None
    got = O.linear(a, w, bias, res, rowvec, 300, flags)
    torch.cuda.synchronize()
    ref = R.linear(a, w, bias, res, rowvec, 300, flags)
    assert_close(got, ref, what=f"linear {rows}x{K}x{N} flags={flags} {extras}")


def test_linear_strided_views(env):
    O, R = env
    big = rnd(700, 960, seed=7)
    a = big[:, 320:640]                       # lda = 960
    w = rnd(320, 320, seed=8, scale=320 ** -0.5)
    outbuf = torch.zeros(700, 640, dtype=torch.half, device="cuda")
    O.linear(a, w, out=outbuf[:, 320:])
    torch.cuda.synchronize()
    assert_close(outbuf[:, 320:], R.linear(a, w), what="strided linear")
    assert (outbuf[:, :320] == 0).all()


@pytest.mark.parametrize("BT,H,W,Cin,Cout,extras", [
    (1, 8, 16, 64, 128, ""),
    (3, 18, 16, 320, 320, "bias"),
    (2, 10, 8, 640, 1280, "bias,rowvec"),
    (2, 17, 27, 320, 4, "bias"),
    (4, 3, 2, 1280, 1280, "bias,res"),
    (2, 34, 32, 960, 320, "bias,rowvec,res"),
    (2, 17, 27, 1280, 1280, "bias,rowvec,res"),
    (3, 33, 20, 128, 256, "bias,res"),
])
def test_conv2d_3x3(env, BT, H, W, Cin, Cout, extras):
    O, R = env
    x = rnd(BT, H, W, Cin, seed=1)
    w9 = rnd(Cout, 3, 3, Cin, seed=2, scale=(9 * Cin) ** -0.5)
    bias = rnd(Cout, seed=3, scale=0.1) if "bias" in extras else None
    rowvec = rnd(BT, Cout, seed=4) if "rowvec" in extras else None
    res = rnd(BT * H * W, Cout, seed=5) if "res" in extras else None
    got = O.conv2d_3x3(x, w9, bias, rowvec, H * W, res)
    torch.cuda.synchronize()
    ref = R.conv2d_3x3(x, w9, bias, rowvec, H * W, res)
    assert_close(got, ref, what=f"conv3x3 {BT}x{H}x{W} {Cin}->{Cout} {extras}")


def test_conv2d_rowvec_column_slice(env):
    """the time-embedding operand is a column slice of the one [B, sum Cout] embedding GEMM (row pitch != Cout)"""
    O, R = env
    x = rnd(4, 10, 8, 320, seed=1)                                   # 2 clips x 2 frames
    w9 = rnd(640, 3, 3, 320, seed=2, scale=(9 * 320) ** -0.5)
    temb_all = rnd(2, 320 + 640 + 1280, seed=3)
    rv = temb_all[:, 320:960]
    assert not rv.is_contiguous()
    got = O.conv2d_3x3(x, w9, None, rv, 2 * 80)
    assert_close(got, R.conv2d_3x3(x, w9, None, rv, 2 * 80), what="conv3x3 + strided rowvec")


@pytest.mark.parametrize("BT,H,W,C", [(2, 18, 16, 320), (3, 10, 8, 640), (1, 34, 32, 64), (2, 122, 216, 64)])
def test_conv2d_s2(env, BT, H, W, C):
    O, R = env
    x = rnd(BT, H, W, C, seed=1)
    w9 = rnd(C, 3, 3, C, seed=2, scale=(9 * C) ** -0.5)
    bias = rnd(C, seed=3, scale=0.1)
    got, Ho, Wo = O.conv2d_3x3_s2(x, w9, bias)
    torch.cuda.synchronize()
    ref, Hr, Wr = R.conv2d_3x3_s2(x, w9, bias)
    assert (Ho, Wo) == (Hr, Wr)
    assert_close(got, ref, what=f"conv s2 {BT}x{H}x{W}x{C}")


@pytest.mark.parametrize("B,T,HW,C", [(1, 8, 288, 320), (2, 5, 6, 640), (1, 40, 130, 64), (1, 3, 459, 1280)])
def test_conv_t3(env, B, T, HW, C):
    O, R = env
    x = rnd(B * T * HW, C, seed=1)
    w3 = rnd(C, 3, C, seed=2, scale=(3 * C) ** -0.5)
    bias = rnd(C, seed=3, scale=0.1)
    res = rnd(B * T * HW, C, seed=4)
    got = O.conv_t3(x, w3, bias, res, B, T, HW)
    torch.cuda.synchronize()
    assert_close(got, R.conv_t3(x, w3, bias, res, B, T, HW), what=f"conv_t3 {B},{T},{HW},{C}")


def test_conv_c4(env):
    O, R = env
    x = rnd(3, 18, 16, 4, seed=1)
    w9 = rnd(320, 3, 3, 4, seed=2, scale=1 / 6)
    bias = rnd(320, seed=3, scale=0.1)
    res = rnd(3 * 18 * 16, 320, seed=4)
    got = O.conv2d_3x3_c4(x, w9, bias, res)
    torch.cuda.synchronize()
    assert_close(got, R.conv2d_3x3_c4(x, w9, bias, res), what="conv c4")


@pytest.mark.parametrize("batch,heads,Nq,Nk,div", [
    (1, 1, 128, 128, 1),
    (2, 5, 288, 288, 1),
    (1, 2, 1000, 1000, 1),
    (8, 5, 288, 77, 4),
    (1, 2, 4096, 4096, 1),
    (2, 10, 72, 72, 1),
])
def test_attention(env, batch, heads, Nq, Nk, div):
    O, R = env
    C = heads * 64
    kvb = (batch + div - 1) // div
    if Nq == Nk and div == 1:                      # fused qkv buffer, like the spatial self-attention
        qkv = rnd(batch * Nq, 3 * C, seed=1)
        q, k, v = qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:]
    else:
        q = rnd(batch * Nq, C, seed=1)
        kv = rnd(kvb * Nk, 2 * C, seed=2)
        k, v = kv[:, :C], kv[:, C:]
    got = O.attention(q, k, v, batch, heads, Nq, Nk, div, 0.125)
    torch.cuda.synchronize()
    ref = R.attention(q, k, v, batch, heads, Nq, Nk, div, 0.125)
    assert_close(got, ref, what=f"attention b{batch} h{heads} {Nq}x{Nk}")


def test_attention_peaky(env):
    """large logits: exercises the running-max rescale path"""
    O, R = env
    q = rnd(1 * 640, 128, seed=1, scale=3.0)
    k = rnd(1 * 640, 128, seed=2, scale=3.0)
    v = rnd(1 * 640, 128, seed=3)
    got = O.attention(q, k, v, 1, 2, 640, 640, 1, 0.125)
    torch.cuda.synchronize()
    assert_close(got, R.attention(q, k, v, 1, 2, 640, 640, 1, 0.125), rel=4e-3, what="attention peaky")


@pytest.mark.parametrize("B,T,HW,heads,Ci", [(1, 8, 288, 5, 320), (1, 40, 50, 8, 512), (2, 32, 33, 10, 640), (1, 3, 7, 1, 64)])
def test_temporal_attention(env, B, T, HW, heads, Ci):
    O, R = env
    qkv = rnd(B * T * HW, 3 * Ci, seed=1)
    got = O.temporal_attention(qkv, B, T, HW, heads, Ci)
    torch.cuda.synchronize()
    assert_close(got, R.temporal_attention(qkv, B, T, HW, heads, Ci), what="temporal attention")


@pytest.mark.parametrize("ns,rps,C,silu", [(8, 288, 320, 1), (1, 8 * 288, 320, 1), (3, 100, 2560, 0), (2, 459, 1280, 1),
                                           (4, 77, 960, 1), (1, 26352, 640, 0), (32, 26352, 320, 1), (5, 129, 1920, 1),
                                           (3, 1, 128, 0), (7, 300, 64, 1)])
def test_groupnorm(env, ns, rps, C, silu):
    O, R = env
    x = rnd(ns * rps, C, seed=1) + 0.5
    gamma = (1 + 0.1 * torch.randn(C, device="cuda")).half()
    beta = (0.1 * torch.randn(C, device="cuda")).half()
    eps = 1e-5
    got = O.groupnorm(x, gamma, beta, ns, eps, silu)
    torch.cuda.synchronize()
    assert_close(got, R.groupnorm(x, gamma, beta, ns, eps, silu), what=f"groupnorm {ns},{rps},{C}")


@pytest.mark.parametrize("rows,C,mode", [(1000, 320, 0), (999, 512, 2), (300, 1280, 1), (64, 640, 2), (5, 320, 1), (1001, 320, 2),
                                         (3, 640, 0), (4097, 640, 1), (26353, 320, 1)])
def test_layernorm(env, rows, C, mode):
    O, R = env
    x = rnd(rows, C, seed=1)
    gamma = (1 + 0.1 * torch.randn(C, device="cuda")).half()
    beta = (0.1 * torch.randn(C, device="cuda")).half()
    gate = torch.rand(rows, device="cuda").half() if mode == 1 else None
    got = O.layernorm(x, gamma, beta, mode, gate, 0.3, -0.7)
    torch.cuda.synchronize()
    assert_close(got, R.layernorm(x, gamma, beta, mode, gate, 0.3, -0.7), what=f"layernorm {rows},{C},mode{mode}")


def test_liem_spatial_gate(env):
    O, R = env
    BT, H, W, C = 3, 18, 16, 320
    x = rnd(BT * H * W, C, seed=1)
    w98 = rnd(98, seed=2, scale=0.2)
    got = O.liem_spatial_gate(x, w98, BT, H, W)
    torch.cuda.synchronize()
    assert_close(got, R.liem_spatial_gate(x, w98, BT, H, W), what="liem gate")


def test_copies(env):
    O, R = env
    a, b, c = rnd(500, 320, seed=1), rnd(500, 640, seed=2), rnd(500, 640, seed=3)
    assert_close(O.concat_add(a, b, c), R.concat_add(a, b, c), what="concat_add")
    assert torch.equal(O.concat_add(a, b), R.concat_add(a, b))
    assert_close(O.add(b, c), R.add(b, c), what="add")
    x = rnd(2 * 9 * 4, 64, seed=4)
    assert torch.equal(O.upsample2x_crop(x, 2, 9, 4), R.upsample2x_crop(x, 2, 9, 4))
    x5 = torch.randn(2, 4, 3, 10, 8, device="cuda")
    tok = O.nchw5_to_tokens(x5)
    assert torch.equal(tok, R.nchw5_to_tokens(x5))
    back = O.tokens_to_nchw5(tok, 2, 4, 3, 10, 8)
    assert torch.equal(back, R.tokens_to_nchw5(tok, 2, 4, 3, 10, 8))
    t = torch.tensor([899, 34], device="cuda")
    assert_close(O.sinusoidal(t, 320), R.sinusoidal(t, 320), rel=2e-3, what="sinusoidal")
    assert_close(O.silu(a), R.silu(a), what="silu")


@pytest.mark.parametrize("shape,H,W,pad", [((4, 3, 24, 40), 96, 160, (560, 560, 312, 312)), ((2, 3, 240, 426), 960, 1704, (0, 24, 0, 16)),
                                          ((1, 3, 17, 9), 50, 31, (1, 2, 3, 0))])
def test_bilinear_pad(env, shape, H, W, pad):
    """F.interpolate(bilinear, align_corners=False) + F.pad(value=1): ref video_to_video_model.py:81-87"""
    O, R = env
    x = torch.rand(*shape, device="cuda") * 2 - 1
    got = O.bilinear_pad(x, H, W, pad, 1.0)
    ref = R.bilinear_pad(x, H, W, pad, 1.0)
    assert got.shape == ref.shape
    assert (got - ref).abs().max().item() <= 2e-6


@pytest.mark.parametrize("B,shape,rescale", [(1, (4, 32, 122, 216), 0.2), (2, (4, 5, 18, 16), 0.2), (1, (4, 3, 10, 8), None)])
def test_cfg_x0(env, B, shape, rescale):
    """CFG combine + std-ratio rescale + v -> x0 (diffusion_sdedit.py:89-99) against the reference's fp16 tensor ops"""
    O, R = env
    y = rnd(B, *shape, seed=1)
    u = (y.float() + 0.3 * torch.randn_like(y.float())).half()
    xt = torch.randn(B, *shape, device="cuda")
    al = torch.full((B, 1, 1, 1, 1), 0.6, device="cuda")
    sg = torch.full((B, 1, 1, 1, 1), 0.8, device="cuda")
    x0, guided = O.cfg_x0(y, u, xt, al, sg, 7.5, rescale, return_guided=True)
    x0r, gr = R.cfg_x0(y, u, xt, al, sg, 7.5, rescale, return_guided=True)
    # the std ratio is rounded to fp16 on both sides; a 1-ulp difference of that scalar moves every element by <= 2^-11
    assert_close(guided, gr, rel=1e-3, max_rel=2e-3, what="guided output")
    assert rel_l2_f(x0, x0r) <= 1e-3
    assert torch.equal(O.cfg_x0(y, u, xt, al, sg, 7.5, rescale), x0)


def test_adain_color_fix(env):
    """tensor2vid + adain_color_fix (inference_utils.py:16-23, color_fix.py:15-74) as three launches"""
    O, R = env
    video = (torch.randn(1, 3, 4, 96, 128, device="cuda") * 0.8).contiguous()
    src = torch.rand(4, 3, 24, 32, device="cuda") * 2 - 1
    got, ref = O.adain_color_fix(video, src), R.adain_color_fix(video, src)
    assert got.shape == ref.shape == (4, 96, 128, 3)
    assert (got - ref).abs().max().item() <= 2e-2                   # on a 0..255 scale
    g8, r8 = O.adain_color_fix(video, src, uint8=True), R.adain_color_fix(video, src, uint8=True)
    assert g8.dtype == torch.uint8 and (g8.int() - r8.int()).abs().max().item() <= 1


def rel_l2_f(a, b):
    return ((a.float() - b.float()).norm() / b.float().norm()).item()


# ---- CogVideoX DiT helpers -------------------------------------------------------------------------
@pytest.mark.parametrize("rows,K,N,flags,extras", [(322, 3072, 3072, 0, "bias,cs,res"), (700, 320, 1280, 8, "bias"),
                                                   (226, 1024, 640, 8, "bias,cs,res")])
def test_linear_ex(env, rows, K, N, flags, extras):
    O, R = env
    a = rnd(rows, K, seed=1)
    w = rnd(N, K, seed=2, scale=K ** -0.5)
    bias = rnd(N, seed=3, scale=0.1) if "bias" in extras else None
    cs = rnd(N, seed=4) if "cs" in extras else None
    res = rnd(rows, N, seed=5) if "res" in extras else None
    got = O.linear_ex(a, w, bias, cs, res, flags)
    torch.cuda.synchronize()
    assert_close(got, R.linear_ex(a, w, bias, cs, res, flags), what=f"linear_ex {rows}x{K}x{N} flags={flags} {extras}")


def test_layernorm_wide(env):
    O, R = env
    x = rnd(500, 3072, seed=1)
    g, b = (1 + 0.1 * torch.randn(3072, device="cuda")).half(), (0.1 * torch.randn(3072, device="cuda")).half()
    assert_close(O.layernorm(x, g, b), R.layernorm(x, g, b), what="layernorm C=3072")


def test_row_gate_and_qk_ln_rope(env):
    O, R = env
    x = rnd(333, 3072, seed=1)
    gate = torch.rand(333, device="cuda").half()
    assert_close(O.row_gate(x, 1, gate), R.row_gate(x, 1, gate), what="row_gate ext")
    assert_close(O.row_gate(x, 2, None, 0.4, -0.3), R.row_gate(x, 2, None, 0.4, -0.3), what="row_gate temporal")
    heads, seq, tl = 6, 50, 10
    qkv = rnd(2 * seq, 3 * heads * 64, seed=2)
    ref_in = qkv.clone()
    qg, qb, kg, kb = (rnd(64, seed=s, scale=0.5) + (1 if s % 2 == 0 else 0) for s in (10, 11, 12, 13))
    ang = torch.rand(seq - tl, 64, device="cuda") * 6.28
    cos, sin = ang.cos().contiguous(), ang.sin().contiguous()
    O.qk_ln_rope(qkv, heads, heads * 64, qg, qb, kg, kb, cos, sin, seq, tl, 1e-6)
    torch.cuda.synchronize()
    R.qk_ln_rope(ref_in, heads, heads * 64, qg, qb, kg, kb, cos, sin, seq, tl, 1e-6)
    assert_close(qkv, ref_in, what="qk_ln_rope")


# ---- temporal VAE helpers ---------------------------------------------------------------------------
@pytest.mark.parametrize("BT,H,W,C,pad", [(2, 16, 24, 128, (0, 1, 0, 1)), (1, 30, 20, 64, (0, 1, 0, 1)),
                                          (3, 9, 11, 256, (1, 1, 1, 1)), (1, 488, 864, 64, (0, 1, 0, 1))])
def test_conv2d_s2_padded(env, BT, H, W, C, pad):
    O, R = env
    x = rnd(BT, H, W, C, seed=1)
    w9 = rnd(C, 3, 3, C, seed=2, scale=(9 * C) ** -0.5)
    bias = rnd(C, seed=3, scale=0.1)
    got, Ho, Wo = O.conv2d_3x3_s2p(x, w9, bias, pad)
    torch.cuda.synchronize()
    ref, Hr, Wr = R.conv2d_3x3_s2p(x, w9, bias, pad)
    assert (Ho, Wo) == (Hr, Wr)
    assert_close(got, ref, what=f"conv s2p {BT}x{H}x{W}x{C} pad {pad}")


@pytest.mark.parametrize("rows,cols,ld", [(300, 1000, 1000), (77, 26352, 26352), (513, 123, 128), (9, 8, 8)])
def test_softmax_rows(env, rows, cols, ld):
    O, R = env
    s = rnd(rows, ld, seed=4, scale=3.0)
    ref = R.softmax_rows(s.clone(), cols)
    got = O.softmax_rows(s, cols)
    torch.cuda.synchronize()
    assert torch.equal(got[:, cols:], torch.zeros_like(got[:, cols:]))
    assert_close(got, ref, what=f"softmax_rows {rows}x{cols}")
    assert (got.float().sum(dim=1) - 1).abs().max() < 2e-2


def test_single_head_attention_as_gemms(env):
    """the VAE mid-block attention path: S = Q K^T (N = tokens, unaligned), row softmax, P V against V^T"""
    O, R = env
    HW, C = 26352 // 8, 512                                       # 3294 tokens: N % 32 != 0 -> direct-store GEMM
    xn = rnd(HW, C, seed=1)
    wq, wk, wv = (rnd(C, C, seed=s, scale=C ** -0.5) for s in (2, 3, 4))
    q, k = O.linear(xn, wq * (C ** -0.5)), O.linear(xn, wk)
    ld = (HW + 7) // 8 * 8
    S = torch.empty(HW, ld, device="cuda", dtype=torch.float16)
    vt = torch.zeros(C, ld, device="cuda", dtype=torch.float16)
    O.linear(wv, xn, out=vt[:, :HW])
    O.linear(q, k, out=S[:, :HW])
    O.softmax_rows(S, HW)
    o = O.linear(S, vt)
    torch.cuda.synchronize()
    qf, kf, vf = q.float(), k.float(), (xn.float() @ wv.float().t())
    ref = torch.softmax(qf @ kf.t(), dim=-1) @ vf
    assert_close(vt[:, :HW], vf.t().half(), what="V^T GEMM")
    assert_close(o, ref, rel=4e-3, what="single-head attention")


def test_vae_head_upsample_and_inplace_groupnorm(env):
    O, R = env
    B, T, H, W = 2, 3, 10, 12
    x = rnd(B * T * H * W, 8, seed=1)
    w27, b3 = rnd(27, seed=2, scale=0.3), rnd(3, seed=3, scale=0.1)
    assert_close(O.vae_head(x, w27, b3, B, T, H, W), R.vae_head(x, w27, b3, B, T, H, W), what="vae_head")
    assert_close(O.vae_head(x[: H * W * 2], w27, b3, 1, 2, H, W), R.vae_head(x[: H * W * 2], w27, b3, 1, 2, H, W), what="vae_head T=2")
    y = rnd(2 * 9 * 4, 128, seed=4)
    assert torch.equal(O.upsample2x(y, 2, 9, 4), R.upsample2x(y, 2, 9, 4))
    g = rnd(6 * 50, 128, seed=5)
    gamma, beta = rnd(128, seed=6), rnd(128, seed=7)
    ref = R.groupnorm(g, gamma, beta, 6, 1e-6, True)
    got = O.groupnorm(g, gamma, beta, 6, 1e-6, True, out=g)
    assert got.data_ptr() == g.data_ptr()
    assert_close(got, ref, what="in-place groupnorm C=128")
    rgb = torch.empty(3 * 16 * 24, 8, device="cuda", dtype=torch.float16)
    xin = rnd(3, 16, 24, 128, seed=8)
    w9, b = rnd(3, 3, 3, 128, seed=9, scale=(9 * 128) ** -0.5), rnd(3, seed=10, scale=0.1)
    O.conv2d_3x3(xin, w9, b, out=rgb[:, :3])
    assert_close(rgb[:, :3], R.conv2d_3x3(xin, w9, b), what="conv 128->3 into ld=8 rows")


# ---- bf16 build of the same kernels (libstar_sm100_bf16.so, -DSTAR_BF16): the CogVideoX DiT's dtype --------------------
@pytest.fixture()
def bf16_ref():
    from oracle import kernel_ref as R
    R.set_dtype(torch.bfloat16)
    yield R
    R.set_dtype(torch.float16)


def test_bf16_library_kernels(env, bf16_ref):
    """GEMM (+bias, residual, tanh-GELU, colscale), flash attention, LayerNorm, the temporal row gate, SiLU, the sinusoidal
    embedding and the spatial LIEM gate on bf16 tokens against the same torch references rounding to bf16 (8-bit mantissa:
    8e-3 relative L2)."""
    O, R = env[0], bf16_ref
    bf = torch.bfloat16

    def rb(*shape, seed=0, scale=1.0):
        return rnd(*shape, seed=seed, scale=scale).to(bf)
    a, w, bias, res = rb(1000, 3072, seed=1), rb(1536, 3072, seed=2, scale=3072 ** -0.5), rb(1536, seed=3, scale=0.1), rb(1000, 1536, seed=4)
    assert_close(O.linear(a, w, bias, res), R.linear(a, w, bias, res), rel=8e-3, max_rel=5e-2, what="bf16 linear")
    cs = rb(1536, seed=5)
    assert_close(O.linear_ex(a, w, bias, cs, res, 8), R.linear_ex(a, w, bias, cs, res, 8), rel=8e-3, max_rel=5e-2, what="bf16 linear_ex")
    qkv = rb(2 * 700, 3 * 256, seed=6)
    got = O.attention(qkv[:, :256], qkv[:, 256:512], qkv[:, 512:], 2, 4, 700, 700, 1, 0.125)
    assert got.dtype == bf
    assert_close(got, R.attention(qkv[:, :256], qkv[:, 256:512], qkv[:, 512:], 2, 4, 700, 700, 1, 0.125), rel=8e-3, max_rel=5e-2,
                 what="bf16 attention")
    x = rb(500, 3072, seed=7)
    g, b = (1 + 0.1 * torch.randn(3072, device="cuda")).to(bf), (0.1 * torch.randn(3072, device="cuda")).to(bf)
    assert_close(O.layernorm(x, g, b), R.layernorm(x, g, b), rel=8e-3, max_rel=5e-2, what="bf16 layernorm")
    assert_close(O.row_gate(x, 2, None, 0.4, -0.3), R.row_gate(x, 2, None, 0.4, -0.3), rel=8e-3, max_rel=5e-2, what="bf16 row_gate")
    assert_close(O.silu(x), R.silu(x), rel=8e-3, max_rel=5e-2, what="bf16 silu")
    t = torch.tensor([731, 12], device="cuda")
    assert_close(O.sinusoidal(t, 3072, dtype=bf), R.sinusoidal(t, 3072), rel=8e-3, max_rel=5e-2, what="bf16 sinusoidal")
    xi = rb(3 * 6 * 10, 256, seed=8)
    w98 = rb(98, seed=9, scale=0.2)
    assert_close(O.liem_spatial_gate(xi, w98, 3, 6, 10), R.liem_spatial_gate(xi, w98, 3, 6, 10), rel=1e-2, max_rel=5e-2, what="bf16 liem")
    # the fp16 library is untouched by the switch
    h = rnd(300, 320, seed=1)
    assert O.linear(h, rnd(320, 320, seed=2, scale=0.05)).dtype == torch.float16
