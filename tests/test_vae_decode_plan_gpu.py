"""Temporal VAE decode under split plans (frames per pass, upsample row bands, temporal pixel bands) on the sm_90a kernels."""
import pytest
import torch

from tests.test_vae import SMALL, _setup
from tests.util import rel_l2

GiB = 1 << 30


@pytest.mark.gpu
@pytest.mark.parametrize("h,w", [(16, 24), (34, 48)])
def test_split_plans_match_one_pass_and_oracle(h, w):
    """1 and 2 frames per pass, temporal bands of 7 / 100 / 1000 pixels and upsample bands of 2 / 6 / 10 rows (none divides a
    stage) against the one-pass decode of the same weights (max |difference| a few fp16 ulps of the output's magnitude), all
    held to test_decode_gpu's bound against the fp32 oracle"""
    from oracle.temporal_vae_ref import decode
    from star_b200.video_to_video.modules.temporal_vae import DecodePlan, decode_plan
    cfg, sd, vae = _setup(SMALL, device="cuda")
    z = torch.randn(3, 4, h, w, generator=torch.Generator().manual_seed(3)).cuda()
    ref = decode({k: v.cuda() for k, v in sd.items()}, z, 3, cfg)
    assert decode_plan(3, 3, h, w, SMALL["block_out_channels"]) == DecodePlan(3, h * w * 64, h * 8)
    one = vae.decode(z, num_frames=3).sample
    assert rel_l2(one, ref) < 4e-3
    scale = one.float().abs().max().item()
    for plan in (DecodePlan(1, 7, 6), DecodePlan(2, 100, 10), DecodePlan(1, 1000, 2), DecodePlan(3, 7, 6)):
        got = vae.decode(z, num_frames=3, plan=plan).sample
        torch.cuda.synchronize()
        err, diff = rel_l2(got, ref), (got.float() - one.float()).abs().max().item()
        print(f"latent {h}x{w} {plan}: rel-L2 vs fp32 oracle {err:.3e}, max |split - one pass| {diff:.3e} (output max {scale:.2f})")
        assert got.shape == one.shape and err < 4e-3
        assert diff <= 8 * 2 ** -10 * max(1.0, scale)


def _parent_res2d(r, x, n, H, W, eps=1e-6):
    """the 2-D resnet as the decoder and encoder ran it before decode plans: fresh outputs, no aliasing"""
    from star_b200 import ops
    cin = x.shape[1]
    t = ops.groupnorm(x, r["n1"][0], r["n1"][1], n, eps, True)
    t = ops.conv2d_3x3(t.view(n, H, W, cin), r["c1"][0], r["c1"][1])
    cout = t.shape[1]
    t = ops.groupnorm(t, r["n2"][0], r["n2"][1], n, eps, True, out=t)
    sc = ops.linear(x, r["sc"][0], r["sc"][1]) if "sc" in r else x
    return ops.conv2d_3x3(t.view(n, H, W, cout), r["c2"][0], r["c2"][1], residual=sc)


def _parent_decode(vae, z, T):
    from star_b200 import ops
    pk = vae._packed()["dec"]
    bf, _, H, W = z.shape
    B = bf // T

    def st_res(r, x, H, W):
        xs = _parent_res2d(r["s"], x, B * T, H, W)
        t = ops.groupnorm(xs, r["tn1"][0], r["tn1"][1], B, 1e-5, True)
        t = ops.conv_t3(t, r["tc1"][0], r["tc1"][1], B=B, T=T, HW=H * W)
        t = ops.groupnorm(t, r["tn2"][0], r["tn2"][1], B, 1e-5, True, out=t)
        return ops.conv_t3(t, r["tc2"][0], r["tc2"][1], residual=xs, B=B, T=T, HW=H * W)
    h = ops.nchw5_to_tokens(z.float().unsqueeze(2))
    h = ops.conv2d_3x3_c4(h.view(bf, H, W, 4), pk["in"][0], pk["in"][1])
    h = st_res(pk["mid"][0], h, H, W)
    for r in pk["mid"][1:]:
        h = vae._attention(pk["attn"], h, bf, H * W)
        h = st_res(r, h, H, W)
    for blk in pk["up"]:
        for r in blk["res"]:
            h = st_res(r, h, H, W)
        if "up" in blk:
            C = h.shape[1]
            h = ops.upsample2x(h, bf, H, W)
            H, W = 2 * H, 2 * W
            h = ops.conv2d_3x3(h.view(bf, H, W, C), blk["up"][0], blk["up"][1])
    h = ops.groupnorm(h, pk["nout"][0], pk["nout"][1], bf, 1e-6, True, out=h)
    rgb = torch.empty((bf * H * W, 8), dtype=torch.float16, device=h.device)
    ops.conv2d_3x3(h.view(bf, H, W, h.shape[1]), pk["out"][0], pk["out"][1], out=rgb[:, :3])
    return ops.vae_head(rgb, pk["head"][0], pk["head"][1], B, T, H, W)


def _parent_encode(vae, x):
    from star_b200 import ops
    pk = vae._packed()["enc"]
    n, c, H, W = x.shape
    x = torch.cat([x.float(), x.new_zeros(n, 4 - c, H, W).float()], dim=1)
    h = ops.nchw5_to_tokens(x.unsqueeze(2))
    h = ops.conv2d_3x3_c4(h.view(n, H, W, 4), pk["in"][0], pk["in"][1])
    for blk in pk["down"]:
        for r in blk["res"]:
            h = _parent_res2d(r, h, n, H, W)
        if "down" in blk:
            h, H, W = ops.conv2d_3x3_s2p(h.view(n, H, W, h.shape[1]), blk["down"][0], blk["down"][1], (0, 1, 0, 1))
    h = _parent_res2d(pk["mid"][0], h, n, H, W)
    h = vae._attention(pk["attn"], h, n, H * W)
    h = _parent_res2d(pk["mid"][1], h, n, H, W)
    h = ops.groupnorm(h, pk["nout"][0], pk["nout"][1], n, 1e-6, True, out=h)
    m = ops.conv2d_3x3(h.view(n, H, W, h.shape[1]), pk["out"][0], pk["out"][1])
    return ops.tokens_to_nchw5(m, n, m.shape[1], 1, H, W)[:, :, 0].float()


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["small", "full_width"])
def test_trivial_plan_equals_the_unplanned_decoder_byte_for_byte(case):
    """decode (trivial plan) and encode against the call sequence they ran before decode plans (fresh outputs, shortcut after
    the first conv, no in-place reuse, whole-window upsample), at test_decode_gpu's shapes"""
    from star_b200.video_to_video.modules.temporal_vae import DecodePlan, decode_plan
    kw = SMALL if case == "small" else {}
    _, _, vae = _setup(kw, device="cuda")
    h, w = (10, 12) if case == "small" else (14, 16)
    z = torch.randn(3, 4, h, w, generator=torch.Generator().manual_seed(1)).cuda()
    assert decode_plan(3, 3, h, w, vae.config.block_out_channels) == DecodePlan(3, h * w * 64, h * 8)
    assert torch.equal(vae.decode(z, num_frames=3).sample, _parent_decode(vae, z, 3))
    x = (torch.rand(1, 3, 8 * h, 8 * w, generator=torch.Generator().manual_seed(2)) * 2 - 1).cuda()
    assert torch.equal(vae.encode(x).latent_dist.parameters, _parent_encode(vae, x))


@pytest.mark.gpu
def test_banded_groupnorm_and_conv_t3_match_the_whole_clip():
    """ops.groupnorm(bands=) and ops.conv_t3(band=) with B = 2 clips of T = 3 frames, HW = 200, bands of 70 (does not divide
    HW) and 50 pixels (under one 128-row tile), against the whole-clip ops and oracle/kernel_ref.py"""
    from oracle import kernel_ref as KR
    from star_b200 import ops
    g = torch.Generator().manual_seed(7)
    B, T, HW, C = 2, 3, 200, 64
    x = (torch.randn(B * T * HW, C, generator=g) * 2 + 0.5)
    x[T * HW:] = x[T * HW:] * 3 - 1                                # the two clips have different statistics
    x = x.half().cuda()
    gamma, beta = (torch.rand(C, generator=g) + 0.5).half().cuda(), (torch.randn(C, generator=g) * 0.1).half().cuda()
    w3 = (torch.randn(C, 3, C, generator=g) / (3 * C) ** 0.5).half().cuda()
    bias, res = (torch.randn(C, generator=g) * 0.1).half().cuda(), torch.randn(B * T * HW, C, generator=g).half().cuda()
    full = ops.groupnorm(x, gamma, beta, B, 1e-5, True)
    want = ops.conv_t3(full, w3, bias, residual=res, B=B, T=T, HW=HW)
    ref = KR.conv_t3(KR.groupnorm(x, gamma, beta, B, 1e-5, True), w3, bias, residual=res, B=B, T=T, HW=HW)
    rows = torch.arange(B * T * HW, device=x.device).view(B * T, HW)
    for band in (70, 50):
        out = torch.full_like(res, float("nan"))
        for (p0, p1), gb in ops.groupnorm(x, gamma, beta, B, 1e-5, True, bands=(HW, band)):
            assert torch.equal(gb, full[rows[:, p0:p1].reshape(-1)])
            ops.conv_t3(gb, w3, bias, residual=res, B=B, T=T, HW=HW, band=(p0, p1), out=out)
        torch.cuda.synchronize()
        diff = (out.float() - want.float()).abs().max().item()
        print(f"bands of {band}: max |banded - whole clip| {diff:.3e}, rel-L2 vs kernel_ref {rel_l2(out, ref):.3e}")
        assert torch.isfinite(out).all() and diff <= 2 ** -8
        assert rel_l2(out, ref) < 2e-3


@pytest.mark.gpu
def test_banded_conv2d_3x3_rows_match_the_whole_frame():
    """ops.conv2d_3x3(rows=) over bands of 2 / 5 / 7 output rows of 2 frames: each band equals those rows of the whole conv"""
    from star_b200 import ops
    g = torch.Generator().manual_seed(8)
    x = torch.randn(2, 13, 24, 64, generator=g).half().cuda()
    w9 = (torch.randn(64, 3, 3, 64, generator=g) / 24).half().cuda()
    bias = (torch.randn(64, generator=g) * 0.1).half().cuda()
    want = ops.conv2d_3x3(x, w9, bias).view(2, 13, 24, 64)
    for step in (2, 5, 7):
        for r0 in range(0, 13, step):
            n = min(step, 13 - r0)
            got = ops.conv2d_3x3(x, w9, bias, rows=(r0, n)).view(2, n, 24, 64)
            assert (got.float() - want[:, r0:r0 + n].float()).abs().max().item() <= 2 ** -8


@pytest.mark.gpu
def test_split_plan_peak_memory_matches_prediction():
    """full-width decoder, 3-frame window at latent 96x160 (768x1280 output), 1 frame per pass, 64 Ki-pixel and 100-row bands:
    torch's peak over the decode within 10 % of decode_peak_bytes"""
    from star_b200.utils.synth import synth_tensor
    from star_b200.video_to_video.modules.temporal_vae import AutoencoderKLTemporalDecoder, DecodePlan, decode_peak_bytes
    dev = torch.device("cuda", 0)
    with torch.device("meta"):
        vae = AutoencoderKLTemporalDecoder()
    vae.load_state_dict({k: synth_tensor(k, v.shape, 0, dev) for k, v in vae.state_dict().items()}, assign=True)
    vae = vae.eval()
    h, w = 96, 160
    z = torch.randn(3, 4, h, w, device=dev)
    plan = DecodePlan(1, 65536, 100)
    vae.decode(z, num_frames=3, plan=plan)                   # packs the weights
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated(dev)
    torch.cuda.reset_peak_memory_stats(dev)
    out = vae.decode(z, num_frames=3, plan=plan).sample
    torch.cuda.synchronize()
    got = torch.cuda.max_memory_allocated(dev) - base
    want = decode_peak_bytes(plan, 3, h, w)
    print(f"decode {plan} latent {h}x{w}: peak {got / GiB:.3f} GiB, predicted {want / GiB:.3f} GiB")
    assert out.shape == (3, 3, 8 * h, 8 * w) and torch.isfinite(out).all()
    assert abs(got - want) <= 0.10 * want


@pytest.mark.gpu
def test_1080p_to_4x_window_decodes_within_prediction():
    """one 3-frame window at the 1080p -> 4x latent (546x968 -> 4368x7744), synthetic weights, planned decode: the peak above
    the resident weights within 2 % of decode_peak_bytes, and under 64 GiB in all"""
    dev = torch.device("cuda", 0)
    free, _ = torch.cuda.mem_get_info(dev)
    if free < 66 * GiB:
        pytest.skip(f"needs ~62 GiB of device memory, {free / GiB:.1f} GiB free")
    from star_b200.utils.synth import synth_tensor
    from star_b200.video_to_video.modules.temporal_vae import AutoencoderKLTemporalDecoder, decode_peak_bytes, decode_plan
    with torch.device("meta"):
        vae = AutoencoderKLTemporalDecoder()
    vae.load_state_dict({k: synth_tensor(k, v.shape, 0, dev) for k, v in vae.state_dict().items()}, assign=True)
    vae = vae.eval()
    z = torch.randn(3, 4, 546, 968, device=dev)
    vae._packed()
    base = torch.cuda.memory_allocated(dev)
    torch.cuda.reset_peak_memory_stats(dev)
    out = vae.decode(z, num_frames=3).sample
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated(dev)
    want = decode_peak_bytes(decode_plan(3, 3, 546, 968), 3, 546, 968)
    print(f"1080p -> 4x decode window: peak {peak / GiB:.1f} GiB including resident weights, predicted {want / GiB:.1f} GiB "
          f"+ {base / GiB:.1f} GiB")
    assert out.shape == (3, 3, 4368, 7744)
    assert torch.isfinite(out[:, :, ::97, ::89]).all()
    assert abs(peak - base - want) <= 0.02 * want and peak <= 64 * GiB
