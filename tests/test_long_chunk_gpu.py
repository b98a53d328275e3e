"""Chunks longer than 64 frames (max_chunk_len >= 52): the T > 64 temporal-attention kernel (csrc/tattn_long.cuh)
against the fp32 torch reference, and the reduced UNet and the chunked sampler at T > 64 against golden outputs of
the reference (tests/golden/long_chunk.pt, written by oracle/make_golden_long_chunk.py).  Tolerances as in
test_kernels_gpu.py (kernels) and test_unet_gpu.py (UNet, sampler)."""
import os

import pytest
import torch

from tests.util import SMALL_KW, assert_close, make_inputs, rel_l2, synth_model

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden", "long_chunk.pt")


@pytest.fixture(scope="module")
def kernels():
    from oracle import kernel_ref as R
    from star_b200 import ops as O
    return O, R


@pytest.fixture(scope="module")
def small_net():
    net, _ = synth_model(SMALL_KW, seed=1, device="cuda")
    return net


@pytest.fixture(scope="module")
def gold():
    return torch.load(GOLD)


def rnd(*shape, seed=0, scale=1.0, dtype=torch.float16):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, generator=g, device="cuda") * scale).to(dtype)


@pytest.mark.parametrize("B,T,HW,heads", [
    (1, 65, 33, 5), (2, 78, 17, 10), (1, 96, 9, 20), (2, 127, 7, 5), (1, 128, 31, 5),
    (2, 129, 5, 10), (1, 200, 11, 5), (2, 256, 3, 20), (1, 1024, 3, 5),
])
def test_temporal_attention_long(kernels, B, T, HW, heads):
    O, R = kernels
    Ci = heads * 64
    qkv = rnd(B * T * HW, 3 * Ci, seed=T)
    got = O.temporal_attention(qkv, B, T, HW, heads, Ci)
    torch.cuda.synchronize()
    assert_close(got, R.temporal_attention(qkv, B, T, HW, heads, Ci), what=f"temporal attention B{B} T{T} HW{HW} h{heads}")


def test_temporal_attention_long_strided_qkv(kernels):
    """q|k|v columns inside wider rows (ld > 3 Ci), as a slice of a larger projection output"""
    O, R = kernels
    B, T, HW, heads, Ci = 2, 90, 13, 5, 320
    buf = rnd(B * T * HW, 3 * Ci + 128, seed=3)
    qkv = buf[:, 64:64 + 3 * Ci]
    assert qkv.stride(0) == 3 * Ci + 128
    got = O.temporal_attention(qkv, B, T, HW, heads, Ci)
    torch.cuda.synchronize()
    assert_close(got, R.temporal_attention(qkv.contiguous(), B, T, HW, heads, Ci), what="temporal attention ld > 3 Ci")


def test_temporal_attention_long_peaky(kernels):
    """large logits whose row maximum sits in the first key block for some pixels and in a later one for others:
    exercises the running-max rescale between 64-frame key blocks"""
    O, R = kernels
    B, T, HW, heads, Ci = 1, 150, 8, 5, 320
    x = rnd(B, T, HW, 3 * Ci, seed=4, scale=2.0).float()
    k = x[..., Ci:2 * Ci]
    k[:, :64, 0::2] *= 2.5           # even pixels: the largest keys in block 0
    k[:, 64:, 1::2] *= 2.5           # odd pixels: in blocks 1 and 2
    qkv = x.half().reshape(B * T * HW, 3 * Ci)
    got = O.temporal_attention(qkv, B, T, HW, heads, Ci)
    torch.cuda.synchronize()
    assert_close(got, R.temporal_attention(qkv, B, T, HW, heads, Ci), rel=4e-3, what="temporal attention peaky")


@pytest.mark.parametrize("T", [78, 128])
def test_temporal_attention_long_level0(kernels, T):
    """the UNet's level-0 shape (960p latent: 26 352 pixels, 5 heads); the fp32 reference runs in pixel chunks"""
    O, R = kernels
    B, HW, heads, Ci = 1, 26352, 5, 320
    qkv = rnd(B * T * HW, 3 * Ci, seed=5)
    got = O.temporal_attention(qkv, B, T, HW, heads, Ci).view(B, T, HW, Ci)
    torch.cuda.synchronize()
    ref = torch.empty_like(got)
    x = qkv.view(B, T, HW, 3 * Ci)
    step = 2048
    for p0 in range(0, HW, step):
        n = min(step, HW - p0)
        part = x[:, :, p0:p0 + n].reshape(B * T * n, 3 * Ci)
        ref[:, :, p0:p0 + n] = R.temporal_attention(part, B, T, n, heads, Ci).view(B, T, n, Ci)
    assert_close(got, ref, what=f"temporal attention level 0 T{T}")


def test_temporal_attention_long_bf16(kernels):
    O, R = kernels
    B, T, HW, heads, Ci = 2, 100, 9, 5, 320
    qkv = rnd(B * T * HW, 3 * Ci, seed=6, dtype=torch.bfloat16)
    R.set_dtype(torch.bfloat16)
    try:
        got = O.temporal_attention(qkv, B, T, HW, heads, Ci)
        torch.cuda.synchronize()
        assert got.dtype == torch.bfloat16
        assert_close(got, R.temporal_attention(qkv, B, T, HW, heads, Ci), rel=8e-3, max_rel=5e-2, what="bf16 temporal attention")
    finally:
        R.set_dtype(torch.float16)


def test_unet_small_long_chunk_vs_golden(small_net, gold):
    for c in gold["cases"]:
        x, hint, y = make_inputs(c["seed"], c["B"], c["F"], c["H"], c["W"])
        out = small_net(x.cuda(), torch.tensor(c["t"]).cuda(), y.cuda(), hint=hint.cuda())
        torch.cuda.synchronize()
        err = rel_l2(out.cpu(), c["out_fp32"])
        print(f"F={c['F']}: rel-L2 vs fp32 oracle {err:.3e} (reference fp16 path: {c['ref_fp16_rel_err']:.3e})")
        assert err <= 1.5 * c["ref_fp16_rel_err"] and err <= 4e-3


def test_sampler_long_chunks_vs_golden(small_net, gold):
    """sample_sr over make_chunks(100, 0, 64) = a 64-frame and a 68-frame chunk, 2 steps, CFG 7.5, identical noise"""
    from star_b200.video_to_video.diffusion.diffusion_sdedit import GaussianDiffusion
    from star_b200.video_to_video.diffusion.schedules_sdedit import noise_schedule
    from star_b200.video_to_video.video_to_video_model import make_chunks
    g = gold["sampler"]
    chunks = [tuple(c) for c in make_chunks(g["F"], 0, g["max_chunk_len"])]
    assert chunks == [tuple(c) for c in g["chunk_inds"]]
    x, hint, y = make_inputs(g["input_seed"], 1, g["F"], g["H"], g["W"])
    _, _, ny = make_inputs(g["neg_seed"], 1, g["F"], g["H"], g["W"])
    sig = noise_schedule(schedule="logsnr_cosine_interp", n=1000, zero_terminal_snr=True, scale_min=2.0, scale_max=4.0)
    diff = GaussianDiffusion(sigmas=sig)
    gen = torch.Generator().manual_seed(g["noise_seed"])
    sampler = lambda a, b: (-torch.randn(x.shape, generator=gen)).cuda()     # noqa: E731
    out = diff.sample_sr(noise=x.cuda(), model=small_net, model_kwargs=[{"y": y.cuda()}, {"y": ny.cuda()},
                                                                        {"hint": hint.cuda()}],
                         guide_scale=7.5, guide_rescale=0.2, solver="dpmpp_2m_sde", solver_mode="normal",
                         steps=g["steps"], t_max=899, t_min=0, discretization="trailing", chunk_inds=chunks,
                         noise_sampler=sampler)
    err = rel_l2(out.cpu(), g["out"])
    print(f"sample_sr chunks {chunks}, 2 steps: rel-L2 vs reference fp32 {err:.3e}")
    assert err <= 1e-2


@pytest.mark.parametrize("frames", [78, 100])
def test_denoise_latents_long_chunks_cuda_graph(small_net, frames):
    """denoise_latents(max_chunk_len=64, cuda_graph=True) == eager, bit for bit: 78 frames are one 78-frame chunk,
    100 frames a 64-frame and a 68-frame chunk (two graphs, blended overlap)"""
    from types import SimpleNamespace
    from star_b200.video_to_video.video_to_video_model import VideoToVideo_sr
    feat = torch.randn(1, 4, frames, 10, 8, generator=torch.Generator().manual_seed(3))
    y, ny = torch.randn(1, 77, 1024, generator=torch.Generator().manual_seed(4)), torch.zeros(1, 77, 1024)
    outs = []
    for graphed in (False, True):
        m = VideoToVideo_sr(SimpleNamespace(model_path=None), device=torch.device("cuda:0"), text_encoder=lambda s: ny, vae=object(),
                            generator=small_net, cuda_graph=graphed)
        g = torch.Generator(device="cuda").manual_seed(5)
        outs.append(m.denoise_latents(feat, y, ny, steps=2, solver_mode="normal", max_chunk_len=64,
                                      noise=torch.randn(feat.shape, generator=torch.Generator().manual_seed(6)).cuda(),
                                      noise_sampler=lambda a, b: torch.randn(feat.shape, device="cuda", generator=g)))
        if graphed:
            assert m._graphed is not None and m._graphed.replays > 0
            assert len(m._graphed._graphs) == (1 if frames == 78 else 2)
    assert torch.isfinite(outs[0]).all()
    assert torch.equal(outs[0], outs[1])
