"""Spatially tiled sampling on the GPU: the CFG + v->x0 + blend kernel (star_cfg_x0_blend, reached through
ops.cfg_x0(..., blend=)) against star_cfg_x0 plus a torch weighted accumulate, and tiled sample_sr / denoise_latents
against the untiled path, a torch restatement of the tile loop, and eager execution under CUDA graphs."""
from types import SimpleNamespace

import pytest
import torch

from tests.util import SMALL_KW, rel_l2, synth_model

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def small_net():
    net, _ = synth_model(SMALL_KW, seed=1, device="cuda")
    return net


@pytest.fixture(scope="module")
def diffusion():
    from star_b200.video_to_video.diffusion.diffusion_sdedit import GaussianDiffusion
    from star_b200.video_to_video.diffusion.schedules_sdedit import noise_schedule
    sig = noise_schedule(schedule="logsnr_cosine_interp", n=1000, zero_terminal_snr=True, scale_min=2.0, scale_max=4.0)
    return GaussianDiffusion(sigmas=sig)


def gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def pipe_for(net, cuda_graph=False):
    from star_b200.video_to_video.video_to_video_model import VideoToVideo_sr
    ny = torch.zeros(1, 77, 1024)
    return VideoToVideo_sr(SimpleNamespace(model_path=None), device=torch.device("cuda:0"), text_encoder=lambda s: ny,
                           vae=object(), generator=net, cuda_graph=cuda_graph)


def latents(F, H, W, seed=3):
    g = torch.Generator().manual_seed(seed)
    feat = 0.5 * torch.randn(1, 4, F, H, W, generator=g)
    y, ny = torch.randn(1, 77, 1024, generator=g), torch.randn(1, 77, 1024, generator=g)
    noise = torch.randn(feat.shape, generator=g).cuda()
    return feat, y, ny, noise


def pinned_sampler(shape, seed):
    g = gen(seed)
    return lambda a, b: torch.randn(shape, device="cuda", generator=g)


# -- kernel -----------------------------------------------------------------------------------------------------------
def blend_case(B, rescale, f0, lo, hi, r0, c0, unit, seed):
    from star_b200 import ops
    C, F, H, W, Ft, th, tw = 4, 12, 30, 44, 7, 10, 16
    g = gen(seed)
    y = torch.randn(B, C, Ft, th, tw, device="cuda", generator=g).half()
    u = (y.float() + 0.3 * torch.randn(y.shape, device="cuda", generator=g)).half()
    xt = torch.randn(B, C, F, H, W, device="cuda", generator=g)
    al = torch.rand(B, 1, 1, 1, 1, device="cuda", generator=g) * 0.5 + 0.3
    sg = torch.sqrt(1 - al ** 2)
    if unit:
        wy, wx = torch.ones(th, device="cuda"), torch.ones(tw, device="cuda")
        acc = torch.zeros_like(xt)
    else:
        wy = torch.rand(th, device="cuda", generator=g) + 0.05
        wx = torch.rand(tw, device="cuda", generator=g) + 0.05
        acc = torch.randn(xt.shape, device="cuda", generator=g)
    x0 = ops.cfg_x0(y, u, xt[:, :, f0:f0 + Ft, r0:r0 + th, c0:c0 + tw].contiguous(), al, sg, 7.5, rescale)
    ref = acc.clone()
    ref[:, :, f0 + lo:f0 + hi, r0:r0 + th, c0:c0 + tw] += (wy[:, None] * wx[None, :]) * x0[:, :, lo:hi]
    got = ops.cfg_x0(y, u, xt, al, sg, 7.5, rescale, blend=ops.TileBlend(acc, f0, lo, hi, r0, c0, wy, wx))
    torch.cuda.synchronize()
    assert got is acc
    return got, ref


@pytest.mark.parametrize("B", [1, 2])
@pytest.mark.parametrize("rescale", [None, 0.2])
@pytest.mark.parametrize("f0,lo,hi,r0,c0", [(0, 0, 7, 0, 0), (3, 2, 5, 7, 13), (5, 0, 6, 20, 28), (2, 6, 7, 1, 3)])
def test_blend_unit_weights_bit_exact(B, rescale, f0, lo, hi, r0, c0):
    """weight 1.0 into a zeroed accumulator == star_cfg_x0 on the cropped tile followed by the slice copy, bit for bit;
    everything outside the kept window stays zero"""
    got, ref = blend_case(B, rescale, f0, lo, hi, r0, c0, unit=True, seed=B + 10 * f0 + r0)
    assert torch.equal(got, ref)


@pytest.mark.parametrize("B", [1, 2])
@pytest.mark.parametrize("rescale", [None, 0.2])
@pytest.mark.parametrize("f0,lo,hi,r0,c0", [(3, 2, 5, 7, 13), (5, 0, 6, 20, 27)])
def test_blend_weighted_accumulate(B, rescale, f0, lo, hi, r0, c0):
    got, ref = blend_case(B, rescale, f0, lo, hi, r0, c0, unit=False, seed=100 + B + r0)
    torch.testing.assert_close(got, ref, rtol=1e-6, atol=1e-6)


@pytest.mark.parametrize("rescale", [None, 0.2])
def test_blend_two_overlapping_tiles(rescale):
    """two tiles whose windows overlap, accumulated one after the other into the same clip buffer"""
    from star_b200 import ops
    B, C, F, H, W, th, tw = 2, 4, 6, 26, 40, 18, 24
    g = gen(7)
    xt = torch.randn(B, C, F, H, W, device="cuda", generator=g)
    al = torch.full((B, 1, 1, 1, 1), 0.6, device="cuda")
    sg = torch.sqrt(1 - al ** 2)
    acc = torch.zeros_like(xt)
    ref = torch.zeros_like(xt)
    for r0, c0 in ((0, 0), (8, 16)):
        y = torch.randn(B, C, F, th, tw, device="cuda", generator=g).half()
        u = (y.float() + 0.3 * torch.randn(y.shape, device="cuda", generator=g)).half()
        wy, wx = torch.rand(th, device="cuda", generator=g) + 0.1, torch.rand(tw, device="cuda", generator=g) + 0.1
        x0 = ops.cfg_x0(y, u, xt[:, :, :, r0:r0 + th, c0:c0 + tw].contiguous(), al, sg, 7.5, rescale)
        ref[:, :, 1:5, r0:r0 + th, c0:c0 + tw] += (wy[:, None] * wx[None, :]) * x0[:, :, 1:5]
        ops.cfg_x0(y, u, xt, al, sg, 7.5, rescale, blend=ops.TileBlend(acc, 0, 1, 5, r0, c0, wy, wx))
    torch.cuda.synchronize()
    torch.testing.assert_close(acc, ref, rtol=1e-6, atol=1e-6)


def test_blend_rejects_windows_outside_the_clip():
    from star_b200 import ops
    from star_b200.lib import StarError
    y = torch.randn(1, 4, 4, 10, 16, device="cuda").half()
    xt = torch.randn(1, 4, 6, 20, 32, device="cuda")
    al = torch.full((1, 1, 1, 1, 1), 0.6, device="cuda")
    w10, w16 = torch.ones(10, device="cuda"), torch.ones(16, device="cuda")
    for f0, lo, hi, r0, c0 in ((3, 0, 4, 0, 0), (0, 0, 4, 11, 0), (0, 0, 4, 0, 17), (0, 2, 2, 0, 0), (0, 0, 5, 0, 0),
                               (-1, 0, 4, 0, 0)):
        with pytest.raises(StarError):
            ops.cfg_x0(y, y, xt, al, al, 7.5, 0.2, blend=ops.TileBlend(torch.zeros_like(xt), f0, lo, hi, r0, c0, w10, w16))


# -- sampler ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("F,max_chunk_len", [(8, 32), (22, 8)])
def test_one_tile_equals_untiled(small_net, F, max_chunk_len):
    """a tile that covers the whole latent is the untiled computation, bit for bit (with and without temporal chunks)"""
    feat, y, ny, noise = latents(F, 26, 32)
    pipe = pipe_for(small_net)
    outs = []
    for tiles in ({}, {"tile_size": (34, 40)}, {"tile_size": (26, 32), "tile_overlap": 8}):
        outs.append(pipe.denoise_latents(feat, y, ny, steps=2, solver_mode="normal", max_chunk_len=max_chunk_len,
                                         noise=noise, noise_sampler=pinned_sampler(feat.shape, 5), **tiles))
    assert torch.isfinite(outs[0]).all()
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])


class LocalDenoiser:
    """a denoiser whose fp16 output at each pixel depends only on (x, hint, y) there: tiling cannot change it"""

    def __call__(self, x, t, y=None, hint=None, hint_chunk=None, variant_info=None):
        h = hint_chunk if hint_chunk is not None else hint
        return (torch.tanh(0.7 * x + 0.3 * h) * (1 + 0.1 * y.mean()) + 0.05 * torch.sin(3 * x)).half()


def test_tiled_exact_for_spatially_local_model(diffusion):
    """one solver step: the tiled x0 is the untiled one times weights that sum to 1, so the two differ by fp32 rounding of
    the blend.  (Over several steps such last-bit differences of the latent flip the rounding of some fp16 model outputs,
    and the gap grows to ~1e-5.)"""
    from star_b200.video_to_video.video_to_video_model import make_tiles
    feat, y, ny, noise = latents(20, 42, 56, seed=11)
    feat = feat.cuda()
    tiles = make_tiles(42, 56, (18, 24), 6)
    assert len(tiles[0]) * len(tiles[1]) >= 9
    outs = []
    for tile_inds in (None, tiles):
        outs.append(diffusion.sample_sr(noise=noise, model=LocalDenoiser(),
                                        model_kwargs=[{"y": y.cuda()}, {"y": ny.cuda()}, {"hint": feat}],
                                        guide_scale=7.5, guide_rescale=None, solver="dpmpp_2m_sde", solver_mode="normal",
                                        steps=1, t_max=999, t_min=0, discretization="trailing",
                                        chunk_inds=[(0, 12), (8, 20)], noise_sampler=pinned_sampler(feat.shape, 9),
                                        tile_inds=tile_inds))
    err = rel_l2(outs[1], outs[0])
    print(f"tiled vs untiled, pixel-local denoiser: rel-L2 {err:.3e}")
    assert err <= 1e-6


def test_tiled_matches_torch_restatement(small_net, diffusion, monkeypatch):
    """reduced UNet, 42x48 latent, tiles 26x32 with overlap 8 (2 x 2 tiles), 2 steps: every x0 evaluation of tiled
    sample_sr against a torch loop over the tiles (forward_cfg_pair on the crops, CFG/x0 of each tile by the untiled
    ops.cfg_x0, weights from make_tiles, weighted sum)"""
    from star_b200 import ops
    from star_b200.video_to_video.diffusion import diffusion_sdedit as D
    from star_b200.video_to_video.video_to_video_model import make_tiles
    feat, y, ny, noise = latents(8, 42, 48, seed=21)
    feat, y, ny = feat.cuda(), y.cuda(), ny.cuda()
    tiles = make_tiles(42, 48, (26, 32), 8)
    assert len(tiles[0]) == 2 and len(tiles[1]) == 2

    records = []
    real = D.sample_dpmpp_2m_sde

    def recording_solver(x, fn, sigmas, **kw):
        def wrapped(xt, sigma, variant_info=None):
            x0 = fn(xt, sigma, variant_info=variant_info)
            records.append((xt.clone(), sigma.clone(), x0.clone()))
            return x0
        return real(x, wrapped, sigmas, **kw)

    monkeypatch.setattr(D, "sample_dpmpp_2m_sde", recording_solver)
    diffusion.sample_sr(noise=noise, model=small_net, model_kwargs=[{"y": y}, {"y": ny}, {"hint": feat}], guide_scale=7.5,
                        guide_rescale=0.2, solver="dpmpp_2m_sde", solver_mode="normal", steps=2, t_max=999, t_min=0,
                        discretization="trailing", noise_sampler=pinned_sampler(feat.shape, 4), tile_inds=tiles)
    assert len(records) >= 2
    rows, cols, row_w, col_w = tiles
    for xt, sigma, x0 in records:
        t = diffusion._sigma_to_t(sigma).repeat(1).round().long()
        al, sg = D._gather_coef(diffusion.alphas, t, xt), D._gather_coef(diffusion.sigmas, t, xt)
        ref = torch.zeros_like(xt)
        for (r0, r1), wy in zip(rows, row_w):
            for (c0, c1), wx in zip(cols, col_w):
                xc = xt[:, :, :, r0:r1, c0:c1].contiguous()
                yo, uo = small_net.forward_cfg_pair(xc, t, (y, ny), hint=feat[:, :, :, r0:r1, c0:c1].contiguous())
                x0c = ops.cfg_x0(yo, uo, xc, al, sg, 7.5, 0.2)
                ref[:, :, :, r0:r1, c0:c1] += (wy.cuda()[:, None] * wx.cuda()[None, :]) * x0c
        err = rel_l2(x0, ref)
        print(f"sigma {float(sigma):.4f}: tiled x0 vs torch restatement rel-L2 {err:.3e}")
        assert err <= 1e-5


def test_tiled_cuda_graph_equals_eager(small_net):
    """tiled denoise_latents under CUDA graphs == eager, bit for bit; equal tile shapes need one graph per distinct chunk
    length (22 frames, max_chunk_len 8: chunks of 8, 8, 8 and 10 frames -> 2 graphs)"""
    from star_b200.video_to_video.video_to_video_model import make_chunks
    feat, y, ny, noise = latents(22, 42, 48, seed=31)
    lengths = {e - s for s, e in make_chunks(22, 0, 8)}
    assert len(lengths) == 2
    outs = []
    for graphed in (False, True):
        pipe = pipe_for(small_net, cuda_graph=graphed)
        outs.append(pipe.denoise_latents(feat, y, ny, steps=2, solver_mode="normal", max_chunk_len=8, noise=noise,
                                         noise_sampler=pinned_sampler(feat.shape, 6), tile_size=(26, 32), tile_overlap=8))
        if graphed:
            assert pipe._graphed is not None and pipe._graphed.replays > 0
            assert len(pipe._graphed._graphs) == len(lengths)
    assert torch.isfinite(outs[0]).all()
    assert torch.equal(outs[0], outs[1])


def test_tiled_errors(small_net, diffusion):
    from star_b200.video_to_video.video_to_video_model import make_tiles
    feat, y, ny, noise = latents(4, 26, 32)
    feat = feat.cuda()
    tiles = make_tiles(26, 32, (18, 16), 4)
    kw = dict(noise=noise, model_kwargs=[{"y": y.cuda()}, {"y": ny.cuda()}, {"hint": feat}], guide_scale=7.5,
              guide_rescale=0.2, solver="dpmpp_2m_sde", solver_mode="normal", steps=1, t_max=999, t_min=0,
              discretization="trailing", tile_inds=tiles)
    fp32 = lambda x, t, y=None, hint=None, hint_chunk=None, variant_info=None: x * 0.5        # noqa: E731
    with pytest.raises(TypeError, match="fp16 CUDA"):
        diffusion.sample_sr(model=fp32, **kw)
    with pytest.raises(ValueError):
        diffusion.sample_sr(model=small_net, **dict(kw, guide_scale=None))


def test_large_frame_memory_is_bounded_by_the_tile():
    """the full UNet (synthetic weights) on a 362x648 latent (720p -> 4x), 8 frames, tiles 90x160 with overlap 16, one
    solver step: finite, and the peak allocation stays within 1.25x of one 90x160 tile's CFG-pair forward"""
    from bench import build_model
    dev = torch.device("cuda", 0)
    net, _, _ = build_model(False, dev)
    feat, y, ny, noise = latents(8, 362, 648, seed=41)
    x, hint = torch.randn(1, 4, 8, 90, 160, device=dev), torch.randn(1, 4, 8, 90, 160, device=dev)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(dev)
    out = net.forward_cfg_pair(x, torch.tensor([500], device=dev), (y.to(dev), ny.to(dev)), hint=hint)
    del out, x, hint
    torch.cuda.synchronize()
    tile_peak = torch.cuda.max_memory_allocated(dev)
    pipe = pipe_for(net)
    torch.cuda.reset_peak_memory_stats(dev)
    z = pipe.denoise_latents(feat, y, ny, steps=1, solver_mode="normal", noise=noise,
                             noise_sampler=pinned_sampler(feat.shape, 8), tile_size=(90, 160), tile_overlap=16)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated(dev)
    print(f"362x648 x 8 frames tiled: peak {peak / 2 ** 30:.2f} GiB, one 90x160 tile {tile_peak / 2 ** 30:.2f} GiB")
    assert z.shape == feat.shape and torch.isfinite(z).all()
    assert peak <= 1.25 * tile_peak
