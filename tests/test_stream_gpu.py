"""VideoToVideo_sr.enhance_frames_iter on the GPU (small UNet, small temporal VAE, synthetic weights, seeded inputs):

* identity: its windows, concatenated, equal ops.adain_color_fix(test(...)) byte for byte under the same seed -- for 1-7
  frames, a target inside the 720x1280 canvas (centred crop) and one past it (bottom / right pad), several denoise chunks and
  spatial tiles;
* ownership and pacing: a slow consumer that overwrites each yielded tensor still gets correct later windows, and a consumer
  that stops after the first window leaves no work on the stream;
* memory: the peak grows with the clip by a few latent frames per frame, not by output-resolution frames.
"""
import time
from types import SimpleNamespace

import pytest
import torch

from tests.test_vae import SMALL, _setup
from tests.util import SMALL_KW, synth_model

LATENT_FRAME = 4 * 90 * 160 * 4              # bytes of one fp32 latent frame of the 720x1280 canvas (230 400)
DECODED_FRAME = 3 * 720 * 1280 * 2           # bytes of one decoded fp16 canvas frame (5.5 MB)


@pytest.fixture(scope="module")
def pipe():
    from star_b200.video_to_video.video_to_video_model import VideoToVideo_sr
    net, _ = synth_model(SMALL_KW, seed=1, device="cuda")
    _, _, vae = _setup(SMALL, device="cuda")
    ny = -torch.randn(1, 77, 1024, generator=torch.Generator().manual_seed(4))
    return VideoToVideo_sr(SimpleNamespace(model_path=None), device=torch.device("cuda"), text_encoder=lambda s: ny, vae=vae,
                           generator=net)


def clip(F, lr, scale=4, seed=7):
    g = torch.Generator().manual_seed(seed)
    video = torch.rand(F, 3, *lr, generator=g) * 2 - 1
    return {"video_data": video, "y": torch.randn(1, 77, 1024, generator=g), "target_res": (lr[0] * scale, lr[1] * scale)}


def whole_clip(pipe, inp, **kw):
    """the whole-clip composition: test() on the device, then the colour fix over all frames at once"""
    from star_b200 import ops
    from star_b200.video_to_video.utils.seed import setup_seed
    setup_seed(666)
    return ops.adain_color_fix(pipe.test(inp, **kw).cuda(), inp["video_data"].cuda(), uint8=True).cpu()


def streamed(pipe, inp, **kw):
    from star_b200.video_to_video.utils.seed import setup_seed
    setup_seed(666)
    return list(pipe.enhance_frames_iter(inp, **kw))


def check_windows(wins, F, H, W, dtype=torch.uint8):
    assert [s for s, _ in wins] == list(range(0, F, 3))
    for s, fr in wins:
        assert fr.shape == (min(3, F - s), H, W, 3) and fr.dtype == dtype and fr.device.type == "cpu"
    return torch.cat([fr for _, fr in wins])


STEPS = dict(steps=2, solver_mode="normal", guide_scale=7.5)
CASES = {   # name: (frames, LR size, max_chunk_len, tile_size)
    **{f"centred F={F}": (F, (96, 160), 32, None) for F in (1, 2, 3, 4, 7)},
    "bottom-right pad F=4": (4, (188, 336), 32, None),          # 752x1344 -> canvas 784x1408
    "chunks F=7": (7, (96, 160), 4, None),
    "tiles F=4": (4, (96, 160), 32, (50, 96)),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_iter_equals_whole_clip(pipe, case):
    F, lr, mcl, tile = CASES[case]
    inp = clip(F, lr)
    kw = dict(STEPS, max_chunk_len=mcl, tile_size=tile)
    want = whole_clip(pipe, inp, **kw)
    got = check_windows(streamed(pipe, inp, **kw), F, *inp["target_res"])
    diff = (got.int() - want.int()).abs()
    print(f"{case}: {got.shape}, max |streamed - whole clip| {diff.max().item()}")
    assert torch.equal(got, want), f"{case}: {int((diff > 0).sum())} bytes differ, max {diff.max().item()}"


@pytest.mark.gpu
def test_iter_fp32_frames(pipe):
    from star_b200 import ops
    from star_b200.video_to_video.utils.seed import setup_seed
    inp = clip(4, (96, 160))
    setup_seed(666)
    want = ops.adain_color_fix(pipe.test(inp, **STEPS).cuda(), inp["video_data"].cuda()).cpu()
    got = check_windows(streamed(pipe, inp, uint8=False, **STEPS), 4, *inp["target_res"], dtype=torch.float32)
    assert torch.equal(got, want)


@pytest.mark.gpu
def test_iter_slow_consumer_and_early_stop(pipe):
    from star_b200.video_to_video.utils.seed import setup_seed
    inp = clip(7, (96, 160))
    want = whole_clip(pipe, inp, **STEPS)
    setup_seed(666)
    got = []
    for _, fr in pipe.enhance_frames_iter(inp, **STEPS):
        got.append(fr.clone())
        fr.fill_(255)                          # the caller owns the tensor
        time.sleep(0.5)                        # the next window is decoded meanwhile
    assert torch.equal(torch.cat(got), want)

    setup_seed(666)
    for s, fr in pipe.enhance_frames_iter(inp, **STEPS):
        assert s == 0 and torch.equal(fr, want[:3])
        break
    assert torch.cuda.current_stream().query(), "work left in flight after the consumer stopped"
    torch.cuda.synchronize()
    assert torch.equal(check_windows(streamed(pipe, inp, **STEPS), 7, *inp["target_res"]), want)


def peak_bytes(fn):
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


@pytest.mark.gpu
def test_iter_memory_does_not_grow_with_the_clip(pipe):
    """720x1280 canvas (LR 180x320, x4), one solver step, chunks of 6 frames so that every denoise window has the same
    shape: the peak's growth from 6 to 30 frames, per frame, against the clip-length fp32 latents the sampler keeps alive."""
    kw = dict(steps=1, solver_mode="normal", guide_scale=7.5, max_chunk_len=6)

    def run_iter(F):
        for _ in pipe.enhance_frames_iter(clip(F, (180, 320)), **kw):
            pass

    run_iter(6)                                # lazy weight packing and every window shape, outside the measurement
    grow = (peak_bytes(lambda: run_iter(30)) - peak_bytes(lambda: run_iter(6))) / 24
    whole = (peak_bytes(lambda: whole_clip(pipe, clip(30, (180, 320)), **kw))
             - peak_bytes(lambda: whole_clip(pipe, clip(6, (180, 320)), **kw))) / 24
    # Clip-length fp32 latents alive at once while denoise_latents / sample_sr / sample_dpmpp_2m_sde run: the encoded LR
    # latent (the hint), the diffused latent and the solver state x throughout; then either the chunks' x0 kept for the
    # stitch (up to 2: each kept slice is a view of its whole chunk's x0, and chunks overlap by half) and the stitched x0,
    # or the stitched x0, s_next * noise and the new x while the old x is still referenced.  k = 3 + 3.
    k = 6
    print(f"peak growth per frame: streamed {grow / 1e6:.3f} MB ({grow / LATENT_FRAME:.2f} latent frames), whole clip "
          f"{whole / 1e6:.2f} MB ({whole / LATENT_FRAME:.1f} latent frames)")
    assert k * LATENT_FRAME < DECODED_FRAME
    assert grow < k * LATENT_FRAME, f"streamed peak grows by {grow / 1e6:.3f} MB per frame"
    # the whole-clip composition keeps every decoded fp16 window until the last one is done: the bound tells the two apart
    assert whole > k * LATENT_FRAME, f"whole-clip peak grows by only {whole / 1e6:.3f} MB per frame"
