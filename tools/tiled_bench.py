#!/usr/bin/env python
"""Spatially tiled sampling on the FULL ControlledV2VUNet (synthetic weights): time of one solver step (one CFG-pair
evaluation per (chunk, tile) window + the solver update, CUDA events, after a warm-up of every model shape) and
torch.cuda.max_memory_allocated, untiled and with tiles of 90x160 latent pixels and an overlap of 16:

  122x216 (240p -> 960p), F = 32: untiled and tiled, and the rel-L2 between the two latents after the step (a number only:
                                  synthetic weights say nothing about visual quality)
  242x432 (480p -> 4x),   F = 32: tiled; untiled only if its peak, predicted from an untiled 90x160 run as linear in tokens,
                                  fits in 80 % of the free memory (otherwise skipped, not measured)
  362x648 (720p -> 4x),   F = 32: tiled only

and the pixel legs of a 720p -> 4x clip (2880x5120): time and peak memory of one frame's bilinear upsample + VAE encode and
of one 3-frame VAE decode window (untiled VAE, synthetic weights), each with the share of its op time spent in the VAE's
mid-block attention (a second, traced run), then enhance_frames(tile_size=(90, 160)) end to end on an 8-frame 720p clip with
one solver step (skipped when a pixel leg fails or, from decode_peak_bytes, would not fit in 90 % of the free memory).  --lr 1080x1920 runs the pixel legs and
enhance_frames of a 1080p -> 4x clip instead (4320x7680 on a 4368x7744 canvas; the decode window runs under a split plan).
python tools/tiled_bench.py [--frames 32] [--skip-e2e | --skip-latent] [--lr 1080x1920]"""
import argparse
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import build_model  # noqa: E402
from star_b200.lib import StarError  # noqa: E402
from tools.long_chunk_bench import card  # noqa: E402

GB = 1024 ** 3
TILE, OVERLAP = (90, 160), 16


def inputs(F, H, W, dev, seed=0):
    g = torch.Generator().manual_seed(seed)
    feat = 0.5 * torch.randn(1, 4, F, H, W, generator=g)
    y, ny = torch.randn(1, 77, 1024, generator=g), torch.randn(1, 77, 1024, generator=g)
    noise = torch.randn(feat.shape, generator=g).to(dev)
    return feat, y, ny, noise


def warm(net, F, H, W, dev):
    """one CFG-pair forward of the model shape a step uses: lazy init, weight packing, tensor maps"""
    x = torch.randn(1, 4, F, H, W, device=dev)
    y = torch.randn(1, 77, 1024, device=dev)
    out = net.forward_cfg_pair(x, torch.tensor([500], device=dev), (y, y), hint=x)
    del out, x
    torch.cuda.synchronize()


def step(pipe, F, H, W, dev, tile):
    """time and peak of one solver step of denoise_latents (the 'normal' plan with steps=1 is one evaluation)"""
    feat, y, ny, noise = inputs(F, H, W, dev)
    g = torch.Generator(device=dev).manual_seed(1)
    sampler = lambda a, b: torch.randn(feat.shape, device=dev, generator=g)       # noqa: E731
    kw = {} if tile is None else {"tile_size": tile, "tile_overlap": OVERLAP}
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(dev)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    z = pipe.denoise_latents(feat, y, ny, steps=1, solver_mode="normal", max_chunk_len=max(32, F), noise=noise,
                             noise_sampler=sampler, **kw)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b), torch.cuda.max_memory_allocated(dev), z


def n_tiles(H, W):
    from star_b200.video_to_video.video_to_video_model import make_tiles
    rows, cols, _, _ = make_tiles(H, W, TILE, OVERLAP)
    return len(rows) * len(cols)


def report(head, ms, peak, F, extra=""):
    print(f"{head}: {ms / 1e3:8.2f} s/step  ({F / ms * 1e3:6.2f} frames/s)  peak {peak / GB:6.1f} GiB{extra}", flush=True)


def latent_legs(pipe, net, F, dev):
    base = torch.cuda.memory_allocated(dev)
    # untiled 90x160 run: activation memory per token for the prediction of larger untiled shapes
    warm(net, F, *TILE, dev)
    ms, peak, _ = step(pipe, F, *TILE, dev, None)
    act_per_token = (peak - base) / (TILE[0] * TILE[1])
    report(f"latent  90x160 F={F} untiled", ms, peak, F)

    H, W = 122, 216
    warm(net, F, H, W, dev)
    ms, peak, z_full = step(pipe, F, H, W, dev, None)
    report(f"latent {H}x{W} F={F} untiled", ms, peak, F)
    ms, peak, z_tiled = step(pipe, F, H, W, dev, TILE)
    err = ((z_tiled - z_full).norm() / z_full.norm()).item()
    report(f"latent {H}x{W} F={F} tiled {TILE[0]}x{TILE[1]}/{OVERLAP} ({n_tiles(H, W)} tiles)", ms, peak, F,
           f"  rel-L2 vs untiled after one step {err:.3e}")
    del z_full, z_tiled

    for H, W in ((242, 432), (362, 648)):
        ms, peak, z = step(pipe, F, H, W, dev, TILE)
        assert torch.isfinite(z).all()
        del z
        report(f"latent {H}x{W} F={F} tiled {TILE[0]}x{TILE[1]}/{OVERLAP} ({n_tiles(H, W)} tiles)", ms, peak, F)
        if H == 242:
            torch.cuda.empty_cache()
            pred = base + act_per_token * H * W
            free = torch.cuda.mem_get_info(dev)[0]
            if pred - torch.cuda.memory_allocated(dev) > 0.8 * free:
                print(f"latent {H}x{W} F={F} untiled: skipped, predicted peak {pred / GB:6.1f} GiB exceeds 80 % of the free "
                      f"{free / GB:.1f} GiB (not measured)", flush=True)
                continue
            warm(net, F, H, W, dev)
            ms, peak, z = step(pipe, F, H, W, dev, None)
            del z
            report(f"latent {H}x{W} F={F} untiled", ms, peak, F, f"  (predicted {pred / GB:.1f} GiB)")
        else:
            print(f"latent {H}x{W} F={F} untiled: not run (predicted {(base + act_per_token * H * W) / GB:.0f} GiB)",
                  flush=True)
    torch.cuda.empty_cache()


def synth_vae(dev):
    from star_b200.utils.synth import synth_tensor
    from star_b200.video_to_video.modules.temporal_vae import AutoencoderKLTemporalDecoder
    with torch.device("meta"):
        vae = AutoencoderKLTemporalDecoder()
    vae.load_state_dict({k: synth_tensor(k, v.shape, 0, dev) for k, v in vae.state_dict().items()}, assign=True)
    return vae.eval().requires_grad_(False)


def timed(fn, dev):
    """fn()'s result, its time (CUDA events) and the peak memory allocated while it ran"""
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats(dev)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = fn()
    b.record()
    torch.cuda.synchronize()
    return out, a.elapsed_time(b), torch.cuda.max_memory_allocated(dev)


def attention_share(fn):
    """fn() traced op by op (ops.trace_begin / trace_end): (ms in the VAE's mid-block attention, ms in all ops)"""
    from star_b200 import ops
    from star_b200.video_to_video.modules.temporal_vae import AutoencoderKLTemporalDecoder as AE
    spans, orig = [], AE.__dict__["_attention"]

    def attention(a, x, n, HW):
        i0 = len(ops._trace)
        out = orig.__func__(a, x, n, HW)
        spans.append((i0, len(ops._trace)))
        return out
    AE._attention = staticmethod(attention)
    try:
        ops.trace_begin()
        fn()
        rec = ops.trace_end()
    finally:
        AE._attention = orig
    return sum(ms for i0, i1 in spans for _, _, ms in rec[i0:i1]), sum(ms for _, _, ms in rec)


def pixel_legs(pipe, dev, lr=(720, 1280), scale=4):
    from star_b200.video_to_video.video_to_video_model import pad_to_fit
    th, tw = lr[0] * scale, lr[1] * scale
    pad = pad_to_fit(th, tw)
    base = torch.cuda.memory_allocated(dev)
    frame = torch.rand(1, 3, *lr, device=dev) * 2 - 1
    encode = lambda: pipe.vae_encode(pipe.upsample_pad(frame, th, tw, pad).unsqueeze(0))   # noqa: E731  (no autocast, as _test_on_device)
    try:
        z, ms, peak = timed(encode, dev)
        att, tot = attention_share(encode)
        print(f"pixel {th}x{tw}: one frame bilinear x{scale} + VAE encode {ms / 1e3:.2f} s, peak {peak / GB:6.1f} GiB "
              f"(VAE weights and model resident {base / GB:.1f} GiB), latent {tuple(z.shape)}; traced: mid-block attention "
              f"{att / 1e3:.2f} of {tot / 1e3:.2f} s of op time ({100 * att / tot:.1f} %)", flush=True)
        del z
    except (torch.cuda.OutOfMemoryError, StarError) as e:
        print(f"pixel {th}x{tw}: one frame upsample + encode failed: {e}", flush=True)
        return False
    zl = torch.randn(1, 4, 3, (th + pad[2] + pad[3]) // 8, (tw + pad[0] + pad[1]) // 8, device=dev)
    from star_b200.video_to_video.modules.temporal_vae import decode_peak_bytes, decode_plan
    torch.cuda.empty_cache()
    need = decode_peak_bytes(decode_plan(3, 3, zl.shape[3], zl.shape[4]), 3, zl.shape[3], zl.shape[4])
    free, _ = torch.cuda.mem_get_info(dev)
    if need > 0.9 * free:
        print(f"pixel {th}x{tw}: one 3-frame decode window not run (predicted {need / GB:.1f} GiB, {free / GB:.1f} GiB free)",
              flush=True)
        return False

    def decode():
        with torch.autocast("cuda"):
            return pipe.vae_decode_chunk(zl, chunk_size=3)
    try:
        out, ms, peak = timed(decode, dev)
        shape = tuple(out.shape)
        del out
        att, tot = attention_share(decode)
        print(f"pixel {th}x{tw}: one 3-frame VAE decode window {ms / 1e3:.2f} s, peak {peak / GB:6.1f} GiB, output {shape}; "
              f"traced: mid-block attention {att / 1e3:.2f} of {tot / 1e3:.2f} s of op time ({100 * att / tot:.1f} %)", flush=True)
    except (torch.cuda.OutOfMemoryError, StarError) as e:
        print(f"pixel {th}x{tw}: one 3-frame decode window failed: {e}", flush=True)
        return False
    torch.cuda.empty_cache()
    return True


def end_to_end(pipe, dev, F=8, lr=(720, 1280), scale=4):
    g = torch.Generator().manual_seed(5)
    video = torch.rand(F, 3, *lr, generator=g) * 2 - 1
    y = torch.randn(1, 77, 1024, generator=g)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(dev)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    frames = pipe.enhance_frames({"video_data": video, "y": y, "target_res": (lr[0] * scale, lr[1] * scale)}, steps=1,
                                 solver_mode="normal", tile_size=TILE, tile_overlap=OVERLAP)
    b.record()
    torch.cuda.synchronize()
    print(f"enhance_frames {lr[0]}x{lr[1]} -> {lr[0] * scale}x{lr[1] * scale}, {F} frames, 1 step, tiles "
          f"{TILE[0]}x{TILE[1]}/{OVERLAP}: {a.elapsed_time(b) / 1e3:.1f} s, peak {torch.cuda.max_memory_allocated(dev) / GB:.1f} GiB, "
          f"output {tuple(frames.shape)} {frames.dtype}", flush=True)


@torch.no_grad()
def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=32)
    ap.add_argument("--skip-e2e", action="store_true", help="latent legs only")
    ap.add_argument("--skip-latent", action="store_true", help="pixel legs and enhance_frames only")
    ap.add_argument("--lr", default="720x1280", help="HxW of the low-resolution clip of the pixel legs and enhance_frames "
                    "(1080x1920: 4320x7680 outputs on a 4368x7744 canvas)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tiled_bench needs a CUDA device")
    from types import SimpleNamespace
    from star_b200.video_to_video.video_to_video_model import VideoToVideo_sr
    dev = torch.device("cuda", 0)
    card()
    net, _, _ = build_model(False, dev)
    ny = torch.zeros(1, 77, 1024)
    pipe = VideoToVideo_sr(SimpleNamespace(model_path=None), device=dev, text_encoder=lambda s: ny, vae=object(), generator=net)
    print(f"# full ControlledV2VUNet, synthetic fp16 weights {torch.cuda.memory_allocated(dev) / GB:.2f} GiB; one solver step "
          "per line", flush=True)
    if not args.skip_latent:
        latent_legs(pipe, net, args.frames, dev)
    if not args.skip_e2e:
        pipe.vae = synth_vae(dev)
        lr = tuple(int(v) for v in args.lr.split("x"))
        if pixel_legs(pipe, dev, lr):
            end_to_end(pipe, dev, lr=lr)


if __name__ == "__main__":
    main()
