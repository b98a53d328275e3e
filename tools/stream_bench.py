#!/usr/bin/env python
"""Clips of any length: wall time and torch.cuda.max_memory_allocated of the two single-GPU ways to get enhanced frames,
per clip length, on the full ControlledV2VUNet and the full temporal VAE (synthetic weights), one solver step:

  streamed    VideoToVideo_sr.enhance_frames_iter, every window consumed (the frames are dropped)
  whole clip  _test_on_device + ops.adain_color_fix over the whole clip + one copy to the host (test() + the colour fix,
              which multi-rank enhance_frames equals byte for byte)

  240p -> 960p (LR 240x426, canvas 976x1728), F = 32, 96, 288
  480p -> 4x   (LR 480x854, canvas 1936x3456), tiles of 90x160 latent pixels, F = 32, 96

Each workload first runs both paths on clips of 3 and 6 frames (the first of them also loads every kernel); these two
lengths are only the first points of the peak prediction.  Every longer run is predicted from the path's two longest runs
so far (the peak is linear in F) and skipped, printed as "skipped, not measured", when the prediction exceeds 80 % of the
free device memory.  The smallest listed F runs twice per path, alternating, for a run-to-run spread.
python tools/stream_bench.py [--only 960p|480p4x]"""
import argparse
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import build_model  # noqa: E402
from tools.long_chunk_bench import card  # noqa: E402
from tools.tiled_bench import synth_vae  # noqa: E402

GB, MB = 1024 ** 3, 1e6
WORKLOADS = {
    "960p": dict(lr=(240, 426), frames=(32, 96, 288), tile=None),
    "480p4x": dict(lr=(480, 854), frames=(32, 96), tile=(90, 160)),
}
CALIBRATION = (3, 6)
KW = dict(total_noise_levels=1000, steps=1, solver_mode="normal", guide_scale=7.5, max_chunk_len=32)


def clip(F, lr, seed=5):
    g = torch.Generator().manual_seed(seed)
    video = torch.rand(F, 3, *lr, generator=g) * 2 - 1
    return {"video_data": video, "y": torch.randn(1, 77, 1024, generator=g), "target_res": (4 * lr[0], 4 * lr[1])}


def streamed(pipe, inp, tile):
    n = 0
    for _, frames in pipe.enhance_frames_iter(inp, tile_size=tile, **KW):
        n += frames.shape[0]
    return n


def whole_clip(pipe, inp, tile):
    from star_b200 import ops
    vid = pipe._test_on_device(inp, tile_size=tile, **KW).float()
    return ops.adain_color_fix(vid, inp["video_data"].to(vid.device).float(), uint8=True).cpu().shape[0]


PATHS = {"streamed": streamed, "whole clip": whole_clip}


def predict(runs, F):
    """peak at F from earlier (F, peak) runs: the largest measured at F, else the line through the two longest shorter runs"""
    if any(f == F for f, _ in runs):
        return max(p for f, p in runs if f == F)
    shorter = {f: p for f, p in sorted(runs) if f < F}
    if len(shorter) < 2:
        return None
    (f0, p0), (f1, p1) = sorted(shorter.items())[-2:]
    return p1 + (p1 - p0) * (F - f1) / (f1 - f0)


def measure(fn, pipe, inp, tile):
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    n = fn(pipe, inp, tile)
    torch.cuda.synchronize()
    return time.perf_counter() - t0, torch.cuda.max_memory_allocated(), n


def workload(pipe, name, lr, frames, tile):
    from star_b200.video_to_video.video_to_video_model import pad_to_fit
    H, W = 4 * lr[0], 4 * lr[1]
    pad = pad_to_fit(H, W)
    latent_frame = 4 * ((H + pad[2] + pad[3]) // 8) * ((W + pad[0] + pad[1]) // 8) * 4
    head = f"{name} {lr[0]}x{lr[1]} -> {H}x{W}" + ("" if tile is None else f", tiles {tile[0]}x{tile[1]}")
    print(f"# {head}: one fp32 latent frame {latent_frame / MB:.2f} MB", flush=True)
    runs = {p: [] for p in PATHS}
    order = [(F, p) for F in CALIBRATION + frames for p in PATHS] + [(frames[0], p) for p in PATHS]
    for F, p in order:
        pred = predict(runs[p], F)
        assert pred is not None or F in CALIBRATION
        torch.cuda.empty_cache()
        free = torch.cuda.mem_get_info()[0]
        if pred is not None and pred - torch.cuda.memory_allocated() > 0.8 * free:
            print(f"{head}, F={F}, {p}: skipped, not measured (predicted peak {pred / GB:.1f} GiB, free {free / GB:.1f} GiB)",
                  flush=True)
            continue
        sec, peak, n = measure(PATHS[p], pipe, clip(F, lr), tile)
        assert n == F
        runs[p].append((F, peak))
        print(f"{head}, F={F}, {p}: {sec:8.1f} s ({sec / F:.3f} s/frame), peak {peak / GB:6.2f} GiB", flush=True)
    for p, r in runs.items():
        r = [(F, peak) for F, peak in r if F not in CALIBRATION]
        if len({F for F, _ in r}) > 1:
            (f0, p0), (f1, p1) = min(r), max(r)
            growth = (p1 - p0) / (f1 - f0)
            print(f"{head}, {p}: peak growth {growth / MB:.2f} MB per frame ({growth / latent_frame:.1f} latent frames) "
                  f"from F={f0} to F={f1}", flush=True)


@torch.no_grad()
def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", choices=list(WORKLOADS))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("stream_bench needs a CUDA device")
    from types import SimpleNamespace
    from star_b200.video_to_video.video_to_video_model import VideoToVideo_sr
    dev = torch.device("cuda", 0)
    card()
    net, _, _ = build_model(False, dev)
    ny = torch.zeros(1, 77, 1024)
    pipe = VideoToVideo_sr(SimpleNamespace(model_path=None), device=dev, text_encoder=lambda s: ny, vae=synth_vae(dev),
                           generator=net)
    print(f"# full ControlledV2VUNet + temporal VAE, synthetic weights, {torch.cuda.memory_allocated(dev) / GB:.2f} GiB "
          "resident; one solver step", flush=True)
    for name, w in WORKLOADS.items():
        if args.only in (None, name):
            workload(pipe, name, **w)


if __name__ == "__main__":
    main()
