#!/usr/bin/env python
"""Time and peak memory of one CFG-pair forward of the FULL ControlledV2VUNet (the model work of one solver step) for
chunks of F frames, F in {32, 64, 78, 128}, at latents 90x160 (720p) and 122x216 (960p).  Chunks over 64 frames run
the T > 64 temporal-attention kernel.

Peak memory is torch.cuda.max_memory_allocated over the forward.  Activations grow linearly in F, so each latent's F = 32
run predicts the peak at larger F (weights + activations(32) * F / 32); a shape predicted not to fit in the free device
memory is skipped and reported with its prediction, never attempted.  python tools/long_chunk_bench.py"""
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import build_model  # noqa: E402

FRAMES = (32, 64, 78, 128)
LATENTS = ((90, 160), (122, 216))
GB = 1024 ** 3


def card():
    try:
        o = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=10).stdout.strip()
    except Exception as e:
        o = f"nvidia-smi failed: {e}"
    print(f"# card: {o}", flush=True)


def run(net, F, H, W, dev, iters=2):
    gen = torch.Generator().manual_seed(0)
    x = torch.randn(1, 4, F, H, W, generator=gen).to(dev)
    hint = torch.randn(1, 4, F, H, W, generator=gen).to(dev)
    y, ny = torch.randn(1, 77, 1024, generator=gen).to(dev), torch.randn(1, 77, 1024, generator=gen).to(dev)
    t = torch.tensor([500], device=dev)
    out = net.forward_cfg_pair(x, t, (y, ny), hint=hint)         # warm-up
    del out
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(dev)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        out = net.forward_cfg_pair(x, t, (y, ny), hint=hint)
        del out
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters, torch.cuda.max_memory_allocated(dev)


@torch.no_grad()
def main():
    if not torch.cuda.is_available():
        raise SystemExit("long_chunk_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    card()
    net, _, _ = build_model(False, dev)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated(dev)
    print(f"# full ControlledV2VUNet (2.04 B params), fp16 weights {base / GB:.2f} GiB; one CFG-pair forward per line", flush=True)
    for (H, W) in LATENTS:
        act32 = None
        for F in FRAMES:
            torch.cuda.empty_cache()
            free = torch.cuda.mem_get_info(dev)[0]
            pred = None if act32 is None else base + act32 * F / 32
            head = f"latent {H:3d}x{W:3d} F={F:3d}"
            # 20 % headroom: the caching allocator fragments (an 8 GiB GEGLU output found 29 GiB reserved but unusable)
            if pred is not None and pred - torch.cuda.memory_allocated(dev) > 0.8 * free:
                print(f"{head}: skipped, predicted peak {pred / GB:6.1f} GiB exceeds 80 % of the free {free / GB:.1f} GiB "
                      "(not measured)", flush=True)
                continue
            ms, peak = run(net, F, H, W, dev)
            if act32 is None:
                act32 = peak - base
            line = f"{head}: {ms:9.1f} ms  ({F / ms * 1e3:6.2f} frames/s)  peak {peak / GB:6.1f} GiB"
            if pred is not None:
                line += f"  (predicted {pred / GB:6.1f} GiB)"
            print(line, flush=True)


if __name__ == "__main__":
    main()
