#!/usr/bin/env python
"""One solver step of the full 42-layer CogVideoX-5B DiT (synthetic weights, bf16) on W ranks, laid out by
cogvideox_parallel (W = 1: one GPU; W = 2: the CFG pair; W = 2P: two CFG groups x P sequence ranks; other W: sequence
parallelism), at the 25- and 49-frame clips (7 and 13 latent frames of 30 x 45 patches).

    torchrun --nproc-per-node W tools/dit_sp_bench.py [--frames 25 49] [--steps 3] [--warmup 1]
    python tools/dit_sp_bench.py ...          (one GPU, no process group)

Per frame count it prints one JSON line (rank 0): the median / min step time over --steps timed steps (CUDA events, after
--warmup untimed ones), each rank's max_memory_allocated, the median per-step time each rank spent in the two all-to-alls
(events around the exchange calls, so it includes waiting for the slowest rank), and the GPU's name, SM clock and power
limit as nvidia-smi reads them in the same run.  With --frames 25 49 the clips alternate step by step (after all
warm-ups), so drift of the shared machine hits both alike."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,clocks.sm,clocks.max.sm,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()
    except (OSError, subprocess.SubprocessError) as e:
        return [f"nvidia-smi unavailable: {e}"]


def synthetic_dit(num_frames, device):
    """the 42-layer DiT with random weights drawn on the device (LoRA off: it is merged into the dense weights at packing
    and costs nothing at run time), packed; the fp32 parameters are released after packing"""
    from star_b200.cogvideox import DiffusionTransformer
    with torch.device(device):
        net = DiffusionTransformer(num_frames=num_frames, lora_r=0, dtype=torch.bfloat16)
    g = torch.Generator(device=device).manual_seed(0)
    for name, p in net.named_parameters():
        p.normal_(generator=g)
        if p.dim() >= 2:
            p.mul_(p[0].numel() ** -0.5)
        elif name.endswith("weight"):
            p.mul_(0.1).add_(1.0)
        else:
            p.mul_(0.02)
    net._pack()
    for p in net.parameters():
        p.data = p.data.new_empty(0)
    return net


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, nargs="+", default=[25, 49])
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    rank = dist.get_rank() if world > 1 else 0
    from star_b200.cogvideox import cogvideox_parallel
    from star_b200.cogvideox import parallel as par

    a2a = []                                                       # (start, end) events of the exchanges of the timed step
    real = par.SeqShard.all_to_all

    def timed_all_to_all(self, send, leg):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        out = real(self, send, leg)
        e.record()
        a2a.append((s, e))
        return out
    par.SeqShard.all_to_all = timed_all_to_all

    runs = {}
    for f in args.frames:
        net = synthetic_dit(f, dev)
        fn = cogvideox_parallel(net) if world > 1 else net
        T, h, w = net.frames, 2 * net.gh, 2 * net.gw
        g = torch.Generator(device=dev).manual_seed(1)
        xin = torch.randn(2, T, 32, h, w, generator=g, device=dev)
        ctx = torch.randn(2, 226, 4096, generator=g, device=dev).to(torch.bfloat16)
        ts = torch.full((2,), 500.0, device=dev)
        runs[f] = (net, fn, xin, ts, ctx)

    def step(f):
        _, fn, xin, ts, ctx = runs[f]
        a2a.clear()
        if world > 1:
            dist.barrier()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn(xin, timesteps=ts, context=ctx)
        e.record()
        torch.cuda.synchronize()
        return s.elapsed_time(e), sum(a.elapsed_time(b) for a, b in a2a)

    for f in args.frames:
        for _ in range(args.warmup):
            step(f)
    torch.cuda.reset_peak_memory_stats()
    times = {f: [] for f in args.frames}
    for _ in range(args.steps):
        for f in args.frames:                                      # alternating clips
            times[f].append(step(f))
    peak = torch.tensor([torch.cuda.max_memory_allocated()], device=dev, dtype=torch.float64)
    info = gpu_info()
    for f in args.frames:
        a2a_ms = torch.tensor([statistics.median(t[1] for t in times[f])], device=dev, dtype=torch.float64)
        peaks, a2as = [peak], [a2a_ms]
        if world > 1:
            peaks = [torch.empty_like(peak) for _ in range(world)]
            a2as = [torch.empty_like(a2a_ms) for _ in range(world)]
            dist.all_gather(peaks, peak)
            dist.all_gather(a2as, a2a_ms)
        step_ms = [t[0] for t in times[f]]
        if rank == 0:
            print(json.dumps({"workload": "cogvideox_dit_step", "frames": f, "ranks": world, "layers": 42,
                              "step_ms_median": round(statistics.median(step_ms), 2), "step_ms_min": round(min(step_ms), 2),
                              "steps": args.steps, "all_to_all_ms_median_per_rank": [round(a.item(), 2) for a in a2as],
                              "max_memory_allocated_GiB_per_rank": [round(p.item() / 2 ** 30, 2) for p in peaks],
                              "gpus": info}), flush=True)
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
