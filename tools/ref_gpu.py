#!/usr/bin/env python
"""The UNMODIFIED reference modules on the GPU, beside star_b200, on identical weights and inputs.

What the north-star's ">= 8x the reference's single-GPU PyTorch frames/sec" and "within 1e-3 relative fp16
tolerance" are written against (BASELINE.md 3/4, SURVEY 8d, VERDICT r1 items 1-2):

  * reference fp16 : ControlledV2VUNet().half() under torch.autocast('cuda', fp16), exactly as
                     video_to_video_model.py:42,98 runs it; xformers.memory_efficient_attention is shimmed to
                     F.scaled_dot_product_attention (xformers is not installed) -- timed.
  * reference fp32 : the same modules in fp32 with TF32 OFF (cudnn + matmul) and an exact chunked fp32
                     attention in place of the fused kernel -- the oracle both fp16 paths are measured against.
  * star_b200      : this repo's forward through the C ABI -- timed, compared with both.

Needs the reference tree: /root/reference (build container) or oracle/_ref (python -m oracle.stage_reference).
TEST / BASELINE INFRASTRUCTURE: nothing in star_b200/ imports this.

  python tools/ref_gpu.py --shape 32,122,216 --out gpurun_out/ref_gpu_c2.json
"""
import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def rel_l2(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def max_rel(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max())


def event_ms(fn, warm, iters):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return out, ts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shape", default="32,122,216", help="frames,latentH,latentW")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--weight-seed", type=int, default=2)
    ap.add_argument("--t", type=int, default=899)
    ap.add_argument("--small", action="store_true")
    ap.add_argument("--no-fp32", action="store_true")
    ap.add_argument("--no-star", action="store_true", help="time the reference only (bench.py's gpu_reference block)")
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    F, H, W = (int(v) for v in args.shape.split(","))
    dev = torch.device("cuda", 0)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.set_float32_matmul_precision("highest")

    from oracle import ref_loader as R
    from star_b200.utils.synth import synth_state_dict
    from tests.util import SMALL_KW, make_inputs
    kw = SMALL_KW if args.small else {}
    ns = R.load_reference()
    U = ns.unet
    import logging
    logging.getLogger("video_to_video").setLevel(logging.ERROR)

    with torch.device("meta"):
        ref = U.ControlledV2VUNet.__new__(U.ControlledV2VUNet)
        U.Vid2VidSDUNet.__init__(ref, **kw)
        ref.VideoControlNet = U.VideoControlNet(**kw)
    manifest = {k: tuple(v.shape) for k, v in ref.state_dict().items()}
    t0 = time.time()
    sd = synth_state_dict(manifest, seed=args.weight_seed, device=dev)
    ref.load_state_dict(sd, assign=True)
    ref.eval().requires_grad_(False)
    print(f"weights: {sum(v.numel() for v in sd.values()) / 1e9:.3f} B parameters in {time.time() - t0:.1f} s", flush=True)

    x, hint, y = make_inputs(args.seed, 1, F, H, W)
    x, hint, y = x.to(dev), hint.to(dev), y.to(dev)
    t = torch.tensor([args.t], device=dev)
    res = {"shape": {"frames": F, "latent_h": H, "latent_w": W}, "t": args.t, "weight_seed": args.weight_seed,
           "input_seed": args.seed, "model": "reduced" if args.small else "ControlledV2VUNet() 2.04 B params, synthetic non-zero weights",
           "gpu": torch.cuda.get_device_name(0), "torch": torch.__version__,
           "attention_shim": "xformers.ops.memory_efficient_attention -> F.scaled_dot_product_attention (fp16) / exact chunked fp32 math (fp32 oracle)",
           "tf32": "off (cudnn.allow_tf32 = cuda.matmul.allow_tf32 = False)"}

    # ---- star_b200 ---------------------------------------------------------------------------------------------
    o_star, ts = None, None
    if not args.no_star:
        from star_b200.video_to_video.modules.unet_v2v import ControlledV2VUNet
        with torch.device("meta"):
            net = ControlledV2VUNet(**kw)
        net.load_state_dict({k: v.to(torch.float16) for k, v in sd.items()}, assign=True)
        net.eval()
        with torch.no_grad():
            o_star, ts = event_ms(lambda: net(x, t, y, hint=hint), 1, args.iters)
        o_star = o_star.float()
        res["star_ms_per_forward"] = ts
        res["star_finite"] = bool(torch.isfinite(o_star).all())
        print(f"star_b200: {min(ts):.1f} ms / forward (min of {ts})", flush=True)
        del net
        torch.cuda.empty_cache()

    # ---- reference fp32 (oracle; TF32 off, exact attention) ---------------------------------------------------------
    o32 = None
    if not args.no_fp32:
        torch.cuda.reset_peak_memory_stats()
        with torch.no_grad():
            a = time.time()
            o32 = ref(x, t, y, hint=hint).float()
            torch.cuda.synchronize()
        res["ref_fp32_s_per_forward"] = time.time() - a
        res["ref_fp32_peak_gb"] = torch.cuda.max_memory_allocated() / 1e9
        print(f"reference fp32: {res['ref_fp32_s_per_forward']:.1f} s, peak {res['ref_fp32_peak_gb']:.1f} GB", flush=True)
        torch.cuda.empty_cache()

    # ---- reference fp16 autocast, the way the reference runs it ---------------------------------------------------
    refh = ref.half()
    torch.cuda.reset_peak_memory_stats()

    def ref16():
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16):
            return refh(x, t, y, hint=hint)
    o16, ts16 = event_ms(ref16, 1, args.iters)
    o16 = o16.float()
    res["ref_fp16_ms_per_forward"] = ts16
    res["ref_fp16_peak_gb"] = torch.cuda.max_memory_allocated() / 1e9
    print(f"reference fp16 autocast: {min(ts16):.1f} ms / forward (min of {ts16}), peak {res['ref_fp16_peak_gb']:.1f} GB", flush=True)

    res["frames_per_s_50step_cfg2"] = {"reference_fp16": F / (100 * min(ts16) / 1e3)}
    res["rel_l2"], res["max_abs_over_max"] = {}, {}
    if o32 is not None:
        res["rel_l2"]["ref_fp16_vs_ref_fp32"] = rel_l2(o16, o32)
        res["max_abs_over_max"]["ref_fp16_vs_ref_fp32"] = max_rel(o16, o32)
    if o_star is not None:
        res["speedup_star_vs_ref_fp16"] = min(ts16) / min(ts)
        res["frames_per_s_50step_cfg2"]["star"] = F / (100 * min(ts) / 1e3)
        res["rel_l2"]["star_vs_ref_fp16"] = rel_l2(o_star, o16)
        res["max_abs_over_max"]["star_vs_ref_fp16"] = max_rel(o_star, o16)
        res["out_checksum"] = {"star_sum": float(o_star.double().sum()), "star_abs_mean": float(o_star.abs().mean())}
    if o32 is not None and o_star is not None:
        res["rel_l2"]["star_vs_ref_fp32"] = rel_l2(o_star, o32)
        res["max_abs_over_max"]["star_vs_ref_fp32"] = max_rel(o_star, o32)
        # per-frame error of the star output (a >2^31-element indexing bug would show up as a bad frame range)
        pf = [(rel_l2(o_star[:, :, f], o32[:, :, f])) for f in range(F)]
        res["star_vs_ref_fp32_per_frame_minmax"] = [min(pf), max(pf)]
    print(json.dumps(res), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        json.dump(res, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
