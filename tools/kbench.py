#!/usr/bin/env python
"""Kernel micro-benchmarks at the shapes of BASELINE config 2 (32 frames, latent 122x216).
CUDA events, 2 warm-up + N timed launches per shape; prints ms, TFLOP/s or GB/s and the fraction of the
measured peak (MEASURED_PEAKS.json), or of the H100 SXM data sheet (989 TFLOP/s dense fp16, 3.35 TB/s HBM3) where no
measured peak is present.  Usage: python tools/kbench.py [attention linear conv rowops tattn ...]"""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
if "--lib" in sys.argv:                       # A/B: a variant build of the library
    i = sys.argv.index("--lib")
    import star_b200.lib as _lib
    _lib.LIB_PATH = os.path.abspath(sys.argv[i + 1])
    del sys.argv[i:i + 2]
    print("# library:", _lib.LIB_PATH)
from star_b200 import ops as O  # noqa: E402

PEAK = {"tflops": 989.0, "gbs": 3350.0}                          # H100 SXM data sheet (700 W)
PEAK_SRC = ("data sheet", "data sheet")
p = os.path.join(ROOT, "MEASURED_PEAKS.json")
if os.path.isfile(p):
    d = json.load(open(p))
    PEAK = {"tflops": d["bf16_tflops"], "gbs": d["hbm_gbs"]}      # kernels timed alone: burst figures
    PEAK_SRC = ("measured burst", "measured copy")


def rnd(*shape, scale=1.0):
    return (torch.randn(*shape, device="cuda") * scale).half()


def timeit(fn, iters=5):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def report(name, ms, flops=None, bytes_=None):
    s = f"{name:58s} {ms:9.3f} ms"
    if flops:
        tf = flops / ms / 1e9
        s += f"  {tf:8.1f} TFLOP/s ({100 * tf / PEAK['tflops']:5.1f}% of {PEAK_SRC[0]})"
    if bytes_:
        gb = bytes_ / ms / 1e6
        s += f"  {gb:8.1f} GB/s ({100 * gb / PEAK['gbs']:5.1f}% of {PEAK_SRC[1]})"
    print(s, flush=True)


F, LEVELS = 32, [(122, 216, 320), (62, 108, 640), (32, 54, 1280), (17, 27, 1280)]


def bench_attention():
    for (H, W, C) in LEVELS[:3]:
        N, heads = H * W, C // 64
        qkv = rnd(F * N, 3 * C)
        fn = lambda: O.attention(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], F, heads, N, N, 1, 0.125)  # noqa: E731
        report(f"attention self  B*h={F * heads} N={N}", timeit(fn, 3), flops=4.0 * N * N * 64 * F * heads)
    H, W, C = LEVELS[0]
    N, heads = H * W, C // 64
    q, kv = rnd(F * N, C), rnd(77, 2 * C)
    fn = lambda: O.attention(q, kv[:, :C], kv[:, C:], F, heads, N, 77, F, 0.125)  # noqa: E731
    report(f"attention cross B*h={F * heads} Nq={N} Nk=77", timeit(fn), flops=4.0 * N * 77 * 64 * F * heads,
           bytes_=2 * F * N * C * 2)


def bench_linear():
    H, W, C = LEVELS[0]
    R = F * H * W
    for (K, N, flags, res, name) in [(320, 320, 0, True, "to_out/proj (K=N=320, +res)"), (320, 960, 0, False, "qkv (320->960)"),
                                     (320, 2560, 1, False, "FF in GEGLU (320->2x1280)"), (1280, 320, 0, True, "FF out (1280->320,+res)"),
                                     (512, 1536, 0, False, "init temporal qkv (512->1536)")]:
        a = rnd(R, K)
        w = rnd(N, K, scale=K ** -0.5)
        n_out = N // 2 if flags else N
        bias = rnd(N, scale=0.1)
        r = rnd(R, n_out) if res else None
        fn = lambda: O.linear(a, w, bias, r, None, 1, flags)  # noqa: E731
        report(f"linear L0 {name}", timeit(fn), flops=2.0 * R * K * N,
               bytes_=2.0 * (R * K + R * n_out * (2 if res else 1) + N * K))
    H, W, C = LEVELS[2]
    R = F * H * W
    a, w, bias = rnd(R, C), rnd(3 * C, C, scale=C ** -0.5), None
    report("linear L2 qkv (1280->3840)", timeit(lambda: O.linear(a, w)), flops=2.0 * R * C * 3 * C)
    H, W, C = LEVELS[1]
    R = F * H * W
    a = rnd(R, C)
    for (N, res, name) in [(C, True, "to_out (640->640,+res)"), (3 * C, False, "qkv (640->1920)")]:
        w, r = rnd(N, C, scale=C ** -0.5), (rnd(R, N) if res else None)
        report(f"linear L1 {name}", timeit(lambda: O.linear(a, w, None, r)), flops=2.0 * R * C * N)
    a4, w4, r4 = rnd(R, 4 * C), rnd(C, 4 * C, scale=(4 * C) ** -0.5), rnd(R, C)
    report("linear L1 FF out (2560->640,+res)", timeit(lambda: O.linear(a4, w4, None, r4)), flops=2.0 * R * 4 * C * C)
    del a4, w4, r4
    for lvl in (1, 2):
        H, W, C = LEVELS[lvl]
        R = F * H * W
        a, w, bias = rnd(R, C), rnd(8 * C, C, scale=C ** -0.5), rnd(8 * C, scale=0.1)
        report(f"linear L{lvl} FF in GEGLU ({C}->2x{4 * C})", timeit(lambda: O.linear(a, w, bias, None, None, 1, 1)),
               flops=2.0 * R * C * 8 * C)


def bench_conv():
    for (H, W, C) in LEVELS:
        x = rnd(F, H, W, C)
        w9 = rnd(C, 3, 3, C, scale=(9 * C) ** -0.5)
        bias = rnd(C, scale=0.1)
        report(f"conv2d 3x3 {C}->{C} @ {H}x{W}", timeit(lambda: O.conv2d_3x3(x, w9, bias), 3), flops=2.0 * F * H * W * 9 * C * C)
        xt = x.view(F * H * W, C)
        w3 = rnd(C, 3, C, scale=(3 * C) ** -0.5)
        report(f"conv_t3 {C}->{C} @ {H}x{W}", timeit(lambda: O.conv_t3(xt, w3, bias, xt, 1, F, H * W), 3),
               flops=2.0 * F * H * W * 3 * C * C)


def bench_rowops():
    H, W, C = LEVELS[0]
    R = F * H * W
    x = rnd(R, C)
    g, b = rnd(C), rnd(C)
    report("groupnorm 4-D (per frame) + SiLU, C=320", timeit(lambda: O.groupnorm(x, g, b, F, 1e-5, True)), bytes_=3.0 * R * C * 2)
    report("groupnorm 5-D (per clip) + SiLU, C=320", timeit(lambda: O.groupnorm(x, g, b, 1, 1e-5, True)), bytes_=3.0 * R * C * 2)
    report("layernorm C=320", timeit(lambda: O.layernorm(x, g, b)), bytes_=2.0 * R * C * 2)
    report("layernorm + temporal LIEM C=320", timeit(lambda: O.layernorm(x, g, b, 2, None, 0.3, -0.2)), bytes_=2.0 * R * C * 2)
    w98 = rnd(98, scale=0.2)
    report("liem spatial gate C=320", timeit(lambda: O.liem_spatial_gate(x, w98, F, H, W)), bytes_=1.0 * R * C * 2)
    qkv = rnd(R, 3 * C)
    report("temporal attention T=32 heads=5", timeit(lambda: O.temporal_attention(qkv, 1, F, H * W, 5, C)),
           flops=4.0 * H * W * 5 * F * F * 64, bytes_=4.0 * R * C * 2)
    a, bb = rnd(R, 320), rnd(R, 320)
    report("concat_add 320|320", timeit(lambda: O.concat_add(a, bb, bb)), bytes_=5.0 * R * 320 * 2)


def bench_tattn():
    """Temporal attention at level 0 of a 960p latent (26 352 pixels, 5 heads, Ci 320) over T frames: T <= 64 runs
    temporal_attn2_kernel (tattn2.cuh), T > 64 temporal_attn_long_kernel (tattn_long.cuh).  Bytes = QKV read + O write,
    FLOP = 4 T^2 64 per (pixel, head); the floor is the larger of bytes / peak bandwidth and FLOP / peak rate."""
    HW, heads, C = 26352, 5, 320
    for T in (32, 64, 65, 78, 128):
        qkv = rnd(T * HW, 3 * C)
        flops, bytes_ = 4.0 * T * T * 64 * HW * heads, 4.0 * T * HW * C * 2
        ms = timeit(lambda: O.temporal_attention(qkv, 1, T, HW, heads, C), 20)
        t_hbm, t_mma = bytes_ / (PEAK["gbs"] * 1e6), flops / (PEAK["tflops"] * 1e9)
        report(f"temporal attention L0 T={T} HW={HW} heads={heads}", ms, flops=flops, bytes_=bytes_)
        print(f"{'':58s} floor {max(t_hbm, t_mma):.3f} ms ({'HBM' if t_hbm >= t_mma else 'MMA'}-bound), "
              f"achieved {100 * max(t_hbm, t_mma) / ms:5.1f}% of it", flush=True)
        del qkv


def bench_softmax():
    """Row softmax of the temporal VAE's mid-block attention: rows of one frame's logits, a row spread over a cluster of
    ceil(cols / 102 400) CTAs.  234 576 columns = a 720p -> 4x frame (362x648 latent), 528 528 = 1080p -> 4x (542x976).
    Bytes = the logits read once and written once (2 x rows x ld x 2 B)."""
    for cols in (26352, 102400, 234576, 528528):
        ld = (cols + 7) // 8 * 8
        rows = max(128, (1 << 28) // ld // 128 * 128)                   # temporal_vae._attention's row block
        n = -(-cols // 102400)
        s = rnd(rows, ld, scale=3.0)
        report(f"softmax_rows {rows}x{cols}, {n} CTA(s) per row", timeit(lambda: O.softmax_rows(s, cols, n), 20),
               bytes_=2.0 * rows * ld * 2)
        del s


def card():
    import subprocess
    try:
        o = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=10).stdout.strip()
        print(f"# card: {o}", flush=True)
    except Exception as e:
        print("# nvidia-smi failed", e)


def clocks():
    import subprocess
    try:
        o = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,clocks.max.sm,power.draw,temperature.gpu,clocks_event_reasons.active",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=10).stdout.strip()
        print(f"# nvidia-smi (idle, after group): {o}", flush=True)
    except Exception as e:
        print("# nvidia-smi failed", e)


if __name__ == "__main__":
    which = sys.argv[1:] or ["attention", "linear", "conv", "rowops"]
    card()
    print(f"# peaks used: {PEAK} ({PEAK_SRC[0]} / {PEAK_SRC[1]})")
    for w in which:
        globals()["bench_" + w]()
        clocks()
