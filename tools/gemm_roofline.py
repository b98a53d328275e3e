#!/usr/bin/env python
"""Per-shape roofline of the tap-GEMM calls of one solver step (32 frames, latent 122x216, 2 CFG forwards).

One bench-shape step is run with `ops.trace_begin()/trace_end()` and every conv / linear call is recorded with its
geometry.  Each distinct shape is then launched alone (CUDA events, warmed up, enough launches for >= 60 ms of work) and
set against its two floors: algorithmic HBM bytes / 3.35 TB/s and FLOP / 989 TFLOP/s (H100 SXM data sheet).  "fill" is what the TMA producer writes to
shared memory under the tiling in use, per SM clock and SM, at the SM clock sampled during the run.  A synthetic sweep runs
the level-0 3x3 conv at N = 256, 320 and 384 so that the 256-, 160- and 128-wide kernels see the same M and K.

The geometry, tiling and byte / FLOP arithmetic (`shape_of_call`, `model`) need no GPU; the measurements do and the script
fails without one.  Usage: python tools/gemm_roofline.py [--lib libstar_sm100.so] [--json out.json] [--no-step]"""
import argparse
import inspect
import json
import math
import os
import sys
from collections import namedtuple

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

PEAK_TFLOPS, PEAK_HBM_GBS = 989.0, 3350.0        # H100 SXM data sheet: dense fp16, HBM3 (700 W card)
NUM_SMS = 132
GEMM_OPS = ("linear", "linear_ex", "conv2d_3x3", "conv2d_3x3_s2", "conv2d_3x3_s2p", "conv_t3", "conv3d_causal")

# op, geometry (sorted (key, value) pairs), flags, epilogue inputs present
Shape = namedtuple("Shape", "op dims flags epi")


def _ceil(a, b):
    return -(-a // b)


# ---- dispatch, restated from star_abi.cu (the one Python copy: tests/test_kernel_bounds_gpu.py plans its cases with it) ----
def tile_width(n, geglu):
    """launch_tapgemm: the tile width that pads N least, the wider on a tie (GEGLU: 64 or 128 value columns)"""
    pad = lambda w: _ceil(n, w) * w                                              # noqa: E731
    if geglu:
        return 256 if pad(128) <= pad(64) else 128
    if pad(256) <= pad(128) and pad(256) <= pad(160):
        return 256
    return 160 if pad(160) <= pad(128) else 128


# epilogue instances (tapgemm.cuh: TapGemmEpi, TG_EPI_KINDS, tg_epi_kind): a call runs the instance compiled for exactly its
# epilogue kind, else the generic one that reads every option at run time
EPI_BITS = {"bias": 1, "geglu": 2, "rowvec": 4, "colscale": 8, "residual": 16, "erf": 32, "tanh": 64, "silu": 128}
EPI_GENERIC = 256
EPI_INSTANCES = (0, 1, 1 | 16, 1 | 4, 1 | 2, 1 | 128, 1 | 32, 1 | 64, 1 | 8 | 16)


def epi_kind(flags, epi):
    """tg_epi_kind: the epilogue kind of a call from its flags and the epilogue inputs it passes"""
    names = set(epi) | {n for bit, n in ((1, "geglu"), (2, "silu"), (4, "erf"), (8, "tanh")) if flags & bit}
    return sum(EPI_BITS[n] for n in names)


def epi_instance(flags, epi):
    """the epilogue instance a call runs: its own kind's, or EPI_GENERIC"""
    k = epi_kind(flags, epi)
    return k if k in EPI_INSTANCES else EPI_GENERIC


# epilogue path (star_abi.cu: launch_tapgemm, tma_addressable): the staged epilogue, which stores the output and loads the
# residual through TMA, runs when TMA can address both: a 16-byte-aligned base, and a row pitch and N that are multiples
# of 8 elements.  Other calls take the direct epilogue, which stores from registers.
def tma_addressable(offset_bytes, ld, n):
    """offset_bytes: of the view's first element from a 16-byte-aligned allocation (torch's CUDA allocator aligns to 512 B)"""
    return offset_bytes % 16 == 0 and ld % 8 == 0 and n % 8 == 0


def staged_epilogue(n, out_offset_bytes, out_ld, res_offset_bytes=None, res_ld=None):
    """whether a call with N = n columns runs the staged epilogue (no residual: res_ld None)"""
    return tma_addressable(out_offset_bytes, out_ld, n) and (res_ld is None or tma_addressable(res_offset_bytes, res_ld, n))


def call_epilogue_views(name, fn, args, kwargs):
    """(N, (offset bytes, ld) of the output, the same of the residual or None) of one ops.<name> call, as the library sees
    them; None for a call the wrapper refuses (a view whose columns are not contiguous)"""
    b = inspect.signature(fn).bind(*args, **kwargs)
    b.apply_defaults()
    a = b.arguments

    def view(t, cols):
        if t is None:                                    # allocated by the wrapper: [rows, cols], contiguous
            return 0, cols
        if t.dim() != 2 or t.stride(1) != 1:             # refused by the wrapper (ops._rowmajor): no launch
            return None
        return t.storage_offset() * t.element_size(), t.stride(0)
    flags = int(a.get("flags", 0) or 0)
    if name in ("linear", "linear_ex"):
        n = a["w"].shape[0] // (2 if flags & 1 else 1)
    else:
        n = a[{"conv_t3": "w3", "conv3d_causal": "w27"}.get(name, "w9")].shape[0]
    out = view(a.get("out"), n)
    res = view(a["residual"], n) if a.get("residual") is not None else None
    if out is None or (res is None and a.get("residual") is not None):
        return None
    if name == "conv_t3" and a.get("band") is not None:  # star_conv_t3 offsets out / residual to the band's first pixel
        p0 = int(a["band"][0])
        out = (out[0] + p0 * out[1] * 2, out[1])
        res = None if res is None else (res[0] + p0 * res[1] * 2, res[1])
    return n, out, res


def best_box_2d(h, w):
    """conv_box: the (h, w) box of at most 128 pixels that covers h x w in the fewest tiles, the wider on a tie"""
    best, th, tw = -1, 1, 1
    for bw in range(1, min(w, 128) + 1):
        bh = min(h, 128 // bw)
        if bh < 1:
            continue
        t = _ceil(w, bw) * _ceil(h, bh)
        if best < 0 or t < best or (t == best and bw > tw):
            best, th, tw = t, bh, bw
    return th, tw


def geometry(op, d):
    """(output extents on[4], box[4], taps, K, N, input rows) of one entry point, as it fills TapGemmParams.  conv2d_3x3 with
    d["rows"] = (row0, n): output rows row0..row0+n of every frame, boxed over n rows (the whole frames are the input);
    conv_t3 with d["band"] = (p0, p1): pixels p0..p1 of every frame.  Input rows are those of the whole clip, B T HW, also for
    a band, whose call reads the band's B T (p1 - p0) of them, compactly (band_input_rows)."""
    if op in ("linear", "linear_ex"):
        return (d["rows"], 1, 1, 1), (128, 1, 1, 1), 1, d["K"], d["N"], d["rows"]
    if op == "conv2d_3x3":
        ho = d["rows"][1] if d.get("rows") is not None else d["H"]
        th, tw = best_box_2d(ho, d["W"])
        return ((d["W"], ho, d["BT"], 1), (tw, th, max(1, min(d["BT"], 128 // (tw * th))), 1), 9, d["Cin"], d["Cout"],
                d["BT"] * d["H"] * d["W"])
    if op in ("conv2d_3x3_s2", "conv2d_3x3_s2p"):
        pt, pb, pl, pr = d.get("pad", (2, 2, 1, 1))
        ho, wo = (d["H"] + pt + pb - 3) // 2 + 1, (d["W"] + pl + pr - 3) // 2 + 1
        th, tw = best_box_2d(ho, wo)
        return (wo, ho, 1, d["BT"]), (tw, th, 1, 1), 9, d["Cin"], d["Cout"], d["BT"] * d["H"] * d["W"]
    if op == "conv_t3":
        t = d["T"]
        hw = d["band"][1] - d["band"][0] if d.get("band") is not None else d["HW"]
        return ((hw, t, d["B"], 1), (min(128, hw), min(t, 128 // hw) if hw < 128 else 1, 1, 1), 3, d["Cin"], d["Cout"],
                d["B"] * t * d["HW"])
    if op == "conv3d_causal":
        th, tw = best_box_2d(d["H"], d["W"])
        return ((d["W"], d["H"], d["T"], 1), (tw, th, max(1, min(d["T"], 128 // (tw * th))), 1), 27, d["Cin"], d["Cout"],
                (d["T"] + 2) * d["H"] * d["W"])
    raise ValueError(op)


def band_input_rows(op, d):
    """rows of the A operand one call reads: a conv_t3 band is passed compactly ([B T (p1 - p0), Cin]), other calls read
    geometry()'s input rows"""
    on, _, _, _, _, rows_in = geometry(op, d)
    return math.prod(on) if op == "conv_t3" else rows_in


def m_tiles(on, box):
    """M tiles: one box of at most 128 rows each"""
    return math.prod(_ceil(o, b) for o, b in zip(on, box))


# ---- from a recorded call to a shape -----------------------------------------------------------------------------------------
def shape_of_call(name, fn, args, kwargs):
    """Shape of one ops.<name>(*args, **kwargs) call (tensors need only .shape), or None if it is not a tap-GEMM"""
    if name not in GEMM_OPS:
        return None
    b = inspect.signature(fn).bind(*args, **kwargs)
    b.apply_defaults()
    a = b.arguments
    has = lambda k: a.get(k) is not None                                         # noqa: E731
    flags = int(a.get("flags", 0) or 0)
    if name in ("linear", "linear_ex"):
        rows, K = a["a"].shape
        nw = a["w"].shape[0]
        d = {"rows": int(rows), "K": int(K), "N": int(nw // 2 if flags & 1 else nw)}
        if has("rowvec"):
            d["rv_div"] = int(a["rowvec_div"])
    elif name in ("conv2d_3x3", "conv2d_3x3_s2", "conv2d_3x3_s2p"):
        BT, H, W, Cin = a["x"].shape
        d = {"BT": int(BT), "H": int(H), "W": int(W), "Cin": int(Cin), "Cout": int(a["w9"].shape[0])}
        if name == "conv2d_3x3_s2p":
            d["pad"] = tuple(int(v) for v in a["pad"])
        if name == "conv2d_3x3" and has("rows"):
            d["rows"] = tuple(int(v) for v in a["rows"])
        if has("rowvec"):
            d["rv_div"] = int(a["rowvec_div"])
    elif name == "conv_t3":
        d = {"B": int(a["B"]), "T": int(a["T"]), "HW": int(a["HW"]), "Cin": int(a["x"].shape[1]), "Cout": int(a["w3"].shape[0])}
        if has("band"):
            d["band"] = tuple(int(v) for v in a["band"])
    else:
        d = {"T": int(a["T"]), "H": int(a["H"]), "W": int(a["W"]), "Cin": int(a["xp"].shape[1]), "Cout": int(a["w27"].shape[0])}
    epi = tuple(k for k in ("bias", "rowvec", "colscale", "residual") if has(k))
    return Shape(name, tuple(sorted(d.items())), flags, epi)


def enumerate_calls(calls, ops_module):
    """[(name, args, kwargs)] -> {Shape: calls}, insertion-ordered"""
    out = {}
    for name, args, kwargs in calls:
        s = shape_of_call(name, getattr(ops_module, name), args, kwargs)
        if s is not None:
            out[s] = out.get(s, 0) + 1
    return out


# ---- bytes, FLOP, floors -------------------------------------------------------------------------------------------------------
def model(shape, sms=NUM_SMS):
    """Tiling and floors of one shape"""
    d = dict(shape.dims)
    on, box, taps, K, N, rows_in = geometry(shape.op, d)
    geglu = bool(shape.flags & 1)
    bn = tile_width(N, geglu)
    npt = bn // 2 if geglu else bn
    M = math.prod(on)
    wrows = 2 * N if geglu else N
    tiles = m_tiles(on, box) * _ceil(N, npt)
    iters = taps * _ceil(K, 64)
    flops = 2.0 * M * taps * K * wrows
    hbm = 2.0 * (band_input_rows(shape.op, d) * K + wrows * taps * K + M * N)
    if "residual" in shape.epi:
        hbm += 2.0 * M * N
    if "rowvec" in shape.epi:
        hbm += 2.0 * _ceil(M, d.get("rv_div", 1)) * N
    if "bias" in shape.epi:
        hbm += 2.0 * wrows
    if "colscale" in shape.epi:
        hbm += 2.0 * N
    fill = float(tiles) * iters * (math.prod(box) * 128 + bn * 128)
    t_mma, t_hbm = flops / (PEAK_TFLOPS * 1e9), hbm / (PEAK_HBM_GBS * 1e6)
    return {"M": M, "N": N, "K": K, "taps": taps, "bn": bn, "tiles": tiles, "waves": tiles / sms, "iters": iters,
            "geglu": geglu, "flops": flops, "hbm_bytes": hbm, "fill_bytes": fill, "mma_floor_ms": t_mma, "hbm_floor_ms": t_hbm,
            "floor_ms": max(t_mma, t_hbm), "bound": "MMA" if t_mma >= t_hbm else "HBM",
            "fill_needed_b_clk_sm": fill / (flops / 4096.0),      # at 2048 dense fp16 FMA per clock per SM
            "epi_instance": epi_instance(shape.flags, shape.epi)}


def label(shape):
    d = dict(shape.dims)
    if shape.op in ("linear", "linear_ex"):
        g = f"{d['rows']}x{d['K']}->{d['N']}"
    elif shape.op == "conv_t3":
        g = f"{d['B']}x{d['T']}x{d['HW']} {d['Cin']}->{d['Cout']}"
    elif shape.op == "conv3d_causal":
        g = f"{d['T']}x{d['H']}x{d['W']} {d['Cin']}->{d['Cout']}"
    else:
        g = f"{d['BT']}x{d['H']}x{d['W']} {d['Cin']}->{d['Cout']}"
    e = "+".join(k[:4] for k in shape.epi) + (f" f{shape.flags}" if shape.flags else "")
    return f"{shape.op.replace('conv2d_3x3', 'c3x3')} {g} {e}".strip()


# ---- GPU part ----------------------------------------------------------------------------------------------------------------------
def make_call(O, shape):
    """closure that launches `shape` alone on fresh random tensors"""
    import torch
    d = dict(shape.dims)
    on, box, taps, K, N, rows_in = geometry(shape.op, d)
    wrows = 2 * N if shape.flags & 1 else N
    M = math.prod(on)
    M_out = rows_in if shape.op == "conv_t3" else M                             # a band is written into the whole clip
    rnd = lambda *s, scale=1.0: (torch.randn(*s, device="cuda") * scale).half()  # noqa: E731
    bias = rnd(wrows, scale=0.1) if "bias" in shape.epi else None
    res = rnd(M_out, N) if "residual" in shape.epi else None
    rv = rnd(_ceil(M, d.get("rv_div", 1)), N) if "rowvec" in shape.epi else None
    cs = rnd(N) if "colscale" in shape.epi else None
    out = torch.empty(M_out, N, dtype=torch.float16, device="cuda")
    sc = (taps * K) ** -0.5
    if shape.op == "linear":
        a, w = rnd(M, K), rnd(wrows, K, scale=sc)
        return lambda: O.linear(a, w, bias, res, rv, d.get("rv_div", 1), shape.flags, out=out)
    if shape.op == "linear_ex":
        a, w = rnd(M, K), rnd(wrows, K, scale=sc)
        return lambda: O.linear_ex(a, w, bias, cs, res, shape.flags, out=out)
    if shape.op == "conv2d_3x3":
        x, w = rnd(d["BT"], d["H"], d["W"], K), rnd(N, 3, 3, K, scale=sc)
        return lambda: O.conv2d_3x3(x, w, bias, rv, d.get("rv_div", 1), res, out=out, rows=d.get("rows"))
    if shape.op == "conv2d_3x3_s2":
        x, w = rnd(d["BT"], d["H"], d["W"], K), rnd(N, 3, 3, K, scale=sc)
        return lambda: O.conv2d_3x3_s2(x, w, bias)
    if shape.op == "conv2d_3x3_s2p":
        x, w = rnd(d["BT"], d["H"], d["W"], K), rnd(N, 3, 3, K, scale=sc)
        return lambda: O.conv2d_3x3_s2p(x, w, bias, d["pad"])
    if shape.op == "conv_t3":
        x, w = rnd(M, K), rnd(N, 3, K, scale=sc)
        return lambda: O.conv_t3(x, w, bias, res, d["B"], d["T"], d["HW"], out=out, band=d.get("band"))
    x, w = rnd(rows_in, K), rnd(N, 3, 3, 3, K, scale=sc)
    return lambda: O.conv3d_causal(x, w, d["T"], d["H"], d["W"], bias, res, out=out)


def time_call(fn, est_ms, min_ms=60.0):
    import torch
    iters = int(max(5, min(2000, math.ceil(min_ms / max(est_ms, 1e-3)))))
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def time_alone(O, shape):
    import torch
    fn = make_call(O, shape)
    fn()
    torch.cuda.synchronize()
    ms = time_call(fn, time_call(fn, 1e9, 0.0))
    del fn
    torch.cuda.empty_cache()
    return ms


def record_step(O):
    """one bench-shape solver step: ({Shape: calls}, {Shape: ms inside the step}, ms of all traced ops)"""
    import torch
    import bench
    dev = torch.device("cuda", 0)
    net, _, _ = bench.build_model(False, dev)
    feat, y, ny = (t.to(dev) for t in bench.synth_inputs(bench.CHUNK, 122, 216))
    from star_b200.video_to_video.video_to_video_model import VideoToVideo_sr

    class Opt:
        model_path = None
    pipe = VideoToVideo_sr(Opt(), device=dev, text_encoder=bench._StubText(ny), vae=object(), generator=net)
    step = lambda: pipe.denoise_latents(feat, y, ny, total_noise_levels=1000, steps=1, solver_mode="normal",  # noqa: E731
                                        guide_scale=7.5, max_chunk_len=bench.CHUNK)
    step()
    calls, saved = [], {}
    for name in GEMM_OPS:
        inner = getattr(O, name)
        saved[name] = inner

        def rec(*a, _n=name, _f=inner, **k):
            calls.append(shape_of_call(_n, _f, a, k))        # the shape only: holding the arguments would pin every activation
            return _f(*a, **k)
        rec.__signature__ = inspect.signature(inner)
        setattr(O, name, rec)
    try:
        O.trace_begin()
        step()
        trace = O.trace_end()
    finally:
        for name, fn in saved.items():
            setattr(O, name, fn)
    gemm_trace = [t for t in trace if t[0] in GEMM_OPS]
    assert len(gemm_trace) == len(calls), "every recorded conv / linear call has one trace entry"
    counts, in_step = {}, {}
    for s, (tname, _sig, ms) in zip(calls, gemm_trace):
        assert s.op == tname
        counts[s] = counts.get(s, 0) + 1
        in_step[s] = in_step.get(s, 0.0) + ms
    total = sum(t[2] for t in trace)
    del pipe, net, calls
    torch.cuda.empty_cache()
    return counts, in_step, total


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--lib", default="", help="load this build of libstar_sm100.so instead of the tree's")
    ap.add_argument("--json", default="", help="also write the rows to this file")
    ap.add_argument("--no-step", action="store_true", help="skip the model step: only the synthetic sweep")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("tools/gemm_roofline.py measures on the GPU and needs one (an H100)")
    if args.lib:
        import star_b200.lib as _lib
        _lib.LIB_PATH = os.path.abspath(args.lib)
    from star_b200 import ops as O
    import bench
    from tools.kbench import card
    card()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    print(f"# floors: {PEAK_TFLOPS} TFLOP/s dense fp16, {PEAK_HBM_GBS} GB/s HBM3 (H100 SXM data sheet); {sms} SMs; "
          f"library {args.lib or 'of the tree'}", flush=True)

    clocks = bench.ClockSampler(0)
    clocks.start()
    counts, in_step, step_total = ({}, {}, 0.0) if args.no_step else record_step(O)
    lvl0 = {"BT": 32, "H": 122, "W": 216, "Cin": 320}
    sweep = [Shape("conv2d_3x3", tuple(sorted(dict(lvl0, Cout=n).items())), 0, ("bias",)) for n in (256, 320, 384)]
    timed = {s: time_alone(O, s) for s in list(counts) + sweep}
    clk = clocks.stop()
    mhz = clk.get("sm_mhz") or 0.0
    print(f"# SM clock while measuring: median {mhz} MHz of max {clk.get('sm_max_mhz')} MHz over {clk.get('samples')} samples; "
          f"throttle reasons {clk.get('reasons')}", flush=True)

    gemm_step = sum(timed[s] * c for s, c in counts.items())
    rows = []
    hdr = (f"{'shape':58s} {'calls':>5s} {'BN':>3s} {'waves':>6s} {'ms':>8s} {'TFLOP/s':>8s} {'HBM fl':>7s} {'MMA fl':>7s} "
           f"{'bound':>5s} {'x floor':>7s} {'fill GB':>8s} {'B/clk/SM':>8s} {'share':>6s}")
    print(hdr)
    order = sorted(counts, key=lambda s: -timed[s] * counts[s]) + sweep
    for s in order:
        ms = timed[s]
        m = model(s, sms=sms)
        c = counts.get(s, 0)
        row = {"shape": label(s), "sweep": s not in counts, "calls": c, "ms": ms, "tflops": m["flops"] / ms / 1e9,
               "fill_b_clk_sm": m["fill_bytes"] / (ms * 1e-3 * mhz * 1e6 * sms) if mhz else float("nan"),
               "share_of_gemm": ms * c / gemm_step if gemm_step else None, "in_step_ms": in_step.get(s),
               **{k: m[k] for k in ("M", "N", "K", "taps", "bn", "tiles", "waves", "flops", "hbm_bytes", "fill_bytes", "hbm_floor_ms",
                                    "mma_floor_ms", "bound", "fill_needed_b_clk_sm", "epi_instance")}}
        rows.append(row)
        print(f"{('sweep ' if row['sweep'] else '') + row['shape']:58s} {c:5d} {m['bn']:3d} {m['waves']:6.1f} {ms:8.3f} "
              f"{row['tflops']:8.1f} {m['hbm_floor_ms']:7.3f} {m['mma_floor_ms']:7.3f} {m['bound']:>5s} {ms / m['floor_ms']:7.2f} "
              f"{m['fill_bytes'] / 1e9:8.2f} {row['fill_b_clk_sm']:8.1f} {100 * (row['share_of_gemm'] or 0):5.1f}%", flush=True)
    if counts:
        print(f"# GEMM shapes timed alone: {gemm_step:.1f} ms per step; the same calls inside the step: {sum(in_step.values()):.1f} ms "
              f"of {step_total:.1f} ms traced over all ops", flush=True)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)) or ".", exist_ok=True)
        with open(args.json, "w") as f:
            json.dump({"clocks": clk, "sms": sms, "gemm_ms_alone": gemm_step, "gemm_ms_in_step": sum(in_step.values()),
                       "step_ms_traced": step_total, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
