"""TEST INFRASTRUCTURE -- generate tests/golden/long_chunk.pt by executing the UNMODIFIED reference
(/root/reference, build container only), CPU, fp32.  Run:  python -m oracle.make_golden_long_chunk

Chunks longer than 64 frames (max_chunk_len >= 52 stretches the last window past 64), which the product runs
on the T > 64 temporal-attention kernel (star_b200/csrc/tattn_long.cuh).  Inputs and weights are regenerated
from seeds by tests/util.py, as for oracle/make_golden.py:
  unet         reduced ControlledV2VUNet (SMALL_KW, weight seed 1) at F = 72 and F = 130, latent 10 x 8: fp32
               output of the real reference + its own fp16-autocast (CPU) output and that output's error
  sampler      sample_sr with the reduced UNet, F = 100, chunks make_chunks(100, 0, 64) = (0, 64), (32, 100):
               a 64-frame and a 68-frame chunk in one run; 2 steps, CFG 7.5, injected noise
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ref_loader as R  # noqa: E402
from oracle.make_golden import build_ref, logging_off  # noqa: E402
from tests.util import SMALL_KW, make_inputs  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "long_chunk.pt")


@torch.no_grad()
def main():
    torch.manual_seed(0)
    ns = R.load_reference()
    logging_off()

    # ---- UNet forward, reduced model, T > 64 frames ---------------------------------------------
    net, _ = build_ref(SMALL_KW, seed=1)
    cases = []
    for (seed, B, F, H, W, t) in [(31, 1, 72, 10, 8, [650]), (32, 1, 130, 10, 8, [120])]:
        x, hint, y = make_inputs(seed, B, F, H, W)
        o32 = net(x, torch.tensor(t), y, hint=hint)
        cases.append(dict(seed=seed, B=B, F=F, H=H, W=W, t=t, out_fp32=o32.clone()))
        print("small", seed, B, F, H, W, float(o32.std()))
    neth = net.half()
    for c in cases:
        x, hint, y = make_inputs(c["seed"], c["B"], c["F"], c["H"], c["W"])
        with torch.autocast("cpu", dtype=torch.float16):
            o16 = neth(x, torch.tensor(c["t"]), y, hint=hint)
        c["out_ref_fp16"] = o16.clone()
        c["ref_fp16_rel_err"] = float((o16.float() - c["out_fp32"]).norm() / c["out_fp32"].norm())
        print("  ref fp16-autocast rel err", c["ref_fp16_rel_err"])

    # ---- sampler with the reduced UNet: chunks of 64 and 68 frames ------------------------------
    net = net.float()
    sig = ns.schedules_sdedit.noise_schedule(schedule="logsnr_cosine_interp", n=1000, zero_terminal_snr=True,
                                             scale_min=2.0, scale_max=4.0)
    diff = ns.diffusion_sdedit.GaussianDiffusion(sigmas=sig)
    F, H, W = 100, 10, 8
    chunks = [tuple(c) for c in ns.make_chunks(F, 0, 64)]
    assert chunks == [(0, 64), (32, 100)], chunks
    x, hint, y = make_inputs(41, 1, F, H, W)
    _, _, ny = make_inputs(42, 1, F, H, W)
    R.InjectedBrownian.seed = 99
    out = diff.sample_sr(noise=x.clone(), model=net, model_kwargs=[{"y": y}, {"y": ny}, {"hint": hint}],
                         guide_scale=7.5, guide_rescale=0.2, solver="dpmpp_2m_sde", solver_mode="normal", steps=2,
                         t_max=899, t_min=0, discretization="trailing", chunk_inds=chunks)
    sampler = dict(input_seed=41, neg_seed=42, noise_seed=99, F=F, H=H, W=W, steps=2, max_chunk_len=64,
                   chunk_inds=chunks, out=out.clone())
    print("sampler+unet chunked", chunks, float(out.std()))

    torch.save(dict(kw=SMALL_KW, weight_seed=1, cases=cases, sampler=sampler), OUT)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
