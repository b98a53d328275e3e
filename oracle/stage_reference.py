"""TEST / BASELINE INFRASTRUCTURE -- stage the reference's hot-path Python files for the GPU box.

/root/reference exists only in the build container.  The GPU-side baseline the north-star's ">= 8x the
reference's single-GPU PyTorch frames/sec" is written against (SURVEY 8d "Reference timed beside it",
VERDICT r1 item 1) needs the UNMODIFIED reference modules on the GPU, so this recipe copies the few files
oracle/ref_loader.py executes into oracle/_ref/ -- git-ignored (no reference source enters the history), not
gpurun-ignored (it travels with the snapshot like a built .so).  Nothing is edited; ref_loader's import shims
are applied at load time exactly as in the container.

    python -m oracle.stage_reference            # idempotent; prints what it staged

Files (relative to /root/reference): the model surface, the sampler, the helpers of the pipeline file and the
tiny utils the sampler imports.  The CogVideoX files are staged for oracle/cogvideox_sat.py (sat shim layer) and
oracle/cogvideox_vae.py (3-D VAE decoder).
"""
import os
import shutil
import sys

SRC = os.environ.get("STAR_REFERENCE_SRC", "/root/reference")
DST = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref")

FILES = [
    "video_to_video/__init__.py",
    "video_to_video/video_to_video_model.py",
    "video_to_video/modules/unet_v2v.py",
    "video_to_video/diffusion/__init__.py",
    "video_to_video/diffusion/diffusion_sdedit.py",
    "video_to_video/diffusion/solvers_sdedit.py",
    "video_to_video/diffusion/schedules_sdedit.py",
    "video_to_video/utils/__init__.py",
    "video_to_video/utils/config.py",
    "video_to_video/utils/logger.py",
    "video_to_video/utils/seed.py",
    "cogvideox-based/transformer.py",
    "cogvideox-based/sat/dit_video_concat.py",
    "cogvideox-based/sat/sgm/modules/diffusionmodules/util.py",
    "cogvideox-based/sat/vae_modules/cp_enc_dec.py",
    "cogvideox-based/sat/sgm/modules/diffusionmodules/sampling_utils.py",
    "cogvideox-based/sat/sgm/modules/diffusionmodules/guiders.py",
    "cogvideox-based/sat/sgm/modules/diffusionmodules/discretizer.py",
    "cogvideox-based/sat/sgm/modules/diffusionmodules/denoiser_scaling.py",
    "cogvideox-based/sat/sgm/modules/diffusionmodules/denoiser_weighting.py",
    "cogvideox-based/sat/sgm/modules/diffusionmodules/denoiser.py",
    "cogvideox-based/sat/sgm/modules/diffusionmodules/wrappers.py",
    "cogvideox-based/sat/sgm/modules/diffusionmodules/sampling.py",
]


def stage(verbose=True):
    if not os.path.isdir(SRC):
        if verbose:
            print(f"stage_reference: {SRC} not present (GPU box?) -- nothing to do")
        return 0
    n = 0
    for rel in FILES:
        s, d = os.path.join(SRC, rel), os.path.join(DST, rel)
        if not os.path.isfile(s):
            if verbose:
                print("  missing in reference:", rel)
            continue
        os.makedirs(os.path.dirname(d), exist_ok=True)
        shutil.copyfile(s, d)
        n += 1
    if verbose:
        print(f"stage_reference: {n} files -> {DST}")
    return n


if __name__ == "__main__":
    sys.exit(0 if stage() >= 0 else 1)
