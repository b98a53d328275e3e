"""Token-sharded CogVideoX DiT over NCCL on 4 and 8 GPUs of one node (skipped below 4): tools/dit_sp_check.py under torchrun,
cogvideox_parallel's sampler latent and the sharded forward against the single-GPU ones, byte for byte on every rank."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.skipif(torch.cuda.device_count() < 4, reason="needs >= 4 GPUs")
@pytest.mark.parametrize("nproc", [4, 8])
def test_nccl_sharded_dit_equals_single_gpu(nproc):
    if torch.cuda.device_count() < nproc:
        pytest.skip(f"needs {nproc} GPUs")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
                        "--master-addr", "127.0.0.1", "--master-port", str(29600 + nproc),
                        os.path.join(ROOT, "tools", "dit_sp_check.py")], cwd=ROOT, capture_output=True, text=True, timeout=900)
    print(r.stdout[-3000:])
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert r.stdout.count("equal: True") == 2 * nproc
