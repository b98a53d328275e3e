#!/usr/bin/env python
"""Token-sharded CogVideoX DiT over NCCL (run under torchrun, one rank per GPU; driven by tests/test_cogvideox_sp_nccl_gpu.py):
the 2-layer hidden-3072 / 48-head DiT of tests/test_cogvideox_sp_gpu.py, 3 solver steps through cogvideox_parallel on all
ranks (W = 4: two CFG groups x 2 sequence ranks; W = 8: two CFG groups x 4), and the sharded forward alone (shard_sequence over
all W ranks, both CFG samples on each), against rank 0's single-GPU runs, byte for byte on every rank.
Prints one "sp check ... equal: True|False" line per rank and check; exits non-zero when a check fails on any rank."""
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    from star_b200.cogvideox import cogvideox_parallel, shard_sequence
    from tests.test_cogvideox import dit_inputs
    from tests.test_cogvideox_sp_gpu import DIT_KW, SAMPLER_DTYPE, _nets, _sample
    net = _nets()[SAMPLER_DTYPE]
    x, t, ctx = dit_inputs(DIT_KW, "cuda")
    got = {"sampler": _sample(cogvideox_parallel(net), SAMPLER_DTYPE)}
    if 48 % world == 0:
        got["forward"] = shard_sequence(net)(x, timesteps=t, context=ctx)
    want = {"sampler": _sample(net, SAMPLER_DTYPE), "forward": net(x, timesteps=t, context=ctx)}
    ok = True
    for name, g in got.items():
        w = want[name].contiguous()
        dist.broadcast(w, 0)                              # rank 0's single-GPU result is the reference of every rank
        eq = torch.equal(g, w)
        ok &= eq
        print(f"sp check {name} rank {rank}/{world}: max diff {(g.float() - w.float()).abs().max().item():.3e} equal: {eq}",
              flush=True)
    flag = torch.tensor([int(ok)], device=dev)
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    dist.destroy_process_group()
    sys.exit(0 if flag.item() else 1)


if __name__ == "__main__":
    main()
