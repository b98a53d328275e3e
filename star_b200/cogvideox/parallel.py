"""One CogVideoX clip on more than two GPUs: token-sharded DiT layers with head-parallel attention (Ulysses-style sequence
parallelism), alone or inside the two-rank CFG split of ``split_cfg_pair``.

Each of P ranks holds a contiguous, balanced shard of every sample's S = text_length + T*gh*gw tokens (text first, image
tokens in (t, h, w) order).  Everything in a layer but attention is per token and runs on the shard; the spatial LIEM gate
all-gathers its 2-value-per-token mean/max map.  Around attention one all-to-all turns "my tokens, all heads" into
"all S tokens, my heads / P": the QKV projection runs as one GEMM per destination rank, straight into that rank's block of
the send buffer, and qk_ln_rope normalises and rotates it in place, so the receive buffer is directly the strided q / k / v
views ``ops.attention`` takes.  A second all-to-all returns each rank's rows of the result, head-blocked, which the dense
projection reads in place (``ops.linear_ex`` on a [source rank, rows, columns] view).  Every per-element sequence is the
unsharded forward's, so each rank's output equals the single-GPU forward byte for byte.
"""
from dataclasses import dataclass
from typing import List

import torch
import torch.distributed as dist

from .sampling import split_cfg_pair


@dataclass(frozen=True)
class RankShard:
    """Rank `rank`'s tokens [start, stop) of every sample; its first `text_rows` tokens are text (only a shard that starts
    inside the text has any, so the text/image boundary lies inside at most one shard).  Split sizes are in tokens (rows
    of the exchanged matrices), indexed by peer rank: qkv_send / qkv_recv for the q|k|v all-to-all (this shard's rows to
    every rank, every rank's shard back), out_send / out_recv for the attention output going back (the mirror image)."""
    rank: int
    start: int
    stop: int
    text_rows: int
    qkv_send: List[int]
    qkv_recv: List[int]
    out_send: List[int]
    out_recv: List[int]

    @property
    def rows(self):
        return self.stop - self.start

    @property
    def image_rows(self):
        return self.rows - self.text_rows


def dit_shard_plan(text_len, frames, gh, gw, P, heads=48):
    """Per-rank token shards of text_len text tokens followed by frames * gh * gw image tokens over P ranks: contiguous,
    balanced to +-1 token, in rank order from the first text token.  Raises ValueError when the heads do not split
    evenly over P ranks or a rank would hold no token."""
    if P < 1 or heads % P:
        raise ValueError(f"{heads} attention heads do not split evenly over {P} ranks")
    S = text_len + frames * gh * gw
    if S < P:
        raise ValueError(f"{S} tokens cannot be sharded over {P} ranks")
    base, extra = divmod(S, P)
    sizes = [base + (1 if r < extra else 0) for r in range(P)]
    plan, lo = [], 0
    for r, n in enumerate(sizes):
        plan.append(RankShard(rank=r, start=lo, stop=lo + n, text_rows=max(0, min(lo + n, text_len) - lo),
                              qkv_send=[n] * P, qkv_recv=list(sizes), out_send=list(sizes), out_recv=[n] * P))
        lo += n
    return plan


class SeqShard:
    """This rank's part of a sequence-parallel group: its shard, the group's plan, and the group's collectives."""

    def __init__(self, plan, group=None):
        self.plan, self.group = plan, group
        self.P, self.rank = dist.get_world_size(group), dist.get_rank(group)
        if len(plan) != self.P:
            raise ValueError(f"a shard plan for {len(plan)} ranks on a group of {self.P}")
        self.me = plan[self.rank]

    def all_to_all(self, send, leg):
        """leg "qkv": send [P * rows, C] (dest-rank-major) -> [S, C] (every rank's shard in rank order); leg "out": the
        reverse, [S, C] -> [P * rows, C] (source-rank-major).  NCCL, and gloo on CPU tensors: one all_to_all_single.
        gloo has no all-to-all for CUDA tensors; there each rank all-gathers the send buffers and keeps its rows."""
        splits = {p.rank: (p.qkv_send, p.qkv_recv) if leg == "qkv" else (p.out_send, p.out_recv) for p in self.plan}
        send_splits, recv_splits = splits[self.rank]
        recv = send.new_empty((sum(recv_splits),) + tuple(send.shape[1:]))
        if not (send.is_cuda and dist.get_backend(self.group) == "gloo"):
            dist.all_to_all_single(recv, send.contiguous(), recv_splits, send_splits, group=self.group)
            return recv
        totals = [sum(splits[r][0]) for r in range(self.P)]
        gathered = self.all_gather_rows(send, totals)
        parts, off = [], 0
        for r in range(self.P):
            s = splits[r][0]
            lo = off + sum(s[:self.rank])
            parts.append(gathered[lo:lo + s[self.rank]])
            off += totals[r]
        torch.cat(parts, 0, out=recv)
        return recv

    def all_gather_rows(self, local, counts):
        """every rank's `local` rows (counts[r] of them on rank r) concatenated in rank order: ONE all-gather"""
        buf = local.new_zeros((max(counts),) + tuple(local.shape[1:]))
        if counts[self.rank]:
            buf[:counts[self.rank]] = local
        parts = [torch.empty_like(buf) for _ in range(self.P)]
        dist.all_gather(parts, buf, group=self.group)
        return torch.cat([parts[r][:counts[r]] for r in range(self.P) if counts[r]], 0)

    def gather_image_rows(self, local):
        """the whole sample's image-token rows from every rank's image rows"""
        return self.all_gather_rows(local, [p.image_rows for p in self.plan])


def shard_sequence(network, group=None):
    """Wraps the DiffusionTransformer ``network`` into a callable with its signature whose forward runs token-sharded over
    the ranks of `group` (every sample of the batch on every rank, one exchange per sample) and returns the whole output
    on every rank: the sampler runs replicated on the ranks, seeded alike, as under ``split_cfg_pair``."""
    P = dist.get_world_size(group)
    text_len, frames, gh, gw, heads = network.text_length, network.frames, network.gh, network.gw, network.cfg["heads"]
    sp = SeqShard(dit_shard_plan(text_len, frames, gh, gw, P, heads), group)

    def sharded(x, timesteps=None, context=None, **kw):
        return network.forward(x, timesteps=timesteps, context=context, shard=sp, **kw)
    return sharded


def cogvideox_parallel(network, world=None):
    """The DiT callable for one clip on the ranks of `world` (default: every rank; all ranks of the default group must
    call this, since it creates process groups), laid out by their number W:
      W = 1             the network itself;
      W = 2             the CFG pair on two ranks (split_cfg_pair), as before;
      even W = 2P > 2   two CFG groups of P ranks, each sequence-parallel over its P ranks;
      other W           sequence parallelism over all W ranks, both CFG samples on every rank.
    Raises ValueError when W does not divide the attention heads (for even W: when P does not)."""
    W = dist.get_world_size(world)
    if W == 1:
        return network
    if W == 2:
        return split_cfg_pair(network, world)
    heads = network.cfg["heads"]
    ranks = dist.get_process_group_ranks(world) if world is not None else list(range(W))
    me = ranks.index(dist.get_rank())
    if W % 2 == 0 and heads % (W // 2) == 0:
        P = W // 2
        seq = [dist.new_group(ranks[b * P:(b + 1) * P]) for b in range(2)]
        pairs = [dist.new_group([ranks[i], ranks[i + P]]) for i in range(P)]
        return split_cfg_pair(shard_sequence(network, seq[me // P]), pairs[me % P])
    if heads % W:
        raise ValueError(f"{W} ranks: {heads} attention heads split over neither {W} ranks nor two CFG groups of {W // 2}")
    return shard_sequence(network, world)
