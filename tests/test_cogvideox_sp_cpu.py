"""Token-sharded CogVideoX DiT without a GPU: the shard plan's properties, and the sharded host graph (parallel.py,
DiTLayer.forward_shard, DiffusionTransformer's sharded forward) on the emulated kernels over 2 and 3 gloo CPU ranks,
against the unsharded forward on the same emulated kernels, bit for bit.

The emulated kernels are oracle/kernel_ref.py's; the two calls the sharded path adds to them -- a head-blocked A for
linear_ex and liem_spatial_gate on a part of the clip -- are emulated here from the same references."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn.functional as F


# ---- the emulated kernels: oracle/kernel_ref.py's, with its GEMMs one row at a time ----------------------------------
def row_by_row(ref):
    """kernel_ref's GEMM reference ``ref`` evaluated one row at a time.  A CPU GEMM library picks its blocking, and with
    it the fp32 summation order, from the row count (a row's result changes with the rows around it), while a row of the
    tap-GEMM is the same whatever rows share its launch; one row per call is the same on every shard.  A head-blocked a
    [blocks, rows, block_cols] is read as the [rows, blocks * block_cols] matrix it stands for."""
    def gemm(a, w, bias=None, residual=None, out=None, colscale=None, flags=0, **kw):
        if a.dim() == 3:
            a = a.permute(1, 0, 2).reshape(a.shape[1], -1)
        extra = dict(kw, flags=flags)
        if colscale is not None:
            extra["colscale"] = colscale
        res = torch.cat([ref(a[i:i + 1], w, bias, residual=None if residual is None else residual[i:i + 1], **extra)
                         for i in range(a.shape[0])])
        if out is not None:
            out.copy_(res)
            return out
        return res
    return gemm


def liem_spatial_gate(x, w98, BT, H, W, part=None):
    """kernel_ref.liem_spatial_gate, and its two steps on a part of the clip (ops.LiemPart)"""
    from oracle import kernel_ref as KR
    if part is None:
        return KR.liem_spatial_gate(x, w98, BT, H, W)
    if x is not None:
        xf = x.float()
        part.mm[part.r0:part.r0 + part.n] = torch.stack([xf.max(dim=-1)[0], xf.mean(dim=-1)], dim=1).to(KR.HALF)
    if w98 is None:
        return part.mm
    m = part.mm.float().reshape(BT, H, W, 2).permute(0, 3, 1, 2)
    conv = F.conv2d(m, w98.float().reshape(1, 2, 7, 7), padding=3).to(KR.HALF).float()
    return torch.sigmoid(conv).reshape(-1).to(KR.HALF)[part.r0:part.r0 + part.n]


def emulate_ops(setattr_):
    """route every star_b200.ops kernel call to its kernel_ref emulation (the GEMMs one row at a time, see row_by_row)"""
    from oracle import kernel_ref as KR
    from star_b200 import ops
    for name in dir(KR):
        if not name.startswith("_") and callable(getattr(KR, name)) and hasattr(ops, name):
            setattr_(ops, name, getattr(KR, name))
    setattr_(ops, "linear", row_by_row(KR.linear))
    setattr_(ops, "linear_ex", row_by_row(KR.linear_ex))
    setattr_(ops, "liem_spatial_gate", liem_spatial_gate)


# ---- shard plan ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("text_len,frames,gh,gw", [(226, 13, 30, 45), (226, 7, 30, 45), (226, 3, 8, 10), (40, 3, 4, 6)])
@pytest.mark.parametrize("P", [1, 2, 3, 4, 6, 8])
def test_shard_plan_owns_every_token_once_balanced(text_len, frames, gh, gw, P):
    from star_b200.cogvideox import dit_shard_plan
    plan = dit_shard_plan(text_len, frames, gh, gw, P)
    S = text_len + frames * gh * gw
    assert [p.rank for p in plan] == list(range(P))
    assert plan[0].start == 0 and plan[-1].stop == S
    assert all(a.stop == b.start for a, b in zip(plan, plan[1:]))                     # contiguous, in rank order
    sizes = [p.rows for p in plan]
    assert max(sizes) - min(sizes) <= 1 and sum(sizes) == S
    assert plan[0].text_rows == min(text_len, sizes[0])                                 # the text starts on rank 0
    assert sum(p.text_rows for p in plan) == text_len
    assert sum(p.image_rows for p in plan) == frames * gh * gw
    assert sum(1 for p in plan if 0 < p.text_rows < p.rows) <= 1                         # at most one shard straddles
    for p in plan:
        assert p.text_rows == max(0, min(p.stop, text_len) - p.start)
        assert p.qkv_send == [p.rows] * P and p.out_recv == [p.rows] * P
        assert p.qkv_recv == sizes and p.out_send == sizes
        assert sum(p.qkv_send) == p.rows * P and sum(p.qkv_recv) == S
    for j in range(P):                                                                  # what i sends to j is what j receives from i
        assert [plan[i].qkv_send[j] for i in range(P)] == plan[j].qkv_recv
        assert [plan[i].out_send[j] for i in range(P)] == plan[j].out_recv


def test_shard_plan_at_the_shipped_sizes():
    from star_b200.cogvideox import dit_shard_plan
    plan = dit_shard_plan(226, 13, 30, 45, 4)                                           # 49 frames: 17 776 tokens
    assert [p.rows for p in plan] == [4444] * 4 and plan[0].text_rows == 226
    plan = dit_shard_plan(226, 7, 30, 45, 8)                                            # 25 frames, 8 ranks
    assert sorted({p.rows for p in plan}) == [1209, 1210]


@pytest.mark.parametrize("P", [5, 7, 9, 0])
def test_shard_plan_refuses_ranks_that_do_not_split_the_heads(P):
    from star_b200.cogvideox import dit_shard_plan
    with pytest.raises(ValueError):
        dit_shard_plan(226, 13, 30, 45, P)


# ---- the shard's emulated calls against the whole clip's -------------------------------------------------------------
@pytest.mark.parametrize("P,tok0", [(2, 0), (3, 5), (6, 40)])
def test_shard_qk_ln_rope_with_moved_text_boundary_equals_rows_of_whole(P, tok0):
    """rows tok0.. of a sequence, in P per-rank blocks, with seq = rows and the text boundary at text_len - tok0"""
    from oracle import kernel_ref as KR
    heads, rows, tl = 6, 20, 12
    d, hp = heads * 64, heads // P
    g = torch.Generator().manual_seed(P)
    S = tok0 + rows + 3
    qkv = torch.randn(S, 3 * d, generator=g).half()
    cos, sin = torch.randn(S, 64, generator=g), torch.randn(S, 64, generator=g)
    ln = [torch.randn(64, generator=g).half() for _ in range(4)]
    want = KR.qk_ln_rope(qkv.clone(), heads, d, *ln, cos, sin, S, tl)[tok0:tok0 + rows]
    blocks = qkv[tok0:tok0 + rows].reshape(rows, 3, P, hp * 64).permute(2, 0, 1, 3).reshape(P * rows, 3 * hp * 64).clone()
    KR.qk_ln_rope(blocks, hp, hp * 64, *ln, cos, sin, rows, tl - tok0)
    got = blocks.reshape(P, rows, 3, hp * 64).permute(1, 2, 0, 3).reshape(rows, 3 * d)
    assert torch.equal(got, want)


def test_liem_on_parts_equals_whole_clip():
    g = torch.Generator().manual_seed(3)
    x = torch.randn(72, 64, generator=g).half()
    w98 = torch.randn(98, generator=g).half()
    want = liem_spatial_gate(x, w98, 3, 4, 6)
    mm = torch.empty(72, 2).half()
    from star_b200.ops import LiemPart
    for a, b in ((0, 30), (30, 72)):
        liem_spatial_gate(x[a:b], None, 3, 4, 6, LiemPart(mm, a, b - a))
    for a, b in ((0, 30), (30, 72)):
        assert torch.equal(liem_spatial_gate(None, w98, 3, 4, 6, LiemPart(mm, a, b - a)), want[a:b])


# ---- sharded host graph on gloo CPU ranks ---------------------------------------------------------------------------
SIX_HEADS = dict(num_layers=2, hidden_size=384, num_attention_heads=6, num_frames=9, latent_height=8, latent_width=12,
                 text_length=40, text_hidden_size=32, lora_r=8, time_embed_dim=64)


def small_net():
    from star_b200.cogvideox import DiffusionTransformer, dit_manifest
    from tests.test_cogvideox import dit_state_dict
    kw = SIX_HEADS
    manifest = dit_manifest(kw["num_layers"], kw["hidden_size"], kw["num_attention_heads"], kw["time_embed_dim"],
                            text_hidden=kw["text_hidden_size"], lora_r=kw["lora_r"])
    net = DiffusionTransformer(**kw, dtype=torch.float16)
    net.load_state_dict(dit_state_dict({"manifest": manifest, "freqs": {}}))
    return net


def _sharded_worker(rank, world, port, q):
    from star_b200.cogvideox import shard_sequence
    from tests.test_cogvideox import dit_inputs
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        emulate_ops(setattr)
        x, t, ctx = dit_inputs(SIX_HEADS, "cpu")
        q.put((rank, shard_sequence(small_net(), None)(x, timesteps=t, context=ctx)))
    except BaseException as e:
        q.put((rank, repr(e)))
        raise
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_host_graph_equals_unsharded(world, monkeypatch):
    from tests.test_cogvideox import dit_inputs
    emulate_ops(monkeypatch.setattr)
    x, t, ctx = dit_inputs(SIX_HEADS, "cpu")
    want = small_net()(x, timesteps=t, context=ctx)
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx_mp = mp.get_context("spawn")
    q = ctx_mp.Queue()
    procs = [ctx_mp.Process(target=_sharded_worker, args=(r, world, port, q)) for r in range(world)]
    try:
        for p in procs:
            p.start()
        res = dict(q.get(timeout=300) for _ in procs)
        for p in procs:
            p.join(timeout=60)
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
                p.join()
    for rank in range(world):
        got = res[rank]
        assert torch.is_tensor(got), f"rank {rank}: {got}"
        assert got.shape == want.shape and torch.isfinite(want.float()).all()
        diff = (got.float() - want.float()).abs().max().item()
        assert torch.equal(got, want), f"rank {rank} of {world}: max |sharded - unsharded| {diff:.3e}"
