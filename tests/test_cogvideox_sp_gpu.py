"""Token-sharded CogVideoX DiT on the GPU (star_b200/cogvideox/parallel.py), byte for byte against the unsharded path:

* the shard's kernel calls against the whole sequence's: the QKV projection as one GEMM per destination rank followed by
  qk_ln_rope in place with the text boundary moved by the shard's offset == the rows of the fused GEMM + qk_ln_rope
  (P = 2, 3, 4, 8; shards before, across and after the text/image boundary), liem_spatial_gate on parts of the clip
  around an all-gathered map == the whole clip's gate, and linear_ex on the head-blocked all-to-all output == linear_ex
  on the concatenated rows;
* a 2-layer DiT at hidden 3072 / 48 heads, in bf16 and fp16, on 2, 3 and 4 gloo ranks sharing the one GPU (NCCL refuses
  two ranks on one device): every rank's output == the single-process forward;
* cogvideox_parallel on 4 ranks (two CFG groups x 2 sequence ranks) over 3 solver steps: the single-process latent;
* the unsharded forward still launches what it launched before the sharded path existed."""
import pytest
import torch

from tests.test_cogvideox import dit_inputs, dit_state_dict
from tests.test_tiles_sharded_gpu import _spawn

pytestmark = pytest.mark.gpu

DTYPES = [torch.bfloat16, torch.float16]
# the shapes of test_cogvideox.py's test_dit_model_gpu_vs_reference_files: 3 latent frames of 8 x 10 patches, S = 466
DIT_KW = dict(num_layers=2, hidden_size=3072, num_attention_heads=48, num_frames=9, latent_height=16, latent_width=20,
              text_length=226, text_hidden_size=4096, lora_r=64, time_embed_dim=512)


def _g(seed):
    return torch.Generator().manual_seed(seed)


# ---- kernel calls --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("P", [2, 3, 4, 8])
@pytest.mark.parametrize("tok0,rows", [(0, 117), (150, 155), (226, 80), (300, 166)])
def test_shard_qkv_and_qk_ln_rope_equal_rows_of_whole(dtype, P, tok0, rows):
    from star_b200 import ops
    heads, d, tl, S = 48, 3072, 226, 466
    c = heads // P * 64
    g = _g(P * 1000 + tok0)
    a = torch.randn(S, d, generator=g).to("cuda", dtype)
    w = (torch.randn(3 * d, d, generator=g) / 40).to("cuda", dtype)
    b = torch.randn(3 * d, generator=g).to("cuda", dtype)
    cos, sin = (torch.randn(S - tl, 64, generator=g).cuda() for _ in range(2))
    ln = [(1 + 0.3 * torch.randn(64, generator=g)).to("cuda", dtype) for _ in range(4)]
    want = ops.qk_ln_rope(ops.linear(a, w, b), heads, d, *ln, cos, sin, S, tl)[tok0:tok0 + rows]
    send = torch.empty((P, rows, 3 * c), dtype=dtype, device="cuda")
    for j in range(P):
        wj, bj = (torch.cat([t[o + j * c:o + (j + 1) * c] for o in (0, d, 2 * d)]).contiguous() for t in (w, b))
        ops.linear(a[tok0:tok0 + rows], wj, bj, out=send[j])
    ops.qk_ln_rope(send.view(P * rows, 3 * c), heads // P, c, *ln, cos, sin, rows, tl - tok0)
    torch.cuda.synchronize()
    got = send.view(P, rows, 3, c).permute(1, 2, 0, 3).reshape(rows, 3 * d)
    assert torch.equal(got, want)


@pytest.mark.parametrize("dtype", DTYPES)
def test_liem_on_parts_equals_whole_clip(dtype):
    from star_b200 import ops
    T, H, W, C = 3, 8, 10, 3072
    g = _g(5)
    x = torch.randn(T * H * W, C, generator=g).to("cuda", dtype)
    w98 = (0.5 * torch.randn(98, generator=g)).to("cuda", dtype)
    want = ops.liem_spatial_gate(x, w98, T, H, W)
    cuts = [0, 37, 80, 81, 163, 240]
    mm = torch.empty((T * H * W, 2), dtype=dtype, device="cuda")
    for a, b in zip(cuts, cuts[1:]):
        ops.liem_spatial_gate(x[a:b], None, T, H, W, part=ops.LiemPart(mm, a, b - a))
    for a, b in zip(cuts, cuts[1:]):
        got = ops.liem_spatial_gate(None, w98, T, H, W, part=ops.LiemPart(mm, a, b - a))
        assert torch.equal(got, want[a:b]), (a, b)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("P", [2, 3, 4, 8])
def test_dense_on_head_blocked_output_equals_linear_ex(dtype, P):
    """the all-to-all's [source rank][my rows][its 3072 / P columns] as the dense GEMM's A, over the row ranges a shard's
    text and image segments take, with the adaLN gate and the residual"""
    from star_b200 import ops
    n, d = 300, 3072
    g = _g(P)
    A = torch.randn(n, d, generator=g).to("cuda", dtype)
    w = (torch.randn(d, d, generator=g) / 40).to("cuda", dtype)
    b, gate = (torch.randn(d, generator=g).to("cuda", dtype) for _ in range(2))
    resid = torch.randn(n, d, generator=g).to("cuda", dtype)
    blocked = A.view(n, P, d // P).transpose(0, 1).contiguous()
    for lo, hi in [(0, n), (0, 117), (117, n), (5, 6)]:
        want = ops.linear_ex(A[lo:hi], w, b, colscale=gate, residual=resid[lo:hi])
        got = ops.linear_ex(blocked[:, lo:hi], w, b, colscale=gate, residual=resid[lo:hi])
        assert torch.equal(got, want), (lo, hi)


# ---- the sharded DiT and sampler -------------------------------------------------------------------------------------
def _nets(device="cuda"):
    from star_b200.cogvideox import DiffusionTransformer, dit_manifest
    kw = DIT_KW
    manifest = dit_manifest(kw["num_layers"], kw["hidden_size"], kw["num_attention_heads"], kw["time_embed_dim"],
                            text_hidden=kw["text_hidden_size"], lora_r=kw["lora_r"])
    sd = dit_state_dict({"manifest": manifest, "freqs": {}})
    nets = {}
    for dt in DTYPES:
        net = DiffusionTransformer(**kw, dtype=dt)
        net.load_state_dict(sd)
        nets[dt] = net.to(device)
    return nets


def _sampler_inputs(dtype):
    g = _g(11)
    T, h, w = 3, DIT_KW["latent_height"], DIT_KW["latent_width"]
    x = torch.randn(1, T, 16, h, w, generator=g).cuda()
    cond = {"crossattn": torch.randn(1, 226, 4096, generator=g).cuda()}
    uc = {"crossattn": torch.randn(1, 226, 4096, generator=g).cuda()}
    lq = torch.randn(1, T, 16, h, w, generator=g).cuda()
    return x, cond, uc, torch.cat([lq, lq])


def _sample(network, dtype):
    from star_b200.cogvideox import VPSDEDPMPP2MSampler
    x, cond, uc, lq = _sampler_inputs(dtype)
    torch.manual_seed(123)
    return VPSDEDPMPP2MSampler(num_steps=3, dtype=dtype)(network, x, cond, uc=uc, lq=lq)


SAMPLER_DTYPE = torch.bfloat16


def _on_ranks(rank, world):
    from star_b200.cogvideox import cogvideox_parallel, shard_sequence
    nets = _nets()
    x, t, ctx = dit_inputs(DIT_KW, "cuda")
    out = {dt: shard_sequence(net, None)(x, timesteps=t, context=ctx).cpu() for dt, net in nets.items()}
    if world == 4:
        out["sampler"] = _sample(cogvideox_parallel(nets[SAMPLER_DTYPE]), SAMPLER_DTYPE).cpu()
    torch.cuda.synchronize()
    return out


@pytest.fixture(scope="module")
def single():
    nets = _nets()
    x, t, ctx = dit_inputs(DIT_KW, "cuda")
    out = {dt: net(x, timesteps=t, context=ctx).cpu() for dt, net in nets.items()}
    out["sampler"] = _sample(nets[SAMPLER_DTYPE], SAMPLER_DTYPE).cpu()
    return out


@pytest.fixture(scope="module", params=[2, 3, 4])
def sharded(request):
    return request.param, _spawn(request.param, _on_ranks, )


def test_sharded_dit_equals_single_process(single, sharded):
    world, per_rank = sharded
    for dt in DTYPES:
        want = single[dt]
        assert torch.isfinite(want.float()).all()
        for rank, res in enumerate(per_rank):
            got = res[dt]
            diff = (got.float() - want.float()).abs().max().item()
            print(f"[{dt}] P = {world}, rank {rank}: max |sharded - single| {diff:.3e}")
            assert torch.equal(got, want), f"[{dt}] rank {rank} of {world} differs from the single-process forward"


def test_cfg_groups_times_sequence_ranks_sampler_equals_single_process(single, sharded):
    world, per_rank = sharded
    if world != 4:
        pytest.skip("the 2 CFG groups x 2 sequence ranks layout runs on 4 ranks")
    want = single["sampler"]
    assert torch.isfinite(want).all()
    for rank, res in enumerate(per_rank):
        assert torch.equal(res["sampler"], want), f"rank {rank}: max diff {(res['sampler'] - want).abs().max().item():.3e}"


def _expected_launches(B, layers):
    """op-by-op launch list of the unsharded DiffusionTransformer.forward"""
    seq = ["linear", "linear"] * B + ["sinusoidal", "linear", "linear"]
    for _ in range(layers):
        seq += ["silu", "linear"] + ["layernorm"] * 2 * B + ["liem_spatial_gate", "row_gate", "row_gate"] * B
        seq += ["linear", "qk_ln_rope", "attention"] + ["linear_ex"] * 2 * B
        seq += ["layernorm"] * 2 * B + ["linear_ex"] + ["linear_ex"] * 2 * B
    return seq + ["silu", "linear"] + ["layernorm", "layernorm", "linear"] * B


def test_unsharded_forward_launch_list_unchanged():
    from star_b200 import ops
    net = _nets()[torch.bfloat16]
    x, t, ctx = dit_inputs(DIT_KW, "cuda")
    net(x, timesteps=t, context=ctx)                                     # weight packing outside the trace
    n0 = ops.launch_count()
    ops.trace_begin()
    net(x, timesteps=t, context=ctx)
    trace = ops.trace_end()
    names = [n for n, _, _ in trace]
    assert names == _expected_launches(2, DIT_KW["num_layers"])
    assert ops.launch_count() - n0 == len(names) + DIT_KW["num_layers"] * 2     # liem_spatial_gate is two kernels
    qk = [sig for n, sig, _ in trace if n == "qk_ln_rope"]
    att = [sig for n, sig, _ in trace if n == "attention"]
    assert all(s[0] == (2 * 466, 3 * 3072) for s in qk)                  # in place on the whole batch's QKV
    assert all(s[3:7] == (2, 48, 466, 466) for s in att)                  # one call over both samples and all 48 heads
