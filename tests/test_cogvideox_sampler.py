"""CogVideoX sampling loop (VPSDEDPMPP2MSampler + DynamicCFG + DiscreteDenoiser / VideoScaling) against the reference's UNMODIFIED
sgm/modules/diffusionmodules files (oracle/cogvideox_sampler.py)."""
import pytest
import torch

from tests.util import rel_l2


class FakeDiT(torch.nn.Module):
    """cheap deterministic stand-in with the DiffusionTransformer call signature: (2B, T, 32, h, w) -> (2B, T, 16, h, w)"""

    def __init__(self):
        super().__init__()
        self.calls = []

    def forward(self, x, timesteps=None, context=None, y=None, **kw):
        self.calls.append(float(timesteps[0]))
        noisy, lq = x.float().chunk(2, dim=2)
        t = timesteps.float().view(-1, 1, 1, 1, 1) / 1000.0
        c = context.float().mean(dim=(1, 2)).view(-1, 1, 1, 1, 1)
        return torch.tanh(0.8 * noisy - 0.3 * lq + 0.1 * noisy.mean(dim=1, keepdim=True)) * (1.0 + 0.2 * c) + 0.05 * t * lq


def test_step_plan_matches_reference_tables():
    """against the reference sampler's tables (tests/golden/cogvideox_path.pt, oracle/make_golden_cogvideox.py): alphas_cumprod_sqrt
    and timesteps of prepare_sampling_loop, the denoiser's quantised sigma and DynamicCFG's scale of every step"""
    import os
    from star_b200.cogvideox.sampling import StepPlan
    gold = torch.load(os.path.join(os.path.dirname(__file__), "golden", "cogvideox_path.pt"))
    acs, timesteps = gold["acs"], gold["timesteps"]
    plan = StepPlan()
    assert len(acs) == 51 and torch.equal(plan.alphas_cumprod_sqrt, acs)
    assert plan.timesteps == timesteps
    for i, st in enumerate(plan.steps):                                   # quantised sigma of the denoiser, guidance scale
        assert st.c_skip == float(gold["sigma_q"][i]) and st.timestep == timesteps[-(i + 1)]
        assert st.cfg_scale == gold["cfg"][i]
    assert [st.last for st in plan.steps] == [False] * 49 + [True]


def sampler_case():
    g = torch.Generator().manual_seed(0)
    lq = torch.randn(1, 3, 16, 6, 8, generator=g)
    randn = torch.randn(1, 3, 16, 6, 8, generator=g)
    cond = {"crossattn": torch.randn(1, 226, 32, generator=g)}
    uc = {"crossattn": torch.zeros(1, 226, 32)}
    return lq, randn, cond, uc


@pytest.mark.parametrize("steps", [50, 6])
def test_sampler_matches_reference(steps):
    """against the reference sampler's output on the same inputs (tests/golden/reference_checks.pt)"""
    import os
    from star_b200.cogvideox.sampling import VPSDEDPMPP2MSampler
    rec = torch.load(os.path.join(os.path.dirname(__file__), "golden", "reference_checks.pt"))[f"sampler{steps}"]
    lq, randn, cond, uc = sampler_case()
    want = rec["want"]
    net_m = FakeDiT()
    mine = VPSDEDPMPP2MSampler(num_steps=steps, dtype=torch.float32)
    torch.manual_seed(123)
    got = mine(net_m, randn.clone(), cond, uc=uc, lq=torch.cat((lq, lq), 0))
    assert net_m.calls == rec["calls"] and len(net_m.calls) == steps
    assert got.shape == want.shape == randn.shape
    assert rel_l2(got, want) < 2e-5
    # random-stream consumption: 1 draw in the first step, 2 in every later one but the last (sampling.py:635,:641)
    after = torch.randn(4)
    torch.manual_seed(123)
    for _ in range(2 * steps - 3):
        torch.randn_like(randn)
    assert torch.equal(after, torch.randn(4))


def _pipeline_pair(dit_kw, vae_kw, dtype, device):
    from tests.test_cogvideox import _dit_pair
    from tests.test_cogvideox_vae import _enc_pair, _pair
    ref_dit, net, _x, _t, ctx = _dit_pair(dit_kw, dtype, device)
    ref_dec, dec, _ = _pair(vae_kw, device=device, dtype=dtype)
    ref_enc, enc, _ = _enc_pair(vae_kw, device=device, dtype=dtype)
    return ref_dit, net, (ref_enc, ref_dec), (enc, dec), ctx


def _reference_pipeline(ref_dit, ref_vae, cond, uc, lq, steps, seed, scale_factor=0.7):
    """sample_sr.py:186-230 / diffusion_video.py:245-292 on the reference's own modules (3-D VAE encoder + Gaussian posterior sample,
    DiT behind the sat shim, sampler stack, 3-D VAE decoder); lq (1, F, 3, H, W)"""
    from oracle.cogvideox_sampler import build_reference_sampler, reference_sample
    from oracle.cogvideox_vae import load_reference_vae, reference_decode_latent, reference_encode_moments
    ref_enc, ref_dec = ref_vae
    sampler, den = build_reference_sampler(num_steps=steps, device=str(lq.device))
    torch.manual_seed(seed)
    F, H, W = lq.shape[1], lq.shape[3], lq.shape[4]
    randn = torch.randn((1, (F - 1) // 4 + 1, 16, H // 8, W // 8), dtype=torch.float32).to(lq.device)
    moments = reference_encode_moments(ref_enc, lq.permute(0, 2, 1, 3, 4).contiguous())
    mean, logvar = torch.chunk(moments, 2, dim=1)                         # DiagonalGaussianDistribution.sample (regularizers.py:10-29)
    zq = mean + torch.exp(0.5 * torch.clamp(logvar, -30.0, 20.0)) * torch.randn_like(mean)
    lq_latent = (scale_factor * zq).permute(0, 2, 1, 3, 4).contiguous()
    z = reference_sample(ref_dit, sampler, den, randn, dict(cond), dict(uc), lq_latent)
    latent = (1.0 / scale_factor) * z.permute(0, 2, 1, 3, 4).contiguous()
    frames = reference_decode_latent(ref_dec, latent).float().permute(0, 2, 1, 3, 4)
    return torch.clamp((frames + 1.0) / 2.0, 0.0, 1.0), z


def pipeline_case(ctx):
    cond, uc = {"crossattn": ctx[:1]}, {"crossattn": torch.zeros_like(ctx[:1])}
    lq = torch.rand(1, 9, 3, 64, 96, generator=torch.Generator().manual_seed(9)) * 2 - 1          # LQ clip, already upsampled
    return cond, uc, lq


def test_cogvideox_pipeline_host_graph_on_emulated_kernels(monkeypatch):
    """LQ frames -> frames through 3-D VAE encode + DiT + sampler + 3-D VAE decode (reduced sizes, 4 steps) against the same chain of
    reference modules (tests/golden/reference_checks.pt: the final latent, and the frames at the seeded sample positions)"""
    import os
    from oracle import kernel_ref as KR
    from star_b200 import ops
    from star_b200.cogvideox import sample_sr
    from star_b200.cogvideox.vae3d import ContextParallelDecoder3D, ContextParallelEncoder3D
    from tests.test_cogvideox import SMALL_DIT, _dit_net, dit_inputs
    from tests.test_cogvideox_vae import SMALL, decoder_state_dict, encoder_state_dict, sample_positions
    for name in dir(KR):
        if not name.startswith("_") and callable(getattr(KR, name)) and hasattr(ops, name):
            monkeypatch.setattr(ops, name, getattr(KR, name))
    gold = torch.load(os.path.join(os.path.dirname(__file__), "golden", "reference_checks.pt"))
    net = _dit_net(SMALL_DIT, gold["dit_small"], torch.float16, "cpu")
    _, _, ctx = dit_inputs(SMALL_DIT, "cpu")
    dec, enc = ContextParallelDecoder3D(**SMALL), ContextParallelEncoder3D(**SMALL)
    dec.load_state_dict(decoder_state_dict(dec.state_dict()))
    enc.load_state_dict(encoder_state_dict(enc.state_dict()))
    dec, enc = dec.to(dtype=torch.float16).eval(), enc.to(dtype=torch.float16).eval()
    cond, uc, lq = pipeline_case(ctx)
    want = gold["pipeline"]
    got, z = sample_sr(net, dec, cond, uc, lq=lq, encoder=enc, num_steps=4, seed=77)
    assert tuple(got.shape) == want["shape"] == (1, 9, 3, 64, 96)
    assert rel_l2(z, want["z"]) < 1e-2 and rel_l2(got.flatten()[sample_positions(got.numel())], want["frames"]) < 1e-2


@pytest.mark.gpu
@pytest.mark.reference
def test_cogvideox_pipeline_gpu():
    """the same chain on the GPU kernels: full-width DiT (2 layers), full-width 3-D VAE decoder, 6 sampler steps, fp16"""
    from oracle.cogvideox_vae import vae_reference_available
    from oracle.cogvideox_sampler import sampler_reference_available
    from star_b200.cogvideox import sample_sr
    if not (vae_reference_available() and sampler_reference_available()):
        pytest.skip("reference files not staged")
    kw = dict(num_layers=2, hidden_size=3072, num_attention_heads=48, num_frames=17, latent_height=16, latent_width=24,
              text_length=226, text_hidden_size=4096, lora_r=64, time_embed_dim=512)
    ref_dit, net, ref_vae, (enc, dec), ctx = _pipeline_pair(kw, {}, torch.float16, "cuda")
    cond, uc = {"crossattn": ctx[:1]}, {"crossattn": torch.zeros_like(ctx[:1])}
    lq = (torch.rand(1, 17, 3, 128, 192, generator=torch.Generator().manual_seed(9)) * 2 - 1).cuda()
    want, z_ref = _reference_pipeline(ref_dit, ref_vae, cond, uc, lq, steps=6, seed=5)
    got, z = sample_sr(net, dec, cond, uc, lq=lq, encoder=enc, num_steps=6, seed=5)
    e_z, e_x = rel_l2(z, z_ref), rel_l2(got, want)
    print(f"[cogvideox pipeline fp16, 6 steps] latent rel-L2 {e_z:.2e}, frames rel-L2 {e_x:.2e}")
    assert got.shape == want.shape == (1, 17, 3, 128, 192) and torch.isfinite(got).all()
    assert e_z < 2e-2 and e_x < 2e-2


# ---------------------------------------------------------------------------------------------------- 2 ranks (gloo, CPU)
def _split_worker(rank, world, port, q):
    import os
    import torch.distributed as dist
    from star_b200.cogvideox.sampling import VPSDEDPMPP2MSampler, split_cfg_pair
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        g = torch.Generator().manual_seed(0)
        lq = torch.randn(1, 3, 16, 6, 8, generator=g)
        randn = torch.randn(1, 3, 16, 6, 8, generator=g)
        cond, uc = {"crossattn": torch.randn(1, 226, 32, generator=g)}, {"crossattn": torch.zeros(1, 226, 32)}
        net = FakeDiT()
        torch.manual_seed(123)
        out = VPSDEDPMPP2MSampler(num_steps=6, dtype=torch.float32)(split_cfg_pair(net), randn, cond, uc=uc, lq=torch.cat((lq, lq), 0))
        q.put((rank, out.numpy(), len(net.calls)))
    finally:
        dist.destroy_process_group()


def test_cfg_pair_split_two_ranks_equals_single():
    """CogVideoX multi-GPU axis: the CFG pair over 2 ranks (one all-gather per step) == the batch-2 run, bit for bit, on both ranks"""
    import socket
    import torch.multiprocessing as mp
    from star_b200.cogvideox.sampling import VPSDEDPMPP2MSampler
    g = torch.Generator().manual_seed(0)
    lq = torch.randn(1, 3, 16, 6, 8, generator=g)
    randn = torch.randn(1, 3, 16, 6, 8, generator=g)
    cond, uc = {"crossattn": torch.randn(1, 226, 32, generator=g)}, {"crossattn": torch.zeros(1, 226, 32)}
    torch.manual_seed(123)
    single = VPSDEDPMPP2MSampler(num_steps=6, dtype=torch.float32)(FakeDiT(), randn, cond, uc=uc, lq=torch.cat((lq, lq), 0))
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_split_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=120) for _ in procs], key=lambda t: t[0])
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for rank, out, ncalls in res:
        assert ncalls == 6                                                     # one single-branch forward per step and rank
        assert torch.equal(torch.from_numpy(out), single)
