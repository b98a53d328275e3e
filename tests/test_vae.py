"""Temporal VAE (rows a3 / a16).  PARITY UNPINNED: the oracle (oracle/temporal_vae_ref.py) restates the published
diffusers 0.30.0 architecture; diffusers itself is not available to pin it."""
import pytest
import torch

from tests.util import rel_l2

SMALL = dict(block_out_channels=(64, 64, 128, 128), layers_per_block=2)


def _setup(cfg_kw, seed=5, device="cpu"):
    from oracle.temporal_vae_ref import VaeCfg, vae_manifest
    from star_b200.utils.synth import synth_state_dict
    from star_b200.video_to_video.modules.temporal_vae import AutoencoderKLTemporalDecoder
    cfg = VaeCfg(**cfg_kw)
    sd = synth_state_dict(vae_manifest(cfg), seed=seed)
    for k in sd:                                   # distinct, non-trivial blend factors
        if k.endswith("mix_factor"):
            sd[k] = sd[k] * 50.0
    vae = AutoencoderKLTemporalDecoder(**cfg_kw)
    vae.load_state_dict(sd)
    vae = vae.eval().to(device)
    return cfg, sd, vae


def _patch(monkeypatch):
    from oracle import kernel_ref as KR
    from star_b200 import ops
    for name in dir(KR):
        if not name.startswith("_") and callable(getattr(KR, name)) and hasattr(ops, name):
            monkeypatch.setattr(ops, name, getattr(KR, name))


def test_checkpoint_layout_matches_oracle_manifest():
    from oracle.temporal_vae_ref import VaeCfg, vae_manifest
    from star_b200.video_to_video.modules.temporal_vae import AutoencoderKLTemporalDecoder
    with torch.device("meta"):
        vae = AutoencoderKLTemporalDecoder()
    got = {k: tuple(v.shape) for k, v in vae.state_dict().items()}
    want = {k: tuple(v) for k, v in vae_manifest(VaeCfg()).items()}
    assert got == want

    def count(pred):
        return sum(torch.Size(s).numel() for k, s in got.items() if pred(k))

    # known-answer: the image parts are the SD-1.x AutoencoderKL (83 653 863 parameters = encoder 34 163 592 +
    # decoder 49 490 179 + quant_conv 72 + post_quant_conv 20); the temporal decoder adds (3,1,1) blocks on top
    assert count(lambda k: k.startswith("encoder.")) == 34_163_592
    assert count(lambda k: k.startswith("quant_conv")) == 72
    assert count(lambda k: k.startswith("decoder.") and "temporal_res_block" not in k and "mix_factor" not in k
                 and "time_conv_out" not in k) == 49_490_179
    assert vae.config.scaling_factor == 0.18215


def test_decode_host_graph_on_emulated_kernels(monkeypatch):
    from oracle.temporal_vae_ref import decode
    _patch(monkeypatch)
    cfg, sd, vae = _setup(SMALL)
    z = torch.randn(6, 4, 4, 6, generator=torch.Generator().manual_seed(1))          # 2 windows of 3 frames
    ref = decode(sd, z, 3, cfg)
    got = vae.decode(z, num_frames=3).sample
    assert got.shape == (6, 3, 32, 48) and got.dtype == torch.float16
    assert rel_l2(got, ref) < 3e-3
    one = vae.decode(z[:3], num_frames=3).sample                                     # windows are independent
    assert rel_l2(one, ref[:3]) < 3e-3
    short = vae.decode(z[:2], num_frames=2).sample                                   # last window of a clip can be shorter
    assert rel_l2(short, decode(sd, z[:2], 2, cfg)) < 3e-3


def test_encode_host_graph_on_emulated_kernels(monkeypatch):
    from oracle.temporal_vae_ref import encode_moments, sample_posterior
    _patch(monkeypatch)
    cfg, sd, vae = _setup(SMALL)
    x = torch.rand(2, 3, 32, 48, generator=torch.Generator().manual_seed(2)) * 2 - 1
    ref = encode_moments(sd, x, cfg)
    dist = vae.encode(x).latent_dist
    assert dist.parameters.shape == (2, 8, 4, 6)
    assert rel_l2(dist.parameters, ref) < 3e-3
    g1, g2 = torch.Generator().manual_seed(9), torch.Generator().manual_seed(9)
    noise = torch.randn(dist.mean.shape, generator=g2)
    assert torch.allclose(dist.sample(generator=g1), sample_posterior(dist.parameters, noise), atol=1e-6)


def test_pipeline_uses_vae_surface(monkeypatch):
    """vae_encode / vae_decode_chunk of the pipeline (ref video_to_video_model.py:141-161) against the oracle"""
    from oracle.temporal_vae_ref import decode, encode_moments
    from star_b200.video_to_video.video_to_video_model import VideoToVideo_sr
    _patch(monkeypatch)
    cfg, sd, vae = _setup(SMALL)
    pipe = VideoToVideo_sr.__new__(VideoToVideo_sr)
    pipe.vae, pipe.device = vae, torch.device("cpu")
    z = torch.randn(1, 4, 5, 4, 6, generator=torch.Generator().manual_seed(3))      # 5 frames -> windows of 3 + 2
    vid = pipe.vae_decode_chunk(z, chunk_size=3)
    zz = z[0].permute(1, 0, 2, 3) / cfg.scaling_factor
    ref = torch.cat([decode(sd, zz[:3], 3, cfg), decode(sd, zz[3:], 2, cfg)])
    assert rel_l2(vid, ref) < 3e-3
    x = torch.rand(1, 2, 3, 32, 48, generator=torch.Generator().manual_seed(4)) * 2 - 1
    torch.manual_seed(0)
    lat = pipe.vae_encode(x)
    assert lat.shape == (1, 4, 2, 4, 6)
    mean = encode_moments(sd, x[0], cfg)[:, :4] * cfg.scaling_factor
    assert (lat[0].permute(1, 0, 2, 3) - mean).abs().max() < 1.0                    # sample = mean + small std * noise


def test_oracle_matches_diffusers():
    diffusers = pytest.importorskip("diffusers", reason="diffusers is not installed: VAE oracle parity unpinned")
    from oracle.temporal_vae_ref import VaeCfg, decode, encode_moments, vae_manifest
    from star_b200.utils.synth import synth_state_dict
    kw = dict(SMALL)
    real = diffusers.AutoencoderKLTemporalDecoder(block_out_channels=kw["block_out_channels"], layers_per_block=2)
    cfg = VaeCfg(**kw)
    sd = synth_state_dict(vae_manifest(cfg), seed=5)
    real.load_state_dict(sd)
    real.eval()
    z = torch.randn(3, 4, 4, 6)
    x = torch.rand(1, 3, 32, 48) * 2 - 1
    with torch.no_grad():
        assert rel_l2(decode(sd, z, 3, cfg), real.decode(z, num_frames=3).sample) < 1e-5
        assert rel_l2(encode_moments(sd, x, cfg), real.encode(x).latent_dist.parameters) < 1e-5


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["small", "full_width"])
def test_decode_gpu(case):
    from oracle.temporal_vae_ref import decode
    kw = SMALL if case == "small" else {}
    cfg, sd, vae = _setup(kw, device="cuda")
    h, w = (10, 12) if case == "small" else (14, 16)
    z = torch.randn(3, 4, h, w, generator=torch.Generator().manual_seed(1))
    sdc = {k: v.cuda() for k, v in sd.items()}
    ref = decode(sdc, z.cuda(), 3, cfg)
    got = vae.decode(z.cuda(), num_frames=3).sample
    torch.cuda.synchronize()
    err = rel_l2(got, ref)
    print(f"temporal VAE decode [{case}] latent {h}x{w}: rel-L2 vs fp32 oracle {err:.3e}")
    assert got.shape == (3, 3, 8 * h, 8 * w) and err < 4e-3


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["small", "full_width"])
def test_encode_gpu(case):
    from oracle.temporal_vae_ref import encode_moments
    kw = SMALL if case == "small" else {}
    cfg, sd, vae = _setup(kw, device="cuda")
    H, W = (80, 96) if case == "small" else (112, 128)
    x = torch.rand(2, 3, H, W, generator=torch.Generator().manual_seed(2)) * 2 - 1
    sdc = {k: v.cuda() for k, v in sd.items()}
    ref = encode_moments(sdc, x.cuda(), cfg)
    got = vae.encode(x.cuda()).latent_dist.parameters
    torch.cuda.synchronize()
    err = rel_l2(got, ref)
    print(f"temporal VAE encode [{case}] {H}x{W}: rel-L2 vs fp32 oracle {err:.3e}")
    assert got.shape == (2, 8, H // 8, W // 8) and err < 4e-3


@pytest.mark.gpu
def test_pixel_pipeline_gpu():
    """VideoToVideo_sr.test() end to end on the GPU (row a1) AGAINST THE ORACLE: the same entry is run twice, once on
    the product members (sm_90a UNet + temporal VAE, fused bilinear+pad and CFG kernels) and once on oracle members (fp32
    restatements: oracle/unet_ref.py -- pinned to the reference -- and oracle/temporal_vae_ref.py -- unpinned) with the
    same seed, so both consume identical posterior / diffuse / SDE noise.  Bilinear x2 upscale + pad_to_fit (720x1280
    canvas -> latent 90x160), per-frame encode, 4-step 'normal' sampler with CFG 7.5, 3-frame decode windows, crop."""
    from types import SimpleNamespace
    from oracle import temporal_vae_ref as VR
    from oracle.unet_ref import UNetCfg, controlled_unet_forward
    from tests.util import SMALL_KW, synth_model
    from star_b200.video_to_video.utils.seed import setup_seed
    from star_b200.video_to_video.video_to_video_model import VideoToVideo_sr
    net, sd_unet = synth_model(SMALL_KW, seed=1, device="cuda")
    cfg, sd_vae, vae = _setup(SMALL, device="cuda")
    sd_unet = {k: v.cuda() for k, v in sd_unet.items()}
    sd_vae = {k: v.cuda() for k, v in sd_vae.items()}
    g = torch.Generator().manual_seed(7)
    emb = torch.randn(1, 77, 1024, generator=g).cuda()

    class Text:
        def __call__(self, s):
            return emb if s == "a prompt" else -emb

    class OracleVAE:
        config = SimpleNamespace(scaling_factor=0.18215)

        def encode(self, x):
            m = VR.encode_moments(sd_vae, x.float(), cfg)
            return SimpleNamespace(latent_dist=SimpleNamespace(
                sample=lambda: VR.sample_posterior(m, torch.randn(m[:, :4].shape, device=m.device, dtype=m.dtype))))

        def decode(self, z, num_frames):
            return SimpleNamespace(sample=VR.decode(sd_vae, z.float(), num_frames, cfg))

    class OracleUNet(torch.nn.Module):
        def forward(self, x, t, y, hint=None, hint_chunk=None, variant_info=None):
            return controlled_unet_forward(sd_unet, x.float(), t, y.float(), (hint_chunk if hint_chunk is not None else hint).float(),
                                           UNetCfg(**SMALL_KW))

        def half(self):
            return self

    class Opt:
        model_path = None

    video = torch.rand(4, 3, 64, 96, generator=g) * 2 - 1
    inp = {"video_data": video, "y": "a prompt", "target_res": (128, 192)}
    kw = dict(steps=4, solver_mode="normal", guide_scale=7.5, max_chunk_len=32)
    star = VideoToVideo_sr(Opt(), device=torch.device("cuda"), text_encoder=Text(), vae=vae, generator=net)
    outs = []
    for _ in range(2):
        setup_seed(666)
        outs.append(star.test(inp, **kw))
    out = outs[0]
    assert out.shape == (1, 3, 4, 128, 192) and out.dtype == torch.float32 and out.device.type == "cpu"
    assert torch.isfinite(out).all()
    assert torch.equal(outs[0], outs[1])            # same seed -> same video (posterior sample, diffuse noise, SDE noise)
    oracle = VideoToVideo_sr(Opt(), device=torch.device("cuda"), text_encoder=Text(), vae=OracleVAE(), generator=OracleUNet())
    with torch.autocast("cuda", enabled=False):
        setup_seed(666)
        ref = oracle.test(inp, **kw)
    err = rel_l2(out, ref)
    print(f"pixel pipeline (4 frames, 64x96 -> 128x192, 4 solver steps, CFG 7.5): rel-L2 vs the fp32 oracle pipeline {err:.3e}")
    # test() + the CLI's tensor2vid / adain_color_fix with the post-processing on the GPU (uint8 frames back)
    from oracle import kernel_ref as KR
    setup_seed(666)
    frames = star.enhance_frames(inp, **kw)
    want = KR.adain_color_fix(out, video, uint8=True)
    assert frames.shape == (4, 128, 192, 3) and frames.dtype == torch.uint8 and frames.device.type == "cpu"
    assert (frames.int() - want.int()).abs().max().item() <= 1
    assert err <= 3e-2              # CFG 7.5 amplifies the two branches' fp16 error over the solver steps; layout / window / crop bugs give O(1)


def test_vae_weights_lookup_and_from_pretrained(tmp_path, monkeypatch):
    """from_pretrained reads a diffusers-layout directory; the pipeline finds it via opt / env / the HF cache layout"""
    import json
    from types import SimpleNamespace
    from safetensors.torch import save_file
    from star_b200.video_to_video.modules.temporal_vae import AutoencoderKLTemporalDecoder
    from star_b200.video_to_video.video_to_video_model import _find_vae_dir
    cfg, sd, _ = _setup(SMALL)
    snap = tmp_path / "hub" / "models--stabilityai--stable-video-diffusion-img2vid" / "snapshots" / "abc" / "vae"
    snap.mkdir(parents=True)
    (snap / "config.json").write_text(json.dumps({"_class_name": "AutoencoderKLTemporalDecoder", "block_out_channels": [64, 64, 128, 128],
                                                  "layers_per_block": 2, "latent_channels": 4, "scaling_factor": 0.18215,
                                                  "down_block_types": ["DownEncoderBlock2D"] * 4}))
    save_file({k: v.half().contiguous() for k, v in sd.items()}, str(snap / "diffusion_pytorch_model.fp16.safetensors"))
    monkeypatch.delenv("STAR_VAE_PATH", raising=False)
    monkeypatch.setenv("HF_HUB_CACHE", str(tmp_path / "hub"))
    assert _find_vae_dir(SimpleNamespace(model_path="x")) == str(snap)
    monkeypatch.setenv("STAR_VAE_PATH", "/somewhere/else")
    assert _find_vae_dir(SimpleNamespace(model_path="x")) == "/somewhere/else"
    assert _find_vae_dir(SimpleNamespace(vae_path="/explicit")) == "/explicit"
    vae = AutoencoderKLTemporalDecoder.from_pretrained(str(snap), variant="fp16")
    got = vae.state_dict()
    assert set(got) == set(sd) and all(torch.equal(got[k].float(), sd[k].half().float()) for k in sd)
    assert vae.config.block_out_channels == (64, 64, 128, 128)
