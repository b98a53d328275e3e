"""CogVideoX 3-D causal VAE decoder (SURVEY 8 row f4) against the reference's UNMODIFIED cp_enc_dec.py
(oracle/cogvideox_vae.py: context-parallel size 1, SafeConv3d = Conv3d); the CPU tests read the reference outputs from
tests/golden/reference_checks.pt (oracle/make_golden_reference.py)."""
import os

import pytest
import torch

from tests.util import assert_close, rel_l2

SMALL = dict(ch=32, ch_mult=(1, 2, 2, 4), num_res_blocks=1)          # 32..128 channels, same topology as the shipped decoder
GOLD = os.path.join(os.path.dirname(__file__), "golden", "reference_checks.pt")


def sample_positions(numel, n=16384):
    """fixed, seeded sample of flat positions at which large reference outputs are stored"""
    return torch.randperm(numel, generator=torch.Generator().manual_seed(0))[:min(n, numel)]


def decoder_state_dict(shapes_of, seed=3):
    from star_b200.utils.synth import synth_state_dict
    sd = synth_state_dict({k: tuple(v.shape) for k, v in shapes_of.items()}, seed=seed)
    for k in sd:                                    # conv_y multiplies the normalised features: keep it O(1), not O(1/sqrt(16))
        if ".conv_y.conv.bias" in k:
            sd[k] = sd[k] + 1.0
    return sd


def encoder_state_dict(shapes_of, seed=6):
    from star_b200.utils.synth import synth_state_dict
    return synth_state_dict({k: tuple(v.shape) for k, v in shapes_of.items()}, seed=seed)


def enc_inputs():
    x = torch.rand(1, 3, 9, 32, 48, generator=torch.Generator().manual_seed(3)) * 2 - 1
    even = torch.rand(1, 3, 8, 16, 16, generator=torch.Generator().manual_seed(4)) * 2 - 1      # even T: plain pair pooling
    return x, even


def _pair(kw, seed=3, device="cpu", dtype=torch.float16):
    from oracle.cogvideox_vae import build_reference_decoder
    from star_b200.cogvideox.vae3d import ContextParallelDecoder3D
    ref = build_reference_decoder(**kw)
    sd = decoder_state_dict(ref.state_dict(), seed)
    ref.load_state_dict(sd)
    mine = ContextParallelDecoder3D(**kw)
    mine.load_state_dict(sd)
    return ref.to(device), mine.to(device=device, dtype=dtype).eval(), sd


def _enc_pair(kw, seed=6, device="cpu", dtype=torch.float16):
    from oracle.cogvideox_vae import build_reference_encoder
    from star_b200.cogvideox.vae3d import ContextParallelEncoder3D
    ref = build_reference_encoder(**kw)
    sd = encoder_state_dict(ref.state_dict(), seed)
    ref.load_state_dict(sd)
    mine = ContextParallelEncoder3D(**kw)
    mine.load_state_dict(sd)
    return ref.to(device), mine.to(device=device, dtype=dtype).eval(), sd


def _patch(monkeypatch):
    from oracle import kernel_ref as KR
    from star_b200 import ops
    for name in dir(KR):
        if not name.startswith("_") and callable(getattr(KR, name)) and hasattr(ops, name):
            monkeypatch.setattr(ops, name, getattr(KR, name))


def test_state_dict_layout_matches_reference():
    """decoder and encoder state-dict layouts == the reference modules' (tests/golden/reference_checks.pt)"""
    import os
    from star_b200.cogvideox.vae3d import ContextParallelDecoder3D, ContextParallelEncoder3D
    gold = torch.load(os.path.join(os.path.dirname(__file__), "golden", "reference_checks.pt"))["vae_layout"]
    with torch.device("meta"):
        mine, enc = ContextParallelDecoder3D(), ContextParallelEncoder3D()
    got = {k: tuple(v.shape) for k, v in mine.state_dict().items()}
    assert got == gold["decoder"]
    assert sum(torch.Size(s).numel() for s in got.values()) == gold["decoder_params"]
    assert {k: tuple(v.shape) for k, v in enc.state_dict().items()} == gold["encoder"]


def test_decoder_host_graph_on_emulated_kernels(monkeypatch):
    """3 + 2 + 2 latent frames through the reference's chunk protocol (sample_sr.py:212-227): odd / even clip lengths, the
    first-frame split of SpatialNorm3D and Upsample3D, and the causal-conv context carried between chunks.  The reference
    outputs are stored at sample_positions()."""
    from star_b200.cogvideox.vae3d import ContextParallelDecoder3D
    _patch(monkeypatch)
    gold = torch.load(GOLD)["vae_chunks"]
    mine = ContextParallelDecoder3D(**SMALL)
    mine.load_state_dict(decoder_state_dict(mine.state_dict()))
    mine = mine.to(dtype=torch.float16).eval()
    z = torch.randn(1, 16, 7, 4, 6, generator=torch.Generator().manual_seed(0))
    got = mine.decode_latent(z)
    assert got.shape == gold["shape"] == (1, 3, 25, 32, 48) and got.dtype == torch.float16
    assert rel_l2(got.flatten()[sample_positions(got.numel())], gold["full"]) < 3e-3
    assert not mine._cache                                                    # the last chunk clears the context
    # a chunk decoded alone (clear cache) replicates its first frame instead of using context
    alone = mine(z[:, :, 3:5].contiguous())
    pos = sample_positions(alone.numel())
    assert tuple(alone.shape) == gold["alone_shape"]
    assert rel_l2(alone.flatten()[pos], gold["alone"]) < 3e-3
    assert rel_l2(got[:, :, 9:17].flatten()[pos], gold["alone"]) > 1e-2     # ... and that differs from the chunked result


def test_encoder_host_graph_on_emulated_kernels(monkeypatch):
    """9 frames of 32x48 -> moments (1, 32, 3, 4, 6): odd clip lengths through both time-compressing DownSample3D levels
    (9 -> 5 -> 3), the (0,1,0,1)-padded stride-2 convs, clip-wide GroupNorm, first-frame replication of the causal convs
    (reference moments from tests/golden/reference_checks.pt)"""
    from star_b200.cogvideox.vae3d import ContextParallelEncoder3D
    _patch(monkeypatch)
    gold = torch.load(GOLD)
    with torch.device("meta"):
        assert {k: tuple(v.shape) for k, v in ContextParallelEncoder3D().state_dict().items()} == gold["vae_layout"]["encoder"]
    mine = ContextParallelEncoder3D(**SMALL)
    mine.load_state_dict(encoder_state_dict(mine.state_dict()))
    mine = mine.to(dtype=torch.float16).eval()
    x, even = enc_inputs()
    want = gold["vae_enc"]["odd"]
    got = mine(x)
    assert got.shape == want.shape == (1, 32, 3, 4, 6)
    assert rel_l2(got, want) < 3e-3
    assert rel_l2(mine(even), gold["vae_enc"]["even"]) < 3e-3
    torch.manual_seed(0)
    z = mine.encode(x)
    torch.manual_seed(0)
    mean, logvar = got.float().chunk(2, dim=1)
    assert torch.allclose(z.float(), mean + torch.exp(0.5 * logvar.clamp(-30, 20)) * torch.randn_like(got[:, :16], dtype=torch.float32), atol=1e-2)


def test_spatial_norm_index_rule():
    """row -> latent-row map of star_groupnorm_mod == F.interpolate(nearest) with the reference's first-frame split"""
    import torch.nn.functional as F
    from oracle.kernel_ref import spatial_norm_src_index
    for (T, Tl) in ((9, 3), (5, 3), (3, 3), (8, 2), (4, 2), (2, 2), (1, 1)):
        H, W, Hl, Wl = 8, 12, 4, 6
        zq = torch.arange(Tl * Hl * Wl, dtype=torch.float32).reshape(1, 1, Tl, Hl, Wl)
        if T > 1 and T % 2 == 1:
            a = F.interpolate(zq[:, :, :1], size=(1, H, W), mode="nearest")
            b = F.interpolate(zq[:, :, 1:], size=(T - 1, H, W), mode="nearest")
            want = torch.cat([a, b], dim=2)
        else:
            want = F.interpolate(zq, size=(T, H, W), mode="nearest")
        got = spatial_norm_src_index(T, H, W, Tl, Hl, Wl, "cpu")
        assert torch.equal(got, want.reshape(-1).long())


# ---------------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def env():
    from star_b200 import ops
    from oracle import kernel_ref as KR
    return ops, KR


@pytest.mark.gpu
@pytest.mark.parametrize("T,H,W,Cin,Cout,res", [(3, 12, 20, 64, 128, False), (9, 30, 44, 128, 128, True), (2, 60, 90, 256, 128, True),
                                                 (8, 17, 23, 64, 3, False), (3, 60, 90, 512, 512, True)])
def test_conv3d_causal(env, T, H, W, Cin, Cout, res):
    ops, KR = env
    g = torch.Generator(device="cuda").manual_seed(T * 100 + Cin)
    xp = torch.randn((T + 2) * H * W, Cin, device="cuda", generator=g).half()
    w = (torch.randn(Cout, 3, 3, 3, Cin, device="cuda", generator=g) * (27 * Cin) ** -0.5).half()
    b = (torch.randn(Cout, device="cuda", generator=g) * 0.1).half()
    r = torch.randn(T * H * W, Cout, device="cuda", generator=g).half() if res else None
    if Cout == 3:
        out = torch.zeros(T * H * W, 8, device="cuda", dtype=torch.float16)
        ops.conv3d_causal(xp, w, T, H, W, b, out=out[:, :3])
        got = out[:, :3]
        assert (out[:, 3:] == 0).all()
    else:
        got = ops.conv3d_causal(xp, w, T, H, W, b, residual=r)
    assert_close(got, KR.conv3d_causal(xp, w, T, H, W, b, residual=r), what="conv3d_causal")


@pytest.mark.gpu
@pytest.mark.parametrize("T,Tl,H,W,Hl,Wl,C", [(9, 3, 32, 48, 4, 6, 128), (8, 2, 32, 48, 4, 6, 256), (3, 3, 60, 90, 60, 90, 512),
                                               (5, 3, 24, 36, 12, 18, 512), (4, 2, 16, 16, 8, 8, 32), (2, 2, 12, 18, 4, 6, 64), (9, 3, 480, 720, 60, 90, 128)])
def test_groupnorm_mod(env, T, Tl, H, W, Hl, Wl, C):
    ops, KR = env
    g = torch.Generator(device="cuda").manual_seed(T + C)
    x = (torch.randn(T * H * W, C, device="cuda", generator=g) * 2 + 0.5).half()
    gam, bet = (1 + 0.1 * torch.randn(C, device="cuda", generator=g)).half(), (0.1 * torch.randn(C, device="cuda", generator=g)).half()
    mod = torch.randn(Tl * Hl * Wl, 2 * C, device="cuda", generator=g).half()
    got = ops.groupnorm_mod(x, gam, bet, mod[:, :C], mod[:, C:], T, H, W, Tl, Hl, Wl, 1e-6, True)
    assert_close(got, KR.groupnorm_mod(x, gam, bet, mod[:, :C], mod[:, C:], T, H, W, Tl, Hl, Wl, 1e-6, True), what="groupnorm_mod")


@pytest.mark.gpu
@pytest.mark.parametrize("dtype,tol", [(torch.float16, 3e-3), (torch.bfloat16, 1.6e-2)])
def test_decoder_vs_reference_gpu(dtype, tol):
    """full-width decoder (ch 128, 3 res blocks per level), 3 + 2 latent frames at 16x24 -> 17 frames of 128x192, against the
    reference's own file in fp32 (TF32 off) and beside the reference run in the same 16-bit dtype"""
    from oracle.cogvideox_vae import reference_decode_latent, vae_reference_available
    if not vae_reference_available():
        pytest.skip("reference VAE file not staged (oracle/_ref)")
    ref, mine, sd = _pair({}, device="cuda", dtype=dtype)
    z = torch.randn(1, 16, 5, 16, 24, generator=torch.Generator().manual_seed(1)).cuda()
    want = reference_decode_latent(ref, z)
    got = mine.decode_latent(z.to(dtype))
    assert got.shape == want.shape == (1, 3, 17, 128, 192)
    err = rel_l2(got, want)
    ref16 = reference_decode_latent(ref.to(dtype), z.to(dtype))
    err_ref = rel_l2(ref16, want)
    print(f"[cogvideox vae {dtype}] star {err:.2e}  reference-in-{dtype} {err_ref:.2e}")
    assert torch.isfinite(got.float()).all()
    assert err < tol and err < 1.5 * err_ref + 1e-3


@pytest.mark.gpu
@pytest.mark.parametrize("T,HW,C", [(9, 640, 128), (8, 1000, 256), (2, 77, 64), (49, 120, 128)])
def test_time_avgpool2(env, T, HW, C):
    ops, KR = env
    x = torch.randn(T * HW, C, device="cuda", generator=torch.Generator(device="cuda").manual_seed(T)).half()
    got, want = ops.time_avgpool2(x, T, HW), KR.time_avgpool2(x, T, HW)
    assert got.shape == want.shape and torch.equal(got, want)                  # one rounding of an exact fp32 sum


@pytest.mark.gpu
@pytest.mark.parametrize("dtype,tol", [(torch.float16, 3e-3), (torch.bfloat16, 1.6e-2)])
def test_encoder_vs_reference_gpu(dtype, tol):
    """full-width encoder (ch 128, 3 res blocks per level), 17 frames of 96x128 -> moments (1, 32, 5, 12, 16)"""
    from oracle.cogvideox_vae import reference_encode_moments, vae_reference_available
    if not vae_reference_available():
        pytest.skip("reference VAE file not staged (oracle/_ref)")
    ref, mine, _ = _enc_pair({}, device="cuda", dtype=dtype)
    x = (torch.rand(1, 3, 17, 96, 128, generator=torch.Generator().manual_seed(2)) * 2 - 1).cuda()
    want = reference_encode_moments(ref, x)
    got = mine(x.to(dtype))
    err = rel_l2(got, want)
    err_ref = rel_l2(reference_encode_moments(ref.to(dtype), x.to(dtype)), want)
    print(f"[cogvideox vae encoder {dtype}] star {err:.2e}  reference-in-{dtype} {err_ref:.2e}")
    assert got.shape == want.shape == (1, 32, 5, 12, 16) and torch.isfinite(got.float()).all()
    assert err < tol and err < 1.5 * err_ref + 1e-3
