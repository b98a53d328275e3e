"""CogVideoX-5B DiT layer (STAR's patched block).  PARITY UNPINNED: the oracle (oracle/cogvideox_ref.py) restates
STAR's layer_forward on top of sat's default leaf modules, which are not in the reference tree."""
import os

import pytest
import torch

from tests.util import rel_l2

GOLD = os.path.join(os.path.dirname(__file__), "golden", "reference_checks.pt")


def _setup(cfg_kw, seed=3):
    from oracle.cogvideox_ref import DiTCfg, layer_manifest, rope_tables
    from star_b200.utils.synth import synth_state_dict
    cfg = DiTCfg(**cfg_kw)
    sd = synth_state_dict(layer_manifest(cfg), seed=seed)
    cos, sin = rope_tables(cfg)
    g = torch.Generator().manual_seed(0)
    S = cfg.text_length + cfg.frames * cfg.height * cfg.width
    hidden = torch.randn(2, S, cfg.hidden, generator=g)
    emb = torch.randn(2, 512, generator=g)
    return cfg, sd, cos, sin, hidden, emb


def test_dit_layer_host_graph_on_emulated_kernels(monkeypatch):
    from oracle import kernel_ref as KR
    from oracle.cogvideox_ref import dit_layer_forward
    from star_b200 import ops
    from star_b200.cogvideox import DiTLayer
    for name in dir(KR):
        if not name.startswith("_") and callable(getattr(KR, name)) and hasattr(ops, name):
            monkeypatch.setattr(ops, name, getattr(KR, name))
    cfg, sd, cos, sin, hidden, emb = _setup(dict(hidden=256, heads=4, text_length=10, frames=3, height=6, width=5))
    ref = dit_layer_forward(sd, hidden, emb, cfg, cos, sin)
    layer = DiTLayer(sd, cfg.hidden, cfg.heads, cfg.text_length, cfg.frames, cfg.height, cfg.width, cfg.ln_eps,
                     cfg.qk_ln_eps, cos, sin, device="cpu")
    assert rel_l2(layer.forward(hidden, emb), ref) < 2e-3


def test_rope_tables_shape():
    from oracle.cogvideox_ref import DiTCfg, rope_tables
    cos, sin = rope_tables(DiTCfg())
    assert cos.shape == (13 * 30 * 45, 64) and torch.allclose(cos ** 2 + sin ** 2, torch.ones_like(cos), atol=1e-5)


@pytest.mark.gpu
@pytest.mark.parametrize("cfg_kw", [dict(hidden=256, heads=4, text_length=10, frames=3, height=6, width=5),
                                    dict(hidden=3072, heads=48, text_length=226, frames=2, height=6, width=10)])
def test_dit_layer_gpu(cfg_kw):
    """full-width layer (3072 / 48 heads / 226 text tokens) at a short sequence, and a small layer"""
    from oracle.cogvideox_ref import dit_layer_forward
    from star_b200.cogvideox import DiTLayer
    cfg, sd, cos, sin, hidden, emb = _setup(cfg_kw)
    ref = dit_layer_forward(sd, hidden, emb, cfg, cos, sin)
    layer = DiTLayer(sd, cfg.hidden, cfg.heads, cfg.text_length, cfg.frames, cfg.height, cfg.width, cfg.ln_eps,
                     cfg.qk_ln_eps, cos, sin, device="cuda")
    out = layer.forward(hidden.cuda(), emb.cuda())
    torch.cuda.synchronize()
    err = rel_l2(out.cpu(), ref)
    print(f"DiT layer {cfg_kw}: rel-L2 vs fp32 oracle {err:.3e}")
    assert err < 3e-3


# ------------------------------------------------------------------------------------------------------------------
# Whole DiffusionTransformer (patch embed, text proj, time embed, N layers with LoRA, final LayerNorm, final layer,
# unpatchify) against the REFERENCE'S OWN FILES executed behind the sat shim (oracle/cogvideox_sat.py): the CPU tests read
# the reference outputs from tests/golden/reference_checks.pt (oracle/make_golden_reference.py); the full-width GPU test
# needs the reference tree (oracle/_ref): marker `reference`.
SMALL_DIT = dict(num_layers=2, hidden_size=128, num_attention_heads=2, num_frames=9, latent_height=8, latent_width=12,
                 text_length=6, text_hidden_size=32, lora_r=8, time_embed_dim=64)


def dit_state_dict(rec, seed=4):
    """synthetic non-zero weights for the state-dict manifest rec["manifest"] (the reference's rotary tables rec["freqs"] as is)"""
    from star_b200.utils.synth import synth_tensor
    sd = {}
    for k, shape in rec["manifest"].items():
        if k in rec["freqs"]:
            sd[k] = rec["freqs"][k]
            continue
        t = synth_tensor(k, torch.Size(shape), seed)
        if k.endswith("temp_local.conv1.weight") or k.endswith("spa_local.conv1.weight"):
            t = t * 0.5
        if ".matrix_B." in k:                              # LoRA B is zero-initialised by sat: make the merge matter
            t = t * 8.0
        sd[k] = t
    return sd


def dit_inputs(kw, device):
    g = torch.Generator().manual_seed(1)
    frames = (kw["num_frames"] - 1) // 4 + 1
    x = torch.randn(2, frames, 32, kw["latent_height"], kw["latent_width"], generator=g).to(device)
    ctx = torch.randn(2, kw["text_length"], kw["text_hidden_size"], generator=g).to(device)
    t = torch.tensor([731, 12]).to(device)
    return x, t, ctx


def _dit_net(kw, rec, dtype, device):
    from star_b200.cogvideox import DiffusionTransformer
    net = DiffusionTransformer(**kw, dtype=dtype)
    net.load_state_dict(dit_state_dict(rec))
    return net.to(device)


def _dit_pair(kw, dtype, device):
    """(reference net with a synthetic non-zero state dict, star_b200 net with the same weights, inputs)"""
    from oracle import cogvideox_sat as S
    ref = S.build_reference_dit(**kw)
    rec = {"manifest": {k: tuple(v.shape) for k, v in ref.state_dict().items()},
           "freqs": {k: v for k, v in ref.state_dict().items() if "freqs_" in k}}
    ref.load_state_dict(dit_state_dict(rec))
    return (ref.to(device), _dit_net(kw, rec, dtype, device)) + dit_inputs(kw, device)


def test_dit_model_host_graph_vs_reference_files(monkeypatch):
    """CPU: star_b200's host graph (im2col patch embed, LoRA merge, adaLN folding, layer stack, final layer, unpatchify) on the
    emulated kernels against the reference's unmodified DiffusionTransformer (sat shimmed)."""
    from oracle import kernel_ref as KR
    from star_b200 import ops
    for name in dir(KR):
        if not name.startswith("_") and callable(getattr(KR, name)) and hasattr(ops, name):
            monkeypatch.setattr(ops, name, getattr(KR, name))
    rec = torch.load(GOLD)["dit_small"]
    net = _dit_net(SMALL_DIT, rec, torch.float16, "cpu")
    x, t, ctx = dit_inputs(SMALL_DIT, "cpu")
    want = rec["want"]
    got = net(x, timesteps=t, context=ctx)
    assert got.shape == want.shape == (2, 3, 16, 8, 12)
    err = rel_l2(got, want)
    print(f"DiT model host graph vs reference files: rel-L2 {err:.3e}")
    assert err < 3e-3


def test_restated_layer_oracle_is_pinned_to_reference_files():
    """oracle/cogvideox_ref.py (the line-by-line restatement the layer tests use) == the reference's layer_forward"""
    from oracle.cogvideox_ref import DiTCfg, dit_layer_forward
    from star_b200.cogvideox import rope_tables
    gold = torch.load(GOLD)
    rec = dict(gold["dit_layer"], freqs={k: gold["dit_small"]["freqs"][k] for k in gold["dit_layer"]["freqs"]})
    sd = dit_state_dict(rec)
    cfg = DiTCfg(hidden=128, heads=2, text_length=6, frames=3, height=4, width=6)
    lsd = {"adaLN_modulation.1.weight": sd["mixins.adaln_layer.adaLN_modulations.0.1.weight"],
           "adaLN_modulation.1.bias": sd["mixins.adaln_layer.adaLN_modulations.0.1.bias"]}
    for k, v in sd.items():
        if k.startswith("transformer.layers.0."):
            lsd[k[len("transformer.layers.0."):]] = v
    for n in ("query", "key"):
        lsd[n + "_layernorm.weight"] = sd[f"mixins.adaln_layer.{n}_layernorm_list.0.weight"]
        lsd[n + "_layernorm.bias"] = sd[f"mixins.adaln_layer.{n}_layernorm_list.0.bias"]
    g = torch.Generator().manual_seed(2)
    hidden, emb = torch.randn(2, 6 + 72, 128, generator=g), torch.randn(2, 64, generator=g)
    cos, sin = rope_tables(3, 4, 6, 64)
    want = rec["want"]
    got = dit_layer_forward(lsd, hidden, emb, cfg, cos, sin)
    assert rel_l2(got, want) < 1e-5


@pytest.mark.gpu
@pytest.mark.reference
@pytest.mark.parametrize("dtype,tol", [(torch.float16, 4e-3), (torch.bfloat16, 2.5e-2)])
def test_dit_model_gpu_vs_reference_files(dtype, tol):
    """GPU: the whole (reduced-depth, full-width) DiT on the fp16 and bf16 kernel libraries vs the reference files in fp32;
    the reference's own low-precision path (module.to(dtype), as sample_sr.py runs it) is measured beside it."""
    kw = dict(num_layers=2, hidden_size=3072, num_attention_heads=48, num_frames=9, latent_height=16, latent_width=20,
              text_length=226, text_hidden_size=4096, lora_r=64, time_embed_dim=512)
    ref, net, x, t, ctx = _dit_pair(kw, dtype, "cuda")
    want = ref(x, timesteps=t, context=ctx).float()
    got = net(x, timesteps=t, context=ctx).float()
    torch.cuda.synchronize()
    ref_lp = ref.to(dtype)
    ref_lp.dtype = dtype
    low = ref_lp(x.to(dtype), timesteps=t, context=ctx.to(dtype)).float()
    err, err_ref = rel_l2(got, want), rel_l2(low, want)
    print(f"DiT model [{dtype}] 2 layers x 3072: rel-L2 vs reference fp32 {err:.3e} (reference's own {dtype} path: {err_ref:.3e})")
    assert torch.isfinite(got).all() and err < tol and err < 2.0 * err_ref + 1e-3
