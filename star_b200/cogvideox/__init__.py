"""STAR's CogVideoX-5B path (cogvideox-based/) on the sm_90a kernels: the DiT (one layer: DiTLayer; the whole
DiffusionTransformer: patch embed, 42 layers with LoRA merged, final layer), the sampling loop (VPSDEDPMPP2MSampler + DynamicCFG +
DiscreteDenoiser / VideoScaling), the 3-D causal VAE (encoder and decoder), and the frames-to-frames glue of sample_sr.py."""
from .dit_block import DiTLayer  # noqa: F401
from .model import DiffusionTransformer, dit_manifest, rope_tables  # noqa: F401
from .parallel import cogvideox_parallel, dit_shard_plan, shard_sequence  # noqa: F401
from .pipeline import sample_sr  # noqa: F401
from .sampling import StepPlan, VPSDEDPMPP2MSampler, sample_sr_latent, split_cfg_pair  # noqa: F401
from .vae3d import ContextParallelDecoder3D, ContextParallelEncoder3D  # noqa: F401
