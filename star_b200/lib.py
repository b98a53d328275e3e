"""ctypes binding of libstar_sm100.so (C ABI: include/star_sm100.h).

The library is the only compute backend of star_b200: there is no CPU or
PyTorch fallback.  ``get_lib()`` raises if the shared object is missing and
``ensure_init()`` raises if no sm_90 (H100) device is available.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libstar_sm100.so")              # fp16 tokens (I2VGen-XL path, VAE)
LIB_PATH_BF16 = os.path.join(_HERE, "libstar_sm100_bf16.so")    # the same sources built with -DSTAR_BF16 (CogVideoX DiT)

_p, _ll, _i, _f = ctypes.c_void_p, ctypes.c_longlong, ctypes.c_int, ctypes.c_float

# name -> (restype, argtypes); mirrors include/star_sm100.h one to one
SIGNATURES = {
    "star_version": (_i, []),
    "star_last_error": (ctypes.c_char_p, []),
    "star_launch_count": (_ll, []),
    "star_init": (_i, [_i]),
    "star_linear": (_i, [_p, _ll, _p, _p, _p, _ll, _p, _ll, _p, _ll, _ll, _i, _i, _i, _p]),
    "star_linear_ex": (_i, [_p, _ll, _p, _p, _p, _ll, _p, _p, _ll, _p, _ll, _ll, _i, _i, _i, _i, _ll, _p]),
    "star_row_gate": (_i, [_p, _p, _ll, _i, _i, _p, _f, _f, _p]),
    "star_qk_ln_rope": (_i, [_p, _ll, _ll, _i, _i, _p, _p, _p, _p, _p, _p, _i, _i, _f, _p]),
    "star_conv2d_3x3": (_i, [_p, _p, _p, _p, _ll, _ll, _p, _ll, _p, _ll, _i, _i, _i, _i, _i, _i, _i, _p]),
    "star_conv2d_s2_workspace_bytes": (_ll, [_i, _i, _i, _i]),
    "star_conv2d_3x3_s2": (_i, [_p, _p, _p, _p, _ll, _p, _i, _i, _i, _i, _i, _p]),
    "star_conv_t3": (_i, [_p, _p, _p, _p, _ll, _p, _ll, _i, _i, _ll, _ll, _ll, _i, _i, _p]),
    "star_conv3d_causal": (_i, [_p, _p, _p, _p, _ll, _p, _ll, _i, _i, _i, _i, _i, _p]),
    "star_conv2d_c4_workspace_bytes": (_ll, [_i, _i, _i, _i]),
    "star_conv2d_3x3_c4": (_i, [_p, _p, _p, _p, _p, _p, _i, _i, _i, _i, _p]),
    "star_attention": (_i, [_p, _ll, _p, _ll, _p, _ll, _p, _ll, _i, _i, _i, _i, _i, _f, _p]),
    "star_attention_causal": (_i, [_p, _ll, _p, _ll, _p, _ll, _p, _ll, _i, _i, _i, _f, _p]),
    "star_temporal_attention": (_i, [_p, _ll, _p, _ll, _i, _i, _ll, _i, _i, _f, _p]),
    "star_groupnorm_workspace_bytes": (_ll, [_i, _i]),
    "star_groupnorm": (_i, [_p, _p, _p, _p, _i, _ll, _i, _f, _i, _ll, _ll, _ll, _i, _p, _p]),
    "star_groupnorm_mod": (_i, [_p, _p, _p, _p, _p, _ll, _p, _i, _i, _i, _i, _i, _i, _i, _f, _i, _p, _p]),
    "star_layernorm": (_i, [_p, _p, _p, _p, _ll, _i, _f, _i, _p, _f, _f, _p]),
    "star_liem_spatial_gate": (_i, [_p, _p, _p, _p, _i, _i, _i, _i, _ll, _ll, _p]),
    "star_concat_add": (_i, [_p, _i, _p, _p, _i, _p, _ll, _p]),
    "star_add": (_i, [_p, _p, _p, _ll, _p]),
    "star_time_avgpool2": (_i, [_p, _p, _i, _ll, _i, _p]),
    "star_upsample2x_crop": (_i, [_p, _p, _i, _i, _i, _i, _p]),
    "star_upsample2x": (_i, [_p, _p, _i, _i, _i, _i, _i, _p]),
    "star_softmax_rows": (_i, [_p, _ll, _ll, _i, _i, _p]),
    "star_vae_head": (_i, [_p, _ll, _p, _p, _p, _i, _i, _ll, _p]),
    "star_conv2d_s2p_workspace_bytes": (_ll, [_i, _i, _i, _i, _i, _i, _i, _i]),
    "star_conv2d_3x3_s2p": (_i, [_p, _p, _p, _p, _ll, _p, _i, _i, _i, _i, _i, _i, _i, _i, _i, _p]),
    "star_nchw5_to_tokens": (_i, [_p, _p, _i, _i, _i, _ll, _p]),
    "star_tokens_to_nchw5": (_i, [_p, _ll, _p, _i, _i, _i, _ll, _p]),
    "star_bilinear_pad": (_i, [_p, _p, _ll, _i, _i, _i, _i, _i, _i, _i, _i, _f, _p]),
    "star_adain_workspace_bytes": (_ll, [_i, _i]),
    "star_adain_color_fix": (_i, [_p, _p, _p, _p, _i, _i, _ll, _ll, _p, _p]),
    "star_cfg_x0_workspace_bytes": (_ll, [_i]),
    "star_cfg_x0": (_i, [_p, _p, _p, _p, _p, _f, _f, _p, _p, _i, _ll, _p, _p]),
    "star_cfg_x0_blend": (_i, [_p, _p, _p, _p, _f, _f, _p, _p, _p, _p] + [_i] * 13 + [_p, _p]),
    "star_sinusoidal": (_i, [_p, _p, _i, _i, _p]),
    "star_silu": (_i, [_p, _p, _ll, _p]),
}

_libs = {}
_inited = set()


class StarError(RuntimeError):
    pass


def _key(dtype):
    return "bf16" if dtype is not None and str(dtype).endswith("bfloat16") else "fp16"


def get_lib(dtype=None):
    """The kernel library for fp16 tokens (default) or bf16 tokens (dtype = torch.bfloat16)."""
    key = _key(dtype)
    lib = _libs.get(key)
    if lib is None:
        path = LIB_PATH_BF16 if key == "bf16" else LIB_PATH
        if not os.path.isfile(path):
            raise StarError(
                f"{path} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(nvcc, sm_90a). star_b200 has no fallback compute path.")
        lib = ctypes.CDLL(path)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)
            fn.restype = res
            fn.argtypes = args
        _libs[key] = lib
    return lib


def check(L, rc, what):
    """Raises StarError with library L's message for the failed call ``what`` (rc != 0)."""
    if rc != 0:
        raise StarError(f"{what}: {L.star_last_error().decode(errors='replace')}")


def ensure_init(device_index, dtype=None):
    key = (_key(dtype), device_index)
    if key in _inited:
        return
    L = get_lib(dtype)
    check(L, L.star_init(int(device_index)), "star_init failed")
    _inited.add(key)


def launch_count():
    """Kernels launched by the loaded libraries since load (the fp16 one is loaded if none is)."""
    return sum(L.star_launch_count() for L in _libs.values()) if _libs else get_lib().star_launch_count()
