"""ctypes binding of the C ABI (include/t2v_b200.h) + in-tree build of the sm_90a shared library.

There is deliberately no fallback: if the library is missing or a call fails, a RuntimeError is raised.
"""
import ctypes
import os
import subprocess
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(_HERE, "csrc")
LIB_DIR = os.path.join(_HERE, "_native")
LIB_PATH = os.path.join(LIB_DIR, "libt2v_b200.so")
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "-shared",
]

_lib = None
_lock = threading.Lock()


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _stale():
    if not os.path.exists(LIB_PATH):
        return True
    t = os.path.getmtime(LIB_PATH)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(_HERE, "..", "include", "t2v_b200.h")]
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


def build(force=False, verbose=False):
    """Compile csrc/*.cu for sm_90a into _native/libt2v_b200.so (nvcc cross-compiles without a GPU)."""
    if not force and not _stale():
        return LIB_PATH
    os.makedirs(LIB_DIR, exist_ok=True)
    nvcc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
    cmd = [nvcc] + NVCC_FLAGS + ["-o", LIB_PATH] + sources()
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + res.stdout + res.stderr)
    if verbose:
        print(res.stderr)
    return LIB_PATH


class Epilogue(ctypes.Structure):
    _fields_ = [("bias", ctypes.c_void_p), ("rowbias", ctypes.c_void_p), ("residual", ctypes.c_void_p),
                ("alpha", ctypes.c_float), ("out_fp32", ctypes.c_int32), ("rowbias_div", ctypes.c_int32),
                ("workspace", ctypes.c_void_p), ("workspace_bytes", ctypes.c_int64),
                ("stats", ctypes.c_void_p), ("stats_ld", ctypes.c_int64), ("stats_rows", ctypes.c_int32), ("pad_", ctypes.c_int32)]


class Mat(ctypes.Structure):
    _fields_ = [("ptr", ctypes.c_void_p), ("ld", ctypes.c_int64), ("stride_z1", ctypes.c_int64),
                ("stride_z2", ctypes.c_int64), ("kmajor", ctypes.c_int32)]


class GemmProblem(ctypes.Structure):
    _fields_ = [(f, ctypes.c_int32) for f in (
        "kind", "N", "H", "W", "Cin", "Cout", "KH", "KW", "stride", "pad_h0", "pad_h1", "pad_w0", "pad_w1",
        "workspace", "stats_rows", "dbias", "gemm_m", "gemm_n", "gemm_k", "z1", "z2", "b_kmajor", "out_mode")]


class GemmPlan(ctypes.Structure):
    _fields_ = [(f, ctypes.c_int32) for f in ("block_n", "num_stages", "splits", "kb_per_split", "ksplit_var", "num_tiles", "grid")] + [
        ("box", ctypes.c_int32 * 3), ("tdim", ctypes.c_int32 * 6), ("kdim", ctypes.c_int32 * 3), ("flags", ctypes.c_int32),
        ("st", ctypes.c_int32 * 5), ("follow", ctypes.c_int32)]


class LossParams(ctypes.Structure):
    """T2VLossParams: the objective of t2v_diffusion_loss (prediction, loss form, Huber schedule, huber_c, snr_gamma)."""
    _fields_ = [("prediction", ctypes.c_int32), ("loss", ctypes.c_int32), ("huber_schedule", ctypes.c_int32),
                ("num_timesteps", ctypes.c_int32), ("huber_c", ctypes.c_float), ("snr_gamma", ctypes.c_float)]


EXPORTS = [
    "t2v_version", "t2v_last_error", "t2v_launch_count", "t2v_stream_capture_id", "t2v_channel_stats", "t2v_conv_fwd", "t2v_conv_dgrad", "t2v_conv_workspace_bytes", "t2v_conv_wgrad", "t2v_conv_wgrad_bias", "t2v_bgemm", "t2v_gemm_plan", "t2v_flash_attn_fwd", "t2v_flash_attn_bwd_splits", "t2v_flash_attn_bwd",
    "t2v_groupnorm_workspace_bytes", "t2v_groupnorm_fwd", "t2v_groupnorm_bwd", "t2v_layernorm_fwd", "t2v_layernorm_bwd",
    "t2v_latents_to_nhwc8", "t2v_nhwc8_to_latents", "t2v_mse_loss", "t2v_velocity_mse_loss", "t2v_diffusion_loss", "t2v_vae_sample", "t2v_geglu_fwd", "t2v_geglu_bwd", "t2v_silu_f32_to_bf16",
    "t2v_silu_bwd_f32", "t2v_silu_bf16", "t2v_silu_bf16_bwd", "t2v_add_bf16", "t2v_add_f32", "t2v_dropout_scale_add", "t2v_scale_bf16", "t2v_cast_f32_bf16", "t2v_embed_tokens", "t2v_embed_tokens_bwd", "t2v_gelu_bf16", "t2v_gelu_bwd_bf16", "t2v_frames_u8_to_nhwc8", "t2v_frames_u8_to_nhwc8_ragged", "t2v_scale_cast_f32_bf16", "t2v_cast_bf16_f32", "t2v_sqnorm_chunks", "t2v_adamw_prepare", "t2v_adamw_chunks", "t2v_adamw8bit_chunks", "t2v_adamw_ema_chunks", "t2v_adamw8bit_ema_chunks", "t2v_ema_swap_chunks", "t2v_counter_add", "t2v_upsample_nearest_fwd",
    "t2v_upsample_nearest_bwd", "t2v_copy_cols", "t2v_colsum", "t2v_colsum_f32", "t2v_softmax_fwd", "t2v_softmax_bwd",
    "t2v_timestep_embedding", "t2v_attn_small_fwd", "t2v_attn_small_bwd",
    "t2v_attn_long_fwd", "t2v_attn_long_bwd",
    "t2v_lora_delta_merge", "t2v_lora_delta_grad",
]


def _declare(lib):
    i32, i64, vp, f32 = ctypes.c_int32, ctypes.c_int64, ctypes.c_void_p, ctypes.c_float
    lib.t2v_version.restype = i32
    lib.t2v_last_error.restype = ctypes.c_char_p
    lib.t2v_launch_count.restype = i64
    lib.t2v_stream_capture_id.restype = i64
    lib.t2v_stream_capture_id.argtypes = [vp]
    lib.t2v_channel_stats.argtypes = [vp, vp, i32, i64, i32, i64, vp]
    conv_args = [vp, vp, vp] + [i32] * 12
    lib.t2v_conv_fwd.argtypes = conv_args + [ctypes.POINTER(Epilogue), vp]
    lib.t2v_conv_dgrad.argtypes = conv_args + [ctypes.POINTER(Epilogue), vp]
    lib.t2v_conv_wgrad.argtypes = conv_args + [vp]
    lib.t2v_conv_wgrad_bias.argtypes = [vp, vp, vp, vp] + conv_args[3:] + [vp]
    lib.t2v_conv_workspace_bytes.restype = i64
    lib.t2v_conv_workspace_bytes.argtypes = [i32] * 13
    lib.t2v_bgemm.argtypes = [ctypes.POINTER(Mat), ctypes.POINTER(Mat), vp, i64, i64, i64, i32, i32, i32, i32, i32, f32, i32, vp]
    lib.t2v_gemm_plan.argtypes = [ctypes.POINTER(GemmProblem), i32, ctypes.POINTER(GemmPlan), i32]
    lib.t2v_flash_attn_fwd.argtypes = [vp] * 5 + [i32] * 5 + [i64] * 8 + [vp]
    lib.t2v_flash_attn_bwd.argtypes = [vp] * 11 + [i32] * 5 + [i64] * 14 + [vp]
    lib.t2v_flash_attn_bwd_splits.restype = i32
    lib.t2v_flash_attn_bwd_splits.argtypes = [i32] * 4
    lib.t2v_groupnorm_workspace_bytes.restype = i64
    lib.t2v_groupnorm_workspace_bytes.argtypes = [i32, i64, i32]
    lib.t2v_groupnorm_fwd.argtypes = [vp] * 7 + [i32, i64, vp, i64, i32, vp, i32, i64, i32, i32, f32, i32, vp]
    lib.t2v_groupnorm_bwd.argtypes = [vp] * 10 + [i32, i64, i32, i32, i32, vp]
    lib.t2v_layernorm_fwd.argtypes = [vp] * 5 + [i64, i32, f32, vp]
    lib.t2v_layernorm_bwd.argtypes = [vp] * 8 + [i64, i32, vp]
    lib.t2v_latents_to_nhwc8.argtypes = [vp] * 5 + [i32] * 4 + [vp]
    lib.t2v_nhwc8_to_latents.argtypes = [vp, vp] + [i32] * 4 + [vp]
    lib.t2v_mse_loss.argtypes = [vp] * 5 + [i32] * 4 + [vp]
    lib.t2v_velocity_mse_loss.argtypes = [vp] * 8 + [i32] * 4 + [vp]
    lib.t2v_diffusion_loss.argtypes = [vp] * 5 + [ctypes.POINTER(LossParams)] + [vp] * 3 + [i32] * 4 + [vp]
    lib.t2v_vae_sample.argtypes = [vp, vp, vp, i32, i32, i32, f32, vp]
    lib.t2v_geglu_fwd.argtypes = [vp, vp, i64, i32, vp]
    lib.t2v_geglu_bwd.argtypes = [vp, vp, vp, i64, i32, vp]
    lib.t2v_silu_f32_to_bf16.argtypes = [vp, vp, i64, i32, vp]
    lib.t2v_silu_bwd_f32.argtypes = [vp, vp, vp, i64, i32, vp]
    lib.t2v_silu_bf16.argtypes = [vp, vp, i64, vp]
    lib.t2v_silu_bf16_bwd.argtypes = [vp, vp, vp, i64, vp]
    lib.t2v_add_bf16.argtypes = [vp, vp, vp, vp, i64, vp]
    lib.t2v_scale_bf16.argtypes = [vp, vp, i64, f32, vp]
    lib.t2v_dropout_scale_add.argtypes = [vp, vp, vp, i64, f32, f32, ctypes.c_uint64, vp, vp]
    lib.t2v_counter_add.argtypes = [vp, i64, vp]
    lib.t2v_add_f32.argtypes = [vp, vp, vp, i64, vp]
    lib.t2v_cast_f32_bf16.argtypes = [vp, vp, i64, vp]
    lib.t2v_scale_cast_f32_bf16.argtypes = [vp, vp, i64, f32, vp]
    lib.t2v_cast_bf16_f32.argtypes = [vp, vp, i64, vp]
    lib.t2v_sqnorm_chunks.argtypes = [vp, vp, vp, i32, vp, vp]
    lib.t2v_adamw_prepare.argtypes = [vp, vp, i32, vp, vp, f32, vp]
    lib.t2v_adamw_chunks.argtypes = [vp] * 6 + [i64, vp, i32, vp, i32, vp]
    lib.t2v_adamw8bit_chunks.argtypes = [vp] * 4 + [i64, vp, i32] + [vp] * 8 + [i32, vp]
    lib.t2v_adamw_ema_chunks.argtypes = lib.t2v_adamw_chunks.argtypes[:-1] + [vp, vp, f32, vp]
    lib.t2v_adamw8bit_ema_chunks.argtypes = lib.t2v_adamw8bit_chunks.argtypes[:-1] + [vp, vp, f32, vp]
    lib.t2v_ema_swap_chunks.argtypes = [vp, vp, vp, i64, vp, i32, vp]
    lib.t2v_upsample_nearest_fwd.argtypes = [vp, vp] + [i32] * 6 + [vp]
    lib.t2v_upsample_nearest_bwd.argtypes = [vp, vp] + [i32] * 6 + [vp]
    lib.t2v_copy_cols.argtypes = [vp, vp, i64] + [i32] * 5 + [vp]
    lib.t2v_colsum.argtypes = [vp, vp, i32, i64, i32, vp]
    lib.t2v_colsum_f32.argtypes = [vp, vp, i32, i32, vp]
    lib.t2v_softmax_fwd.argtypes = [vp, vp, i64, i32, i32, i32, i32, vp]
    lib.t2v_embed_tokens.argtypes = [vp, vp, vp, vp, i64, i32, i32, i32, vp]
    lib.t2v_embed_tokens_bwd.argtypes = [vp, vp, vp, vp, i64, i32, i32, i32, vp]
    lib.t2v_gelu_bf16.argtypes = [vp, vp, i64, i32, vp]
    lib.t2v_gelu_bwd_bf16.argtypes = [vp, vp, vp, i64, i32, vp]
    lib.t2v_frames_u8_to_nhwc8.argtypes = [vp, vp, i32, i32, i32, i32, i32, vp]
    lib.t2v_frames_u8_to_nhwc8_ragged.argtypes = [vp, vp, i32, i64, vp, i32, i32, vp]
    lib.t2v_softmax_bwd.argtypes = [vp, vp, vp, i64, i32, i32, i32, f32, vp]
    lib.t2v_timestep_embedding.argtypes = [vp, vp, i32, i32, vp]
    lib.t2v_attn_small_fwd.argtypes = [vp] * 4 + [i64, i32, i64, i64, i64, i64, i64, i32, i32, i32, vp]
    lib.t2v_attn_small_bwd.argtypes = [vp] * 7 + [i64, i32, i64, i64, i64, i64, i64, i32, i32, i32, vp]
    lib.t2v_attn_long_fwd.argtypes = [vp] * 5 + [i64, i32, i64, i64, i64, i64, i64, i32, i32, i32, vp]
    lib.t2v_attn_long_bwd.argtypes = [vp] * 9 + [i64, i32, i64, i64, i64, i64, i64, i32, i32, i32, vp]
    lib.t2v_lora_delta_merge.argtypes = [vp, vp, vp, f32] + [i32] * 5 + [vp, vp]
    lib.t2v_lora_delta_grad.argtypes = [vp, vp, vp, f32] + [i32] * 5 + [vp, vp, vp]
    for name in EXPORTS:
        getattr(lib, name)  # every declared symbol must be exported
    return lib


def lib():
    """Returns the loaded library; raises if it has not been built (no CPU fallback exists)."""
    global _lib
    if _lib is None:
        with _lock:
            if _lib is None:
                if not os.path.exists(LIB_PATH):
                    raise RuntimeError(
                        f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                        "(the sm_90a CUDA extension is the only implementation of this path)")
                _lib = _declare(ctypes.CDLL(LIB_PATH))
    return _lib


def check(rc):
    if rc != 0:
        raise RuntimeError(f"t2v_b200 native call failed ({rc}): {lib().t2v_last_error().decode()}")


def launch_count():
    return int(lib().t2v_launch_count())
