"""ctypes binding of libladi_b200.so (the C ABI declared in include/ladi_b200.h).

There is deliberately NO fallback: if the shared library is missing or a call fails, a RuntimeError is raised.
Build it with `python __graft_entry__.py build` (or `make -C ladi_vton_b200/csrc`).
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("LADI_B200_LIB") or os.path.join(_HERE, "libladi_b200.so")  # override: another build of the library


class ConvDesc(C.Structure):
    _fields_ = [
        ("n", C.c_int), ("h_out", C.c_int), ("w_out", C.c_int), ("c_out", C.c_int),
        ("h_in", C.c_int), ("w_in", C.c_int),
        ("ksize", C.c_int), ("stride", C.c_int), ("pad_lo", C.c_int),
        ("n_src", C.c_int), ("src", C.c_void_p * 2), ("src_c", C.c_int * 2), ("src_pitch", C.c_int * 2),
        ("n_sc", C.c_int), ("sc", C.c_void_p * 2), ("sc_c", C.c_int * 2), ("sc_pitch", C.c_int * 2),
        ("weight", C.c_void_p), ("k_total", C.c_int), ("weight_pitch", C.c_int),
        ("bias", C.c_void_p), ("bias_per_row", C.c_int), ("bias_step_stride", C.c_int), ("step_ptr", C.c_void_p),
        ("residual", C.c_void_p), ("residual_pitch", C.c_int),
        ("row_scale", C.c_void_p), ("act", C.c_int),
        ("out", C.c_void_p), ("out_pitch", C.c_int), ("out_fp32", C.c_int), ("force_bn", C.c_int), ("force_direct_epilogue", C.c_int), ("splitk_ws", C.c_void_p), ("splitk_ws_bytes", C.c_int64),
        ("pair_mode", C.c_int),
        ("rowstat_out", C.c_void_p), ("ln_stats", C.c_void_p), ("ln_colsum", C.c_void_p), ("ln_eps", C.c_float),
        ("up2x", C.c_int),
    ]


class ConvPlan(C.Structure):  # ladi_conv_plan: the path ladi_conv2d_bf16 takes for a descriptor (ladi_conv2d_plan)
    _fields_ = [(f, C.c_int) for f in ("bn", "splits", "kb_per_split", "pair", "staged", "stages", "tiles_m", "tiles_n", "total_kb")]

    def items(self):
        """Work items of the persistent grid: (tile, K split) per CTA, or (pair of M tiles, N tile) per CTA pair."""
        return (self.tiles_m + 1) // 2 * self.tiles_n if self.pair else self.tiles_m * self.tiles_n * self.splits


class GroupNormPlan(C.Structure):  # ladi_gn_plan: the grids ladi_groupnorm_stats / ladi_groupnorm_apply launch
    _fields_ = [(f, C.c_int) for f in ("chunks", "gsplit", "block_channels", "lanes_v", "k", "px_per_chunk", "px_per_block", "apply_blocks",
                                        "dv", "dp", "slices")]


class LayerNormPlan(C.Structure):  # ladi_ln_plan (ladi_layernorm_plan)
    _fields_ = [(f, C.c_int) for f in ("T", "vpl", "rows_per_block", "blocks")]


class SmallAttnPlan(C.Structure):  # ladi_sa_plan (ladi_attention_small_plan, ladi_cls_attention_plan)
    _fields_ = [(f, C.c_int) for f in ("chunks", "rows_per_block", "smem_bytes", "smem_optin")]


class AttnPlan(C.Structure):  # ladi_attn_plan (ladi_attention_plan): the launch ladi_attention_bf16 / ladi_attention_d512_bf16 run
    _fields_ = [(f, C.c_int) for f in ("head_dim", "grid_x", "grid_y", "grid_z", "q_tile", "kv_tile", "stages", "consumers", "n_q_tiles",
                                        "n_kv_tiles", "n_items", "items_min", "items_max", "idle_consumers_last_q_tile", "smem_bytes")]


class AttnDesc(C.Structure):
    _fields_ = [
        ("batch", C.c_int), ("heads", C.c_int), ("nq", C.c_int), ("nkv", C.c_int),
        ("q", C.c_void_p), ("q_pitch", C.c_int), ("q_batch_stride", C.c_int64),
        ("k", C.c_void_p), ("k_pitch", C.c_int), ("k_batch_stride", C.c_int64),
        ("v", C.c_void_p), ("v_pitch", C.c_int), ("v_batch_stride", C.c_int64),
        ("out", C.c_void_p), ("out_pitch", C.c_int), ("out_batch_stride", C.c_int64),
        ("scale", C.c_float), ("variant", C.c_int), ("trace", C.c_void_p), ("head_dim", C.c_int),
    ]


class Weight(C.Structure):  # ladi_weight
    _fields_ = [("name", C.c_char_p), ("ptr", C.c_void_p), ("rows", C.c_int), ("cols", C.c_int)]


class EngineConfig(C.Structure):  # ladi_engine_config, field for field
    _fields_ = [
        ("unet_channels", C.c_int * 4), ("unet_heads", C.c_int * 4), ("unet_down_attn", C.c_int * 4), ("unet_up_attn", C.c_int * 4),
        ("unet_layers_per_block", C.c_int), ("unet_in_channels", C.c_int), ("unet_out_channels", C.c_int), ("unet_norm_eps", C.c_float),
        ("norm_groups", C.c_int), ("fuse_upsample", C.c_int),
        ("vae_channels", C.c_int * 4), ("vae_layers_per_block", C.c_int), ("vae_latent_channels", C.c_int), ("vae_in_channels", C.c_int),
        ("vae_out_channels", C.c_int),
        ("emasc_scales", C.c_int), ("emasc_in", C.c_int * 8), ("emasc_out", C.c_int * 8), ("emasc_stride", C.c_int * 8),
        ("adapter_dim", C.c_int), ("adapter_heads", C.c_int), ("adapter_mlp", C.c_int), ("adapter_hidden", C.c_int), ("adapter_out", C.c_int),
        ("plan_only", C.c_int),
    ]


_P, _I, _F, _L = C.c_void_p, C.c_int, C.c_float, C.c_int64
_PP = C.POINTER(C.c_void_p)
SIGNATURES = {
    "ladi_abi_version": ([], C.c_int),
    "ladi_last_error": ([], C.c_char_p),
    "ladi_launch_count": ([], C.c_longlong),
    "ladi_conv2d_bf16": ([C.POINTER(ConvDesc), _P], _I),
    "ladi_conv2d_plan": ([C.POINTER(ConvDesc), _I, C.POINTER(ConvPlan)], _I),
    "ladi_attention_bf16": ([C.POINTER(AttnDesc), _P], _I),
    "ladi_attention_d512_bf16": ([C.POINTER(AttnDesc), _P], _I),
    "ladi_attention_plan": ([C.POINTER(AttnDesc), _I, _I, C.POINTER(AttnPlan)], _I),
    "ladi_groupnorm_chunks": ([_I], _I),
    "ladi_groupnorm_stats": ([_P, _I, _I, _P, _I, _I, _I, _I, _I, _P, _P], _I),
    "ladi_groupnorm_apply": ([_P, _I, _I, _P, _I, _I, _I, _I, _I, _P, _P, _P, _F, _I, _P, _I, _P, _I, _P], _I),
    "ladi_groupnorm_plan": ([_P, _I, _I, _P, _I, _I, _I, _I, _I, _P, _P, _P, _F, _I, _P, _I, _P, _I, _I, C.POINTER(GroupNormPlan)], _I),
    "ladi_layernorm": ([_P, _I, _I, _I, _P, _P, _F, _P, _I, _P], _I),
    "ladi_layernorm_plan": ([_P, _I, _I, _I, _P, _P, _F, _P, _I, _I, C.POINTER(LayerNormPlan)], _I),
    "ladi_softmax_rows": ([_P, _I, _I, _I, _F, _P, _I, _P], _I),
    "ladi_cls_attention": ([_P, _I, _P, _I, _I, _I, _I, _I, _F, _P, _I, _P], _I),
    "ladi_cls_attention_plan": ([_P, _I, _P, _I, _I, _I, _I, _I, _F, _P, _I, _I, C.POINTER(SmallAttnPlan)], _I),
    "ladi_add_bf16": ([_P, _P, _P, _L, _P], _I),
    "ladi_upsample2x_nhwc": ([_P, _I, _I, _I, _I, _P, _P], _I),
    "ladi_nchw_f32_to_nhwc_bf16": ([_P, _I, _I, _I, _I, _I, _F, _P, _P, _I, _I, _P], _I),
    "ladi_nhwc_to_nchw_f32": ([_P, _I, _I, _I, _I, _I, _I, _I, _P, _P], _I),
    "ladi_posterior_sample": ([_P, _I, _P, _I, _I, _I, _I, _F, _P, _P], _I),
    "ladi_inv_mask_rows": ([_P, _I, _I, _I, _I, _P, _P], _I),
    "ladi_bilinear_down8": ([_P, _I, _I, _I, _I, _P, _P], _I),
    "ladi_ddim_cfg_step": ([_P, _I, _P, _P, _I, _I, _I, _I, _I, _F, _P, _P, _I, _P, _P], _I),
    "ladi_check_binarise": ([_P, _L, _P, _L, _P, _P], _I),
    "ladi_image_out": ([_P, _I, _I, _I, _I, _I, _P, _P], _I),
    "ladi_image_out_u8": ([_P, _I, _I, _I, _I, _I, _P, _P], _I),
    "ladi_image_save_u8": ([_P, _I, _I, _I, _I, _P, _P], _I),
    "ladi_pose_heatmaps": ([_P, _I, _I, _I, _F, _P, _P], _I),
    "ladi_attention_small": ([_P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _L, _L, _L, _L, _F, _I, _P], _I),
    "ladi_attention_small_plan": ([_P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _L, _L, _L, _L, _F, _I, _I,
                                   C.POINTER(SmallAttnPlan)], _I),
    "ladi_clip_embed": ([_P, _P, _P, _P, _P, _I, _I, _I, _I, _P], _I),
    "ladi_patchify": ([_P, _P, _I, _I, _I, _I, _I, _I, _P], _I),
    "ladi_vit_assemble": ([_P, _I, _P, _P, _P, _I, _I, _I, _P], _I),
    "ladi_resize_aa": ([_P, _I, _I, _I, _I, _I, _I, _P, _I, _I, _P], _I),
    "ladi_clip_preprocess": ([_P, _I, _I, _I, _I, _I, _I, _P, _P, _I, _P, _P], _I),
    "ladi_space_to_depth2": ([_P, _I, _I, _I, _I, _I, _P, _I, _P], _I),
    "ladi_channel_affine": ([_P, _L, _I, _I, _P, _P, _P], _I),
    "ladi_l2norm_channels": ([_P, _L, _I, _I, _P], _I),
    "ladi_feature_correlation": ([_P, _P, _I, _I, _I, _I, _P, _I, _P], _I),
    "ladi_tps_grid": ([_P, _I, _P, _P, _I, _I, _I, _P, _P, _P], _I),
    "ladi_warp_grid_sample": ([_P, _I, _I, _P, _I, _I, _I, _I, _P, _I, _I, _P], _I),
    "ladi_resize_aa_f32": ([_P, _I, _I, _I, _I, _I, _I, _P, _P], _I),
    "ladi_warp_grid_sample_f32": ([_P, _I, _I, _P, _I, _I, _I, _I, _P, _P], _I),
    "ladi_maxpool2_nhwc": ([_P, _I, _I, _I, _I, _P, _P], _I),
    "ladi_upsample2x_bilinear_ac": ([_P, _I, _I, _I, _I, _P, _P], _I),
    "ladi_nhwc_f32_to_nchw_clamp": ([_P, _I, _I, _I, _I, _I, _F, _F, _P, _P], _I),
    # ---- image-quality metrics (csrc/metrics.cu)
    "ladi_im2col_bf16": ([_P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _P, _P, _P, _I, _P], _I),
    "ladi_pool2d_bf16": ([_P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _P, _I, _I, _P], _I),
    "ladi_lpips_layer": ([_P, _P, _I, _I, _I, _I, _I, _P, _P, _P], _I),
    "ladi_ssim_partials": ([_I, _I], _I),
    "ladi_ssim_f32": ([_P, _P, _I, _I, _I, _I, _P, _P, _P], _I),
    "ladi_resize_tf1_u8": ([_P, _I, _I, _I, _I, _I, _I, _P, _P], _I),
    "ladi_gemm_tf32": ([_P, _I, _I, _I, _P, _I, _I, _P, _I, _P, _I, _I, _P], _I),
    "ladi_im2col_f32": ([_P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _P, _P, _P, _I, _P], _I),
    "ladi_pool2d_f32": ([_P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _P, _I, _I, _P], _I),
    "ladi_lpips_layer_f32": ([_P, _P, _I, _I, _I, _I, _I, _P, _P, _P], _I),
    "ladi_l1_mean_f32": ([_P, _I, _P, _I, _L, _I, _F, _P, _P, _P], _I),
    # ---- module-level ABI (csrc/engine.cu)
    "ladi_engine_create": ([C.POINTER(EngineConfig), C.POINTER(Weight), _I, _PP], _I),
    "ladi_engine_destroy": ([_P], _I),
    "ladi_engine_query": ([_P, _I], _I),
    "ladi_workspace_bytes": ([_P, _I, _I, _I, _I], _L),
    "ladi_engine_trace": ([_P], C.c_char_p),
    "ladi_unet_forward": ([_P, _P, _P, _P, _P, _I, _I, _I, _I, _P, _P, _L, _P], _I),
    "ladi_unet_plan_steps": ([_P, _P, _I, _P, _P, _L, _P], _I),
    "ladi_unet_plan_context": ([_P, _P, _I, _I, _P, _P], _I),
    "ladi_timestep_embedding": ([_P, _I, _I, _I, _P, _P], _I),
    "ladi_vae_encode": ([_P, _P, _I, _I, _I, _P, _PP, _P, _L, _P], _I),
    "ladi_vae_decode_emasc": ([_P, _P, _I, _I, _I, _PP, _I, C.POINTER(C.c_int), _P, _P, _L, _P], _I),
    "ladi_emasc_forward": ([_P, _PP, _PP, _I, _I, _I, _PP, _P, _L, _P], _I),
    "ladi_inversion_adapter_forward": ([_P, _P, _I, _I, _P, _P, _L, _P], _I),
    "ladi_denoise_loop": ([_P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _F, _I, _P, _P, _L, _P], _I),
}

ABI_VERSION = 2
_lib = None
RECORD = None  # tests/test_engine_trace.py: a list -> call() appends (name, args) and launches nothing (CPU-side sequencing check)
launches = 0  # kernels launched by this process through the library (bench.py reports differences of it as gpu_launches): every ABI call adds the
# library's own count of the launches it made (an op-level call 1-3, ladi_unet_forward ~400); a captured graph adds its node count per replay (pipeline._run)


def load():
    """Load the extension (once).  Raises RuntimeError if it has not been built -- no fallback."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(f"{LIB_PATH} not found: the CUDA extension is not built (run `python __graft_entry__.py build`). "
                           "ladi_vton_b200 has no CPU or library fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, (argtypes, restype) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the .so does not export a declared symbol
        fn.argtypes, fn.restype = argtypes, restype
    if lib.ladi_abi_version() != ABI_VERSION:
        raise RuntimeError("libladi_b200.so ABI version mismatch")
    _lib = lib
    return lib


def call(name, *args):
    """Invoke an ABI entry point; non-zero return -> RuntimeError(ladi_last_error())."""
    global launches
    if RECORD is not None:
        RECORD.append((name, args))
        return 0
    lib = load()
    before = lib.ladi_launch_count()
    rc = getattr(lib, name)(*args)
    if rc != 0:
        raise RuntimeError(f"{name} failed ({rc}): {lib.ladi_last_error().decode()}")
    launches += lib.ladi_launch_count() - before
    return rc


def conv_plan(desc, sms=0):
    """The plan ladi_conv2d_bf16 runs for `desc` on `sms` SMs (0: this device's); launches nothing.  Invalid -> RuntimeError."""
    plan = ConvPlan()
    lib = load()
    if lib.ladi_conv2d_plan(C.byref(desc), sms, C.byref(plan)) != 0:
        raise RuntimeError(f"ladi_conv2d_plan failed: {lib.ladi_last_error().decode()}")
    return plan
