"""ctypes mirror of include/rfx.h and loader of the in-tree CUDA library (csrc/librfx.so).

There is no CPU fallback: if the library is missing or a call fails, RfxError is raised.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "librfx.so")

# ---- enums -----------------------------------------------------------------------------
RFX_OK = 0
FMT_R32F, FMT_RGBA32F, FMT_RGBA16F, FMT_RGBA8 = 0, 1, 2, 3
FMT_BYTES = {FMT_R32F: 4, FMT_RGBA32F: 16, FMT_RGBA16F: 8, FMT_RGBA8: 4}
SSGI_IMPORTANCE_SAMPLING, SSGI_MISSED_RAYS, SSGI_USE_DIRECT_LIGHT, SSGI_USE_ENVMAP = 1, 2, 4, 8
MODE_SSGI, MODE_SSR = 0, 1
GROUP_ID_BYTES = 128
ERR_INVALID_ARG = 1
ERR_NOT_READY = 5
ERR_UNSUPPORTED = 6
ERR_NCCL = 7
INPUT_DIFFUSE_SPECULAR, INPUT_DIFFUSE, INPUT_SPECULAR = 0, 1, 2
DENOISE_FULL, DENOISE_FULL_TEMPORAL, DENOISE_TEMPORAL = 0, 1, 2  # option denoiseMode (src/denoise/Denoiser.js:7)
DENOISE_MODES = {"full": 0, "full_temporal": 1, "temporal": 2}
# rfx_ssgi_chain_set_debug_view (include/rfx.h): chain output n is DEBUG_VIEW_OUTPUT + n, GBufferDebugPass mode m DEBUG_VIEW_GBUFFER_CHANNEL + m
DEBUG_VIEW_NONE, DEBUG_VIEW_OUTPUT, DEBUG_VIEW_DEPTH, DEBUG_VIEW_VELOCITY, DEBUG_VIEW_GBUFFER, DEBUG_VIEW_GBUFFER_CHANNEL = -1, 0, 8, 9, 10, 16
GBUFFER_DEBUG_MODES = ["diffuse", "alpha", "normal", "roughness", "metalness", "emissive"]  # SSGIEffect.js:237

F16 = C.c_float * 16
F3 = C.c_float * 3
F2 = C.c_float * 2
I2 = C.c_int32 * 2


class RfxError(RuntimeError):
    pass


class Plane(C.Structure):
    _fields_ = [("ptr", C.c_void_p), ("width", C.c_uint32), ("height", C.c_uint32), ("pitch", C.c_uint64),
                ("format", C.c_int32), ("_reserved", C.c_int32)]


class CameraS(C.Structure):
    _fields_ = [("projection", F16), ("projection_inverse", F16), ("camera_matrix_world", F16), ("view_matrix", F16),
                ("near_plane", C.c_float), ("far_plane", C.c_float), ("perspective", C.c_int32), ("_pad", C.c_int32)]


class SsgiParams(C.Structure):
    _fields_ = [("cam", CameraS), ("ray_distance", C.c_float), ("thickness", C.c_float), ("env_blur", C.c_float),
                ("max_env_map_mip_level", C.c_float), ("steps", C.c_int32), ("refine_steps", C.c_int32), ("mode", C.c_int32),
                ("flags", C.c_uint32), ("blue_noise_index", C.c_int32), ("_pad", C.c_int32)]


class TemporalParams(C.Structure):
    _fields_ = [("cam", CameraS), ("prev_view_matrix", F16), ("prev_camera_matrix_world", F16), ("prev_projection", F16),
                ("prev_projection_inverse", F16), ("camera_pos", F3), ("max_blend", C.c_float), ("prev_camera_pos", F3),
                ("neighborhood_clamp_intensity", C.c_float), ("keep_data", C.c_float), ("confidence_power", C.c_float),
                ("full_accumulate", C.c_int32), ("texture_count", C.c_int32), ("input_type", C.c_int32), ("log_transform", C.c_int32),
                ("reproject_specular", I2), ("history_linear", C.c_int32), ("_pad", C.c_int32)]


class PoissonParams(C.Structure):
    _fields_ = [("radius", C.c_float), ("phi", C.c_float), ("luma_phi", C.c_float), ("depth_phi", C.c_float), ("normal_phi", C.c_float),
                ("roughness_phi", C.c_float), ("specular_phi", C.c_float), ("texture_count", C.c_int32), ("is_texture_specular", I2),
                ("gbuffer_texture", C.c_int32), ("input_linear", C.c_int32), ("blue_noise_index", C.c_int32), ("_pad", C.c_int32)]


class ComposeParams(C.Structure):
    _fields_ = [("cam", CameraS), ("input_type", C.c_int32), ("_pad", C.c_int32)]


class SsgiComposeParams(C.Structure):
    _fields_ = [("use_fog", C.c_int32), ("fog_exp2", C.c_int32), ("fog_color", F3), ("fog_near", C.c_float), ("fog_far", C.c_float),
                ("fog_density", C.c_float), ("camera_near", C.c_float), ("camera_far", C.c_float), ("perspective", C.c_int32), ("is_debug", C.c_int32)]


class TraaTailOptions(C.Structure):
    _fields_ = [("compose", SsgiComposeParams), ("max_blend", C.c_float), ("neighborhood_clamp_intensity", C.c_float), ("confidence_power", C.c_float),
                ("log_transform", C.c_int32), ("full_accumulate", C.c_int32), ("_pad", C.c_int32)]


def make_traa_tail_options(compose: "SsgiComposeParams | None" = None, full_accumulate: bool = False) -> TraaTailOptions:
    """The chain's TRAA tail with the values TRAAEffect forces (src/traa/TRAAEffect.js:21-31: maxBlend 0.9, neighborhoodClampIntensity 1,
    confidencePower 4, logTransform true); `compose`: the K5 fog / isDebug uniforms (None: no fog, no debug)."""
    o = TraaTailOptions()
    if compose is not None:
        o.compose = compose
    o.max_blend, o.neighborhood_clamp_intensity, o.confidence_power, o.log_transform = 0.9, 1.0, 4.0, 1
    o.full_accumulate = int(bool(full_accumulate))
    return o


class HbaoParams(C.Structure):
    _fields_ = [("projection_view", F16), ("projection_inverse", F16), ("camera_matrix_world", F16), ("ao_distance", C.c_float),
                ("distance_power", C.c_float), ("bias", C.c_float), ("thickness", C.c_float), ("spp", C.c_int32), ("blue_noise_index", C.c_int32),
                ("view_matrix", F16), ("resolution", F2)]


class HbaoHorizonParams(C.Structure):
    _fields_ = [("projection", F16), ("projection_inverse", F16), ("camera_matrix_world", F16), ("view_matrix", F16), ("resolution", F2),
                ("distance", C.c_float), ("angle_bias", C.c_float), ("intensity", C.c_float), ("max_radius_pixels", C.c_float),
                ("directions", C.c_int32), ("steps", C.c_int32), ("blue_noise_index", C.c_int32), ("_pad", C.c_int32 * 3)]


class AoComposeParams(C.Structure):
    _fields_ = [("power", C.c_float), ("color", F3)]


class MotionBlurParams(C.Structure):
    _fields_ = [("intensity", C.c_float), ("jitter", C.c_float), ("delta_time", C.c_float), ("resolution", F2), ("frame", C.c_int32),
                ("samples", C.c_int32), ("_pad", C.c_int32)]


class IngestParams(C.Structure):
    _fields_ = [("motion_scale", F2), ("normalize_normals", C.c_int32), ("_pad", C.c_int32)]


FX_SHARPNESS, FX_LENS_DISTORTION, FX_GRADUAL_BACKGROUND, FX_SPARKLE = 1, 2, 3, 4


class EffectsParams(C.Structure):
    _fields_ = [("cam", CameraS), ("n_effects", C.c_int32), ("effects", C.c_int32 * 4), ("sharpness", C.c_float), ("alphax", C.c_float), ("alphay", C.c_float),
                ("aberration", C.c_float), ("background_color", F3), ("max_distance", C.c_float), ("spread", C.c_float), ("intensity", C.c_float),
                ("sparkle_perspective", C.c_int32), ("_pad", C.c_int32)]


class TaaParams(C.Structure):
    _fields_ = [("camera_not_moved_frames", C.c_float), ("srgb_output", C.c_int32)]


def make_effects_params(cam_u: dict, effects, *, sharpness=1.0, alphax=-0.05, alphay=-0.05, aberration=1.0, background_color=(0.0, 0.0, 0.0), max_distance=5.0,
                        spread=1.0, intensity=1.0, sparkle_perspective=False, perspective=True) -> "EffectsParams":
    """defaults: SharpnessEffect.js:32-34, LensDistortionEffect.js:49, GradualBackgroundEffect.js:49, SparkleEffect.js:110-111"""
    p = EffectsParams()
    p.cam = make_camera(cam_u, perspective)
    p.n_effects = len(effects)
    for i, e in enumerate(effects):
        p.effects[i] = int(e)
    p.sharpness, p.alphax, p.alphay, p.aberration = sharpness, alphax, alphay, aberration
    p.background_color[:] = [float(c) for c in background_color]
    p.max_distance, p.spread, p.intensity, p.sparkle_perspective = max_distance, spread, intensity, int(bool(sparkle_perspective))
    return p


class EnvDesc(C.Structure):
    _fields_ = [("map_rgba16f", C.c_void_p), ("width", C.c_uint32), ("height", C.c_uint32), ("marginal", C.c_void_p),
                ("conditional", C.c_void_p), ("total_sum_whole", C.c_float), ("total_sum_decimal", C.c_float)]


class ChainOptions(C.Structure):
    _fields_ = [("width", C.c_uint32), ("height", C.c_uint32), ("denoise_iterations", C.c_int32), ("steps", C.c_int32),
                ("refine_steps", C.c_int32), ("distance", C.c_float), ("thickness", C.c_float), ("env_blur", C.c_float),
                ("radius", C.c_float), ("phi", C.c_float), ("luma_phi", C.c_float), ("depth_phi", C.c_float), ("normal_phi", C.c_float),
                ("roughness_phi", C.c_float), ("specular_phi", C.c_float), ("ssgi_flags", C.c_uint32), ("mode", C.c_int32),
                ("blue_noise_start", C.c_int32), ("denoise_mode", C.c_int32), ("resolution_scale", C.c_float), ("_pad", C.c_int32)]


class SsgiFrame(C.Structure):
    _fields_ = [("cam", CameraS), ("depth", C.POINTER(Plane)), ("gbuffer", C.POINTER(Plane)), ("velocity", C.POINTER(Plane)),
                ("direct_light", C.POINTER(Plane)), ("camera_pos", F3), ("camera_moved", C.c_int32)]


class SsgiHostFrame(C.Structure):
    _fields_ = [("cam", CameraS), ("depth", C.c_void_p), ("gbuffer", C.c_void_p), ("velocity", C.c_void_p), ("direct_light", C.c_void_p),
                ("camera_pos", F3), ("camera_moved", C.c_int32), ("out_composed", C.c_void_p), ("out_color", C.c_void_p)]


AO_HBAO, AO_HORIZON = 0, 1  # rfx_ao_chain_options.algorithm: K6 (HBAOEffect) or K6h (HorizonAOEffect)


class AoChainOptions(C.Structure):
    _fields_ = [("width", C.c_uint32), ("height", C.c_uint32), ("algorithm", C.c_int32), ("resolution_scale", C.c_float),
                ("use_normal_plane", C.c_int32), ("spp", C.c_int32), ("distance", C.c_float), ("distance_power", C.c_float), ("bias", C.c_float),
                ("thickness", C.c_float), ("directions", C.c_int32), ("steps", C.c_int32), ("angle_bias", C.c_float), ("intensity", C.c_float),
                ("max_radius_pixels", C.c_float), ("iterations", C.c_int32), ("radius", C.c_float), ("phi", C.c_float), ("luma_phi", C.c_float),
                ("depth_phi", C.c_float), ("normal_phi", C.c_float), ("power", C.c_float), ("color", F3), ("blue_noise_start", C.c_int32),
                ("denoise_blue_noise_start", C.c_int32), ("_pad", C.c_int32)]


class AoFrame(C.Structure):
    _fields_ = [("projection", F16), ("projection_inverse", F16), ("camera_matrix_world", F16), ("view_matrix", F16),
                ("depth", C.POINTER(Plane)), ("velocity", C.POINTER(Plane)), ("normal", C.POINTER(Plane)), ("input", C.POINTER(Plane)),
                ("output", C.POINTER(Plane))]


class AoTraaFrame(C.Structure):
    """rfx_ao_traa_frame: the TRAA tail's un-jittered camera, its position and didCameraMove"""
    _fields_ = [("cam", CameraS), ("camera_pos", F3), ("camera_moved", C.c_int32)]


class AoHostFrame(C.Structure):
    """rfx_ao_host_frame: the camera matrices, host pointers of the input planes and of the two downloads, and the TRAA camera"""
    _fields_ = [("projection", F16), ("projection_inverse", F16), ("camera_matrix_world", F16), ("view_matrix", F16),
                ("depth", C.c_void_p), ("velocity", C.c_void_p), ("normal", C.c_void_p), ("input", C.c_void_p),
                ("out_color", C.c_void_p), ("out_ao", C.c_void_p), ("traa", C.POINTER(AoTraaFrame))]


def make_camera(u: dict, perspective: "bool | None" = None) -> CameraS:
    """u: dict from synth.Camera.uniforms() (float32 column-major arrays); perspective: camera.isPerspectiveCamera (default: u["perspective"], else True)."""
    if perspective is None:
        perspective = bool(u.get("perspective", True))
    c = CameraS()
    for k in ("projection", "projection_inverse", "camera_matrix_world", "view_matrix"):
        getattr(c, k)[:] = [float(x) for x in np.asarray(u[k], np.float32)]
    c.near_plane = float(u["near"])
    c.far_plane = float(u["far"])
    c.perspective = 1 if perspective else 0
    return c


def set_f16(dst, arr):
    dst[:] = [float(x) for x in np.asarray(arr, np.float32).reshape(-1)]


# ---- library ---------------------------------------------------------------------------
_lib = None

_P = C.POINTER


def _sig(lib):
    vp = C.c_void_p
    PP = _P(Plane)
    lib.rfx_ctx_create.argtypes = [C.c_int, _P(vp)]
    lib.rfx_ctx_destroy.argtypes = [vp]
    lib.rfx_ctx_destroy.restype = None
    lib.rfx_last_error.argtypes = [vp]
    lib.rfx_last_error.restype = C.c_char_p
    lib.rfx_version.restype = C.c_int
    lib.rfx_ctx_stream.argtypes = [vp]
    lib.rfx_ctx_stream.restype = vp
    lib.rfx_ctx_sync.argtypes = [vp]
    lib.rfx_launch_count.argtypes = [vp]
    lib.rfx_launch_count.restype = C.c_uint64
    lib.rfx_ctx_set_fast_math.argtypes = [vp, C.c_int32]
    lib.rfx_blue_noise_set.argtypes = [vp, vp, C.c_uint32, C.c_uint32]
    lib.rfx_env_set.argtypes = [vp, _P(EnvDesc)]
    lib.rfx_env_clear.argtypes = [vp]
    lib.rfx_env_build.argtypes = [vp, vp, C.c_uint32, C.c_uint32, C.c_int32]
    lib.rfx_env_tables_download.argtypes = [vp, vp, vp, _P(C.c_double)]
    lib.rfx_plane_alloc.argtypes = [vp, C.c_int32, C.c_uint32, C.c_uint32, PP]
    lib.rfx_plane_free.argtypes = [vp, PP]
    lib.rfx_plane_clear.argtypes = [vp, vp, PP]
    lib.rfx_plane_upload.argtypes = [vp, vp, PP, vp, C.c_uint64]
    lib.rfx_plane_download.argtypes = [vp, vp, PP, vp, C.c_uint64]
    lib.rfx_host_alloc.argtypes = [vp, C.c_uint64, _P(vp)]
    lib.rfx_host_free.argtypes = [vp, vp]
    lib.rfx_format_bytes.argtypes = [C.c_int32]
    lib.rfx_format_bytes.restype = C.c_uint32
    u32 = C.c_uint32
    lib.rfx_ssgi_trace_launch.argtypes = [vp, vp, _P(SsgiParams), PP, PP, PP, PP, PP, PP, u32, u32]
    lib.rfx_temporal_reproject_launch.argtypes = [vp, vp, _P(TemporalParams), PP, PP, PP, PP, PP, PP, u32, u32]
    lib.rfx_poisson_denoise_launch.argtypes = [vp, vp, _P(PoissonParams), PP, PP, PP, PP, PP, PP, u32, u32]
    lib.rfx_gi_compose_launch.argtypes = [vp, vp, _P(ComposeParams), PP, PP, PP, PP, PP, PP, u32, u32]
    lib.rfx_ssgi_compose_launch.argtypes = [vp, vp, _P(SsgiComposeParams), PP, PP, PP, PP, u32, u32]
    lib.rfx_hbao_launch.argtypes = [vp, vp, _P(HbaoParams), PP, PP, u32, u32]
    lib.rfx_hbao_launch_ex.argtypes = [vp, vp, _P(HbaoParams), PP, PP, PP, u32, u32]
    lib.rfx_hbao_horizon_launch.argtypes = [vp, vp, _P(HbaoHorizonParams), PP, PP, PP]
    lib.rfx_hbao_horizon_directions.argtypes = [C.c_int32, vp]
    lib.rfx_ao_compose_launch.argtypes = [vp, vp, _P(AoComposeParams), PP, PP, PP, PP, u32, u32]
    lib.rfx_motion_blur_launch.argtypes = [vp, vp, _P(MotionBlurParams), PP, PP, PP, u32, u32]
    lib.rfx_traa_compose_launch.argtypes = [vp, vp, PP, PP, u32, u32]
    lib.rfx_traa_motion_blur_launch.argtypes = [vp, vp, _P(MotionBlurParams), PP, PP, PP, PP, u32, u32]
    lib.rfx_gbuffer_debug_launch.argtypes = [vp, vp, C.c_int32, PP, PP, u32, u32]
    lib.rfx_ssgi_chain_set_debug_view.argtypes = [vp, C.c_int32]
    lib.rfx_effects_launch.argtypes = [vp, vp, _P(EffectsParams), PP, PP, PP, PP, u32, u32]
    lib.rfx_taa_launch.argtypes = [vp, vp, _P(TaaParams), PP, PP, PP, u32, u32]
    lib.rfx_gbuffer_ingest_launch.argtypes = [vp, vp, _P(IngestParams), PP, PP, PP, PP, PP, PP, PP, PP, u32, u32]
    lib.rfx_ssgi_chain_create.argtypes = [vp, _P(ChainOptions), _P(vp)]
    lib.rfx_ssgi_chain_destroy.argtypes = [vp]
    lib.rfx_ssgi_chain_destroy.restype = None
    lib.rfx_ssgi_chain_reset.argtypes = [vp]
    lib.rfx_ssgi_chain_set_options.argtypes = [vp, _P(ChainOptions)]
    lib.rfx_ssgi_chain_render.argtypes = [vp, vp, _P(SsgiFrame)]
    lib.rfx_ssgi_chain_output.argtypes = [vp, C.c_int32, PP]
    lib.rfx_ssgi_chain_enable_traa.argtypes = [vp, _P(TraaTailOptions)]
    lib.rfx_ssgi_chain_set_motion_blur.argtypes = [vp, _P(MotionBlurParams)]
    lib.rfx_ssgi_chain_set_effects.argtypes = [vp, _P(EffectsParams)]
    lib.rfx_ssgi_chain_set_compose.argtypes = [vp, _P(SsgiComposeParams)]
    lib.rfx_ssgi_chain_render_sharded_finish.argtypes = [vp, vp]
    lib.rfx_ao_chain_render_sharded_finish.argtypes = [vp, vp]
    lib.rfx_ssgi_chain_render_host.argtypes = [vp, _P(SsgiHostFrame)]
    lib.rfx_ssgi_chain_submit_host.argtypes = [vp, _P(SsgiHostFrame)]
    lib.rfx_ssgi_chain_wait_host.argtypes = [vp, C.c_int32]
    lib.rfx_ssgi_chain_set_profiling.argtypes = [vp, C.c_int32]
    lib.rfx_ssgi_chain_get_profile.argtypes = [vp, _P(C.c_double), _P(C.c_uint64)]
    lib.rfx_plane_download_rows.argtypes = [vp, vp, PP, vp, u32, u32]
    # row-sharded multi-GPU groups
    U32P = _P(C.c_uint32)
    lib.rfx_group_get_unique_id.argtypes = [vp]
    lib.rfx_group_create.argtypes = [vp, C.c_char_p, C.c_int32, C.c_int32, _P(vp)]
    lib.rfx_group_create_inprocess.argtypes = [vp, C.c_int32, C.c_int32, _P(vp)]
    lib.rfx_group_attach_chains_inprocess.argtypes = [_P(vp), _P(vp), C.c_int32]
    lib.rfx_group_destroy.argtypes = [vp]
    lib.rfx_group_destroy.restype = None
    lib.rfx_group_rank.argtypes = [vp]
    lib.rfx_group_world.argtypes = [vp]
    lib.rfx_group_uses_peer_reads.argtypes = [vp]
    lib.rfx_group_attach_chain.argtypes = [vp, vp]
    lib.rfx_group_get_bounds.argtypes = [vp, U32P]
    lib.rfx_group_set_bounds.argtypes = [vp, U32P]
    lib.rfx_group_set_rebalance.argtypes = [vp, C.c_int32, C.c_int32]
    lib.rfx_group_last_costs.argtypes = [vp, _P(C.c_float)]
    lib.rfx_group_begin_frame.argtypes = [vp, U32P]
    lib.rfx_group_get_last_bounds.argtypes = [vp, U32P]
    lib.rfx_group_allgather_rows.argtypes = [vp, vp, PP, U32P]
    lib.rfx_ssgi_chain_render_sharded.argtypes = [vp, vp, _P(SsgiFrame)]
    lib.rfx_shard_ranges.argtypes = [u32, u32, u32, u32, C.c_int32, C.c_float, C.c_int32, U32P, u32]
    lib.rfx_shard_rebalance.argtypes = [U32P, U32P, _P(C.c_float), C.c_int32, U32P]
    # AO chain
    lib.rfx_ao_chain_create.argtypes = [vp, _P(AoChainOptions), _P(vp)]
    lib.rfx_ao_chain_destroy.argtypes = [vp]
    lib.rfx_ao_chain_destroy.restype = None
    lib.rfx_ao_chain_set_options.argtypes = [vp, _P(AoChainOptions)]
    lib.rfx_ao_chain_reset.argtypes = [vp]
    lib.rfx_ao_chain_render.argtypes = [vp, vp, _P(AoFrame)]
    lib.rfx_ao_chain_output.argtypes = [vp, C.c_int32, PP]
    lib.rfx_ao_chain_enable_traa.argtypes = [vp, _P(TraaTailOptions)]
    lib.rfx_ao_chain_set_motion_blur.argtypes = [vp, _P(MotionBlurParams)]
    lib.rfx_ao_chain_set_effects.argtypes = [vp, _P(EffectsParams)]
    lib.rfx_fx_stage_rows.argtypes = [u32, u32, _P(EffectsParams), u32, u32, _P(u32)]
    lib.rfx_ao_chain_render_traa.argtypes = [vp, vp, _P(AoFrame), _P(AoTraaFrame)]
    lib.rfx_ao_chain_render_sharded_traa.argtypes = [vp, vp, _P(AoFrame), _P(AoTraaFrame)]
    lib.rfx_group_attach_ao_chain.argtypes = [vp, vp]
    lib.rfx_group_attach_ao_chains_inprocess.argtypes = [_P(vp), _P(vp), C.c_int32]
    lib.rfx_ao_chain_render_sharded.argtypes = [vp, vp, _P(AoFrame)]
    lib.rfx_ao_shard_ranges.argtypes = [u32, u32, u32, u32, C.c_int32, C.c_float, U32P, u32]
    lib.rfx_ao_chain_render_host.argtypes = [vp, _P(AoHostFrame)]
    lib.rfx_ao_chain_submit_host.argtypes = [vp, _P(AoHostFrame)]
    lib.rfx_ao_chain_wait_host.argtypes = [vp, C.c_int32]


EXPORTS = [
    "rfx_ctx_create", "rfx_ctx_destroy", "rfx_last_error", "rfx_version", "rfx_ctx_stream", "rfx_ctx_sync", "rfx_launch_count",
    "rfx_ctx_set_fast_math",
    "rfx_blue_noise_set", "rfx_env_set", "rfx_env_clear", "rfx_env_build", "rfx_env_tables_download", "rfx_plane_alloc", "rfx_plane_free", "rfx_plane_clear", "rfx_plane_upload",
    "rfx_plane_download", "rfx_host_alloc", "rfx_host_free", "rfx_format_bytes", "rfx_ssgi_trace_launch",
    "rfx_temporal_reproject_launch", "rfx_poisson_denoise_launch", "rfx_gi_compose_launch", "rfx_ssgi_compose_launch", "rfx_hbao_launch", "rfx_hbao_launch_ex",
    "rfx_hbao_horizon_launch", "rfx_hbao_horizon_directions", "rfx_ao_compose_launch", "rfx_motion_blur_launch", "rfx_traa_compose_launch", "rfx_gbuffer_ingest_launch", "rfx_effects_launch", "rfx_taa_launch", "rfx_ssgi_chain_create", "rfx_ssgi_chain_destroy",
    "rfx_ssgi_chain_reset", "rfx_ssgi_chain_render", "rfx_ssgi_chain_output", "rfx_ssgi_chain_enable_traa", "rfx_ssgi_chain_render_host",
    "rfx_ssgi_chain_submit_host", "rfx_ssgi_chain_wait_host",
    "rfx_ssgi_chain_set_profiling", "rfx_ssgi_chain_get_profile", "rfx_ssgi_chain_set_options",
    "rfx_plane_download_rows", "rfx_group_get_unique_id", "rfx_group_create", "rfx_group_create_inprocess", "rfx_group_attach_chains_inprocess", "rfx_group_destroy", "rfx_group_rank", "rfx_group_world", "rfx_group_uses_peer_reads",
    "rfx_group_attach_chain", "rfx_group_get_bounds", "rfx_group_set_bounds", "rfx_group_set_rebalance", "rfx_group_last_costs",
    "rfx_group_begin_frame", "rfx_group_get_last_bounds", "rfx_group_allgather_rows", "rfx_ssgi_chain_render_sharded", "rfx_shard_ranges",
    "rfx_shard_rebalance", "rfx_gbuffer_debug_launch", "rfx_ssgi_chain_set_debug_view",
    "rfx_ao_chain_create", "rfx_ao_chain_destroy", "rfx_ao_chain_set_options", "rfx_ao_chain_reset", "rfx_ao_chain_render", "rfx_ao_chain_output",
    "rfx_group_attach_ao_chain", "rfx_group_attach_ao_chains_inprocess", "rfx_ao_chain_render_sharded", "rfx_ao_shard_ranges",
    "rfx_ao_chain_enable_traa", "rfx_ao_chain_render_traa", "rfx_ao_chain_render_sharded_traa",
    "rfx_traa_motion_blur_launch", "rfx_ssgi_chain_set_motion_blur", "rfx_ao_chain_set_motion_blur",
    "rfx_ssgi_chain_render_sharded_finish", "rfx_ao_chain_render_sharded_finish",
    "rfx_ssgi_chain_set_effects", "rfx_ao_chain_set_effects", "rfx_fx_stage_rows",
    "rfx_ao_chain_render_host", "rfx_ao_chain_submit_host", "rfx_ao_chain_wait_host", "rfx_ssgi_chain_set_compose",
]


def lib():
    """Load csrc/librfx.so (built by __graft_entry__.build()).  Raises RfxError when absent."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RfxError(f"{LIB_PATH} not found — run `python -c 'import __graft_entry__ as g; g.build()'` (there is no CPU fallback)")
        try:
            l = C.CDLL(LIB_PATH, mode=C.RTLD_GLOBAL)
        except OSError as e:
            raise RfxError(f"cannot load {LIB_PATH}: {e}") from e
        _sig(l)
        _lib = l
    return _lib
