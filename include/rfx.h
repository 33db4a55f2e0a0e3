/*
 * rfx.h — C ABI of the H100-native screen-space post-processing engine.
 *
 * This is the drop-in boundary for the per-pixel hot path of 0beqz/realism-effects
 * (SSGI trace -> temporal reprojection -> Poisson denoise -> GI compose, plus HBAO,
 * TRAA and motion blur).  Every entry point is `extern "C"`, takes plain pointers /
 * sizes / POD structs, returns an rfx_status, never throws and never aborts.
 *
 * The reference has no native interface (it is WebGL2 fragment shaders driven by JS);
 * what an FFI for this path would bind is one call per fullscreen draw.  Each launch
 * function below names the reference draw it replaces (paths relative to the
 * reference checkout, `src/...`).
 *
 * Conventions
 *  - Matrices are 16 fp32, column-major (three.js Matrix4.elements layout).
 *  - Planes are pitched 2-D arrays in device memory, row 0 = GL texel row 0 (v = 0).
 *    Pixel centre uv = ((x+0.5)/W, (y+0.5)/H)            (src/utils/shader/basic.vert:3-4)
 *  - The context is NOT thread-safe.  Launches are enqueued on the given stream (or the
 *    context's own stream when `stream == NULL`) and return immediately.
 *  - Uniform values the reference derives from non-deterministic sources (blue-noise
 *    index, delta time, window size) are explicit parameters (SURVEY.md §8b).
 */
#ifndef RFX_H
#define RFX_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RFX_VERSION 3

typedef enum rfx_status {
  RFX_OK = 0,
  RFX_ERR_INVALID_ARG = 1,   /* NULL pointer, bad enum, bad count                */
  RFX_ERR_BAD_FORMAT = 2,    /* plane has the wrong rfx_format for this binding  */
  RFX_ERR_SIZE_MISMATCH = 3, /* plane sizes inconsistent with each other         */
  RFX_ERR_CUDA = 4,          /* a CUDA runtime call failed (see rfx_last_error)  */
  RFX_ERR_NOT_READY = 5,     /* e.g. env map / blue noise not set                */
  RFX_ERR_UNSUPPORTED = 6,   /* valid in the reference, not implemented here     */
  RFX_ERR_NCCL = 7
} rfx_status;

/* Texel formats at the boundary = the reference's GL formats (SURVEY.md §8 table). */
typedef enum rfx_format {
  RFX_FMT_R32F = 0,    /* depth (DEPTH32F), marginal / conditional CDF tables      */
  RFX_FMT_RGBA32F = 1, /* gBuffer, velocity, ssgi trace output, TR output, composed */
  RFX_FMT_RGBA16F = 2, /* Poisson targets, AO target, composer buffers, env map     */
  RFX_FMT_RGBA8 = 3    /* blue noise                                                */
} rfx_format;

typedef struct rfx_plane {
  void* ptr;          /* device pointer (cudaMalloc / cudaMallocPitch), 16-B aligned */
  uint32_t width;     /* texels */
  uint32_t height;    /* texels */
  uint64_t pitch;     /* bytes between rows, multiple of 16                          */
  int32_t format;     /* rfx_format                                                  */
  int32_t _reserved;
} rfx_plane;

typedef struct rfx_ctx rfx_ctx;

/* Camera block shared by the passes.  Mirrors the uniforms
 *   projectionMatrix / projectionMatrixInverse / cameraMatrixWorld / viewMatrix /
 *   cameraNear / cameraFar and the PERSPECTIVE_CAMERA define
 * (src/ssgi/pass/SSGIPass.js:33-38,82-87; src/temporal-reproject/TemporalReprojectPass.js:89-93;
 *  src/denoise/pass/DenoiserComposePass.js:88-99). */
typedef struct rfx_camera {
  float projection[16];
  float projection_inverse[16];
  float camera_matrix_world[16];
  float view_matrix[16]; /* camera.matrixWorldInverse */
  float near_plane;
  float far_plane;
  int32_t perspective; /* 1 = PERSPECTIVE_CAMERA defined */
  int32_t _pad;
} rfx_camera;

/* ------------------------------------------------------------------------------------
 * K1  SSGI / SSR trace     replaces the fullscreen draw of src/ssgi/pass/SSGIPass.js:93-94
 *     (shader src/ssgi/shader/ssgi.frag + ssgi_utils.frag; uniforms SSGIMaterial.js:15-42,
 *      defines :44-51, per-frame SSGIPass.js:82-91, options SSGIOptions.js:26-48)
 * ---------------------------------------------------------------------------------- */
enum {
  RFX_SSGI_IMPORTANCE_SAMPLING = 1u << 0, /* #define importanceSampling            */
  RFX_SSGI_MISSED_RAYS = 1u << 1,         /* #define missedRays                    */
  RFX_SSGI_USE_DIRECT_LIGHT = 1u << 2,    /* #define useDirectLight                */
  RFX_SSGI_USE_ENVMAP = 1u << 3           /* #define USE_ENVMAP                    */
};
enum { RFX_MODE_SSGI = 0, RFX_MODE_SSR = 1 };

typedef struct rfx_ssgi_params {
  rfx_camera cam;
  float ray_distance;          /* uniform rayDistance  (option `distance`)          */
  float thickness;             /* uniform thickness                                  */
  float env_blur;              /* uniform envBlur                                    */
  float max_env_map_mip_level; /* uniform maxEnvMapMipLevel (Utils.js:30-34)         */
  int32_t steps;               /* #define steps                                      */
  int32_t refine_steps;        /* #define refineSteps                                */
  int32_t mode;                /* RFX_MODE_SSGI / RFX_MODE_SSR                       */
  uint32_t flags;              /* RFX_SSGI_*                                         */
  int32_t blue_noise_index;    /* uniform blueNoiseIndex (BlueNoiseUtils.js:19-28)   */
  int32_t _pad;
} rfx_ssgi_params;

/* ------------------------------------------------------------------------------------
 * K2  temporal reprojection   replaces src/temporal-reproject/TemporalReprojectPass.js:192-193
 *     (shader temporal_reproject.frag + reproject.frag; uniforms
 *      material/TemporalReprojectMaterial.js:45-68; defines TemporalReprojectPass.js:77-117)
 * ---------------------------------------------------------------------------------- */
enum { RFX_INPUT_DIFFUSE_SPECULAR = 0, RFX_INPUT_DIFFUSE = 1, RFX_INPUT_SPECULAR = 2 };

typedef struct rfx_temporal_params {
  rfx_camera cam; /* un-jittered projection (TemporalReprojectPass.js:168-175) */
  float prev_view_matrix[16];
  float prev_camera_matrix_world[16];
  float prev_projection[16];
  float prev_projection_inverse[16];
  float camera_pos[3];
  float max_blend;
  float prev_camera_pos[3]; /* uploaded by the reference, unused by the shader */
  float neighborhood_clamp_intensity;
  float keep_data;        /* 1, or 0 for the frame after reset()                    */
  float confidence_power; /* #define confidencePower                                */
  int32_t full_accumulate; /* uniform fullAccumulate (already AND-ed with !didCameraMove) */
  int32_t texture_count;   /* 1 or 2                                                 */
  int32_t input_type;      /* RFX_INPUT_*                                            */
  int32_t log_transform;   /* #define logTransform                                   */
  int32_t reproject_specular[2];
  int32_t history_linear;  /* 1: history planes are sampled LINEAR (Poisson targets /
                              FramebufferTexture), 0: NEAREST                        */
  int32_t _pad;
} rfx_temporal_params;

/* ------------------------------------------------------------------------------------
 * K3  Poisson denoise pass   replaces ONE iteration of the loop at
 *     src/denoise/pass/PoissonDenoisePass.js:135-149 (shader poisson_denoise.frag;
 *     uniforms PoissonDenoisePass.js:48-69)
 * ---------------------------------------------------------------------------------- */
typedef struct rfx_poisson_params {
  float radius, phi, luma_phi, depth_phi, normal_phi, roughness_phi, specular_phi;
  int32_t texture_count;          /* 1 or 2                                          */
  int32_t is_texture_specular[2]; /* #define isTextureSpecular                       */
  int32_t gbuffer_texture;        /* 1: GBUFFER_TEXTURE (packed gBuffer plane),
                                     0: velocity-layout plane (normal in .b, depth in .a) */
  int32_t input_linear;           /* filter of in0/in1: 0 NEAREST (pass 0 reads the TR
                                     targets), 1 LINEAR (passes >= 1 read dnA/dnB)   */
  int32_t blue_noise_index;
  int32_t _pad;
} rfx_poisson_params;

/* K4  GI compose   replaces src/denoise/pass/DenoiserComposePass.js:129-135 */
typedef struct rfx_compose_params {
  rfx_camera cam;
  int32_t input_type; /* RFX_INPUT_* */
  int32_t _pad;
} rfx_compose_params;

/* K6  HBAO   replaces src/ao/AOPass.js:108-109 with src/hbao/shader/hbao.frag
 *     (uniforms AOPass.js:36-54, defaults src/ao/AOEffect.js:8-21) */
typedef struct rfx_hbao_params {
  float projection_view[16]; /* projectionMatrix * matrixWorldInverse (AOPass.js:93-96) */
  float projection_inverse[16];
  float camera_matrix_world[16];
  float ao_distance, distance_power, bias, thickness;
  int32_t spp;
  int32_t blue_noise_index;
  /* read by rfx_hbao_launch_ex only (rfx_hbao_launch reads the fields above, so callers of the shorter struct keep working): */
  float view_matrix[16];     /* camera.matrixWorldInverse: turns the normal plane's view-space normals to world space
                                (hbao_utils.glsl:70-79); used only with a normal plane                            */
  float resolution[2];       /* uniform resolution = the AO target's UNROUNDED size (width * resolutionScale, ...;
                                AOPass.js:79-83); {0, 0}: the out plane's size                                    */
} rfx_hbao_params;

/* K6h  horizon-march AO   an extension: the reference has no such draw (its hbao.frag takes cosine-hemisphere samples, SURVEY.md D1).
 *      The per-sample horizon form of Bavoil, Sainz and Dimitrov, "Image-Space Horizon-Based Ambient Occlusion" (SIGGRAPH 2008): D
 *      screen-space directions x S steps per pixel; same inputs and output layout as K6. */
typedef struct rfx_hbao_horizon_params {
  float projection[16];          /* camera.projectionMatrix: row 4 gives the clip w of the pixel, [5] the vertical scale          */
  float projection_inverse[16];
  float camera_matrix_world[16];
  float view_matrix[16];         /* camera.matrixWorldInverse; used only with a normal plane                                      */
  float resolution[2];           /* the AO target's UNROUNDED size (as rfx_hbao_params.resolution); {0, 0}: the out plane's size */
  float distance;                /* world-space radius, > 0                                                                      */
  float angle_bias;              /* subtracted from each tap's cosine, [0, 1)                                                    */
  float intensity;               /* >= 0                                                                                          */
  float max_radius_pixels;       /* the projected radius is clamped to this many texels, >= 1                                     */
  int32_t directions;            /* 1..32                                                                                         */
  int32_t steps;                 /* 1..64                                                                                         */
  int32_t blue_noise_index;      /* != 0                                                                                          */
  int32_t _pad[3];
} rfx_hbao_horizon_params;

/* K7  AO compose   src/ao/shader/ao_compose.frag:6-16 */
typedef struct rfx_ao_compose_params {
  float power;
  float color[3];
} rfx_ao_compose_params;

/* K8  motion blur   src/motion-blur/shader/motion_blur.frag:11-44,
 *     host values src/motion-blur/MotionBlurEffect.js:87-102 */
typedef struct rfx_motion_blur_params {
  float intensity, jitter;
  float delta_time;    /* already max(1/1000, deltaTime)                            */
  float resolution[2]; /* uniform resolution (window.innerWidth/innerHeight)        */
  int32_t frame;       /* blue-noise index; 0 selects the tiled lookup              */
  int32_t samples;     /* #define samples                                           */
  int32_t _pad;
} rfx_motion_blur_params;

/* G-buffer ingest (SURVEY.md §8f row 2): a conventional deferred renderer's planes -> the reference's packed layouts.
 *   gBuffer  = packGBuffer(diffuse, worldNormal, roughness, metalness, emissive)   src/gbuffer/shader/gbuffer_packing.glsl:166-178
 *              (what GBufferMaterial.js:94-98 writes); a zero emissive is encoded as 0 (the shader takes a log2(0) path there;
 *              it decodes to 0 on every back-end);
 *   velocity = (motion.xy * motion_scale, packNormal(worldNormal), depth)            src/temporal-reproject/material/
 *              VelocityDepthNormalMaterial.js:76-83,186-188;
 *   a pixel with depth == 1 gets the cleared targets' texel (0,0,0,1) in both planes (GBufferPass.js:42-44, SURVEY §8 plane table). */
typedef struct rfx_ingest_params {
  float motion_scale[2];       /* uv-space motion = motion.xy * scale ((1,1): already uv-space cur - prev; (.5,.5): NDC)  */
  int32_t normalize_normals;   /* 1: worldNormal = normalize(normal.xyz) as the reference's producers do; 0: taken as stored */
  int32_t _pad;
} rfx_ingest_params;

/* Cosmetic effects of the plugin surface (SURVEY.md §8f row 3), merged the way postprocessing's EffectPass merges the effects of one pass:
 * every effect samples the SAME input buffer through `inputTexture`, and the colour flows from one effect's outputColor into the next
 * effect's inputColor.  One launch applies up to 4 effects in the given order — one pass over memory instead of one per effect.
 *   RFX_FX_SHARPNESS           src/sharpness/SharpnessEffect.js:4-30                (3x3 box unsharp mask)
 *   RFX_FX_LENS_DISTORTION     src/lens-distortion/LensDistortionEffect.js:5-46     (radial undistortion + chromatic aberration; replaces the colour)
 *   RFX_FX_GRADUAL_BACKGROUND  src/gradual-background/GradualBackgroundEffect.js:3-47 (needs depth)
 *   RFX_FX_SPARKLE             src/sparkle/SparkleEffect.js:4-100                    (needs the velocity plane) */
#define RFX_FX_SHARPNESS 1
#define RFX_FX_LENS_DISTORTION 2
#define RFX_FX_GRADUAL_BACKGROUND 3
#define RFX_FX_SPARKLE 4
typedef struct rfx_effects_params {
  rfx_camera cam;             /* gradual background / sparkle; cam.perspective = `#if PERSPECTIVE_CAMERA == 1`                            */
  int32_t n_effects;          /* 1..4                                                                                                  */
  int32_t effects[4];         /* RFX_FX_* in application order                                                                         */
  float sharpness;            /* SharpnessEffect option (default 1)                                                                    */
  float alphax, alphay, aberration; /* LensDistortionEffect (defaults -0.05, -0.05, 1)                                                 */
  float background_color[3];  /* GradualBackgroundEffect                                                                               */
  float max_distance;         /* default 5                                                                                             */
  float spread, intensity;    /* SparkleEffect uniforms (default 1, 1)                                                                 */
  int32_t sparkle_perspective; /* SparkleEffect never defines PERSPECTIVE_CAMERA, so the reference takes the orthographic getViewZ branch:
                                  0 = that behaviour, 1 = what a host that defines it gets                                              */
  int32_t _pad;
} rfx_effects_params;

/* TAAPass   src/taa/TAAPass.js:68-94 + src/taa/shader/taa.frag: the still-camera accumulator that renders to the screen.
 * out = cameraNotMovedFrames == 0 ? c : mix(history, c, 1 / (cameraNotMovedFrames + 1)),  c = linearToOutputTexel(input) */
typedef struct rfx_taa_params {
  float camera_not_moved_frames;
  int32_t srgb_output;        /* 1: the renderer's output colour space is sRGB (three's default): linearToOutputTexel = LinearTosRGB  */
} rfx_taa_params;

/* Environment map + importance-sampling tables (struct EquirectHdrInfo, ssgi.frag:27-36;
 * built by src/ssgi/utils/EquirectHdrInfoUniform.js:149-245). */
typedef struct rfx_env_desc {
  const void* map_rgba16f; /* HOST pointer, mip 0, width*height*4 halfs, tightly packed */
  uint32_t width, height;
  const float* marginal;    /* HOST, `height` floats (may be NULL when no importance sampling) */
  const float* conditional; /* HOST, width*height floats                                       */
  float total_sum_whole, total_sum_decimal;
} rfx_env_desc;

/* ---- context ---------------------------------------------------------------------- */
rfx_status rfx_ctx_create(int device, rfx_ctx** out);
void rfx_ctx_destroy(rfx_ctx* ctx);
const char* rfx_last_error(const rfx_ctx* ctx);
int rfx_version(void);
void* rfx_ctx_stream(rfx_ctx* ctx);      /* the context's cudaStream_t             */
rfx_status rfx_ctx_sync(rfx_ctx* ctx);   /* cudaStreamSynchronize(ctx stream)      */
uint64_t rfx_launch_count(const rfx_ctx* ctx); /* kernels launched so far by this ctx */
/* Kernel variants: 1 (default) = transcendentals on the SFU pipe (lg2/ex2.approx, ~2^-22 relative
 * error, well inside the 1e-3 parity budget); 0 = exact-libm variants whose non-transcendental
 * arithmetic is bit-identical to the parity oracle.  Both are CUDA kernels; neither is a CPU path. */
rfx_status rfx_ctx_set_fast_math(rfx_ctx* ctx, int32_t enable);

/* blue noise: 128x128 RGBA8 in GL texel order (flipY already applied)
 * (src/utils/BlueNoiseUtils.js:6-15) */
rfx_status rfx_blue_noise_set(rfx_ctx* ctx, const uint8_t* rgba8_host, uint32_t width, uint32_t height);
/* env map: uploads mip 0, builds the box-filter mip chain on the device
 * (generateMipmaps, src/ssgi/SSGIEffect.js:324-329) and uploads the CDF tables */
rfx_status rfx_env_set(rfx_ctx* ctx, const rfx_env_desc* env);
/* env map with the importance-sampling tables built ON THE DEVICE (replaces the reference's Web Worker:
 * src/ssgi/utils/EquirectHdrInfoUniform.js:323-358 -> gatherData :149-245; same summation order, bit-identical tables).
 * flip_y = texture.flipY of the source (RGBELoader sets it): the reference's in-place "un-flip" is reproduced as written */
rfx_status rfx_env_build(rfx_ctx* ctx, const void* map_rgba16f_host, uint32_t width, uint32_t height, int32_t flip_y);
/* host copies of the current tables: marginal[height], conditional[width*height], totalSum (any pointer may be NULL) */
rfx_status rfx_env_tables_download(rfx_ctx* ctx, float* marginal, float* conditional, double* total_sum);
rfx_status rfx_env_clear(rfx_ctx* ctx);

/* ---- planes ------------------------------------------------------------------------ */
rfx_status rfx_plane_alloc(rfx_ctx* ctx, int32_t format, uint32_t width, uint32_t height, rfx_plane* out);
rfx_status rfx_plane_free(rfx_ctx* ctx, rfx_plane* plane);
rfx_status rfx_plane_clear(rfx_ctx* ctx, void* stream, const rfx_plane* plane);
/* host <-> device, asynchronous on `stream` when the host memory is pinned */
rfx_status rfx_plane_upload(rfx_ctx* ctx, void* stream, const rfx_plane* dst, const void* host, uint64_t host_pitch);
rfx_status rfx_plane_download(rfx_ctx* ctx, void* stream, const rfx_plane* src, void* host, uint64_t host_pitch);
/* rows [row0, row1) of a plane to tightly packed host memory (a row-sharded rank reads back only its own band) */
rfx_status rfx_plane_download_rows(rfx_ctx* ctx, void* stream, const rfx_plane* src, void* host, uint32_t row0, uint32_t row1);
rfx_status rfx_host_alloc(rfx_ctx* ctx, uint64_t bytes, void** out); /* pinned */
rfx_status rfx_host_free(rfx_ctx* ctx, void* p);
uint32_t rfx_format_bytes(int32_t format);

/* ---- pass launches ------------------------------------------------------------------
 * `row0,row1` select the output rows [row0,row1) this call writes (row-block sharding,
 * SURVEY.md §8e); pass 0,0 for the whole plane.  Input planes are always full frames. */

/* K1. velocity / direct_light / accumulated may be NULL (null sampler => (0,0,0,1),
 * SURVEY.md D4).  out: RGBA32F (8 packed halfs, gbuffer_packing.glsl:65-83). */
rfx_status rfx_ssgi_trace_launch(rfx_ctx* ctx, void* stream, const rfx_ssgi_params* p,
                                 const rfx_plane* depth, const rfx_plane* gbuffer,
                                 const rfx_plane* velocity, const rfx_plane* direct_light,
                                 const rfx_plane* accumulated, const rfx_plane* out,
                                 uint32_t row0, uint32_t row1);

/* K2. input: K1 output (RGBA32F packed) for DIFFUSE_SPECULAR, RGBA16F colour for DIFFUSE
 * (TRAA).  history[i]/out[i], i < texture_count.  history RGBA16F, out RGBA32F (SSGI) or
 * RGBA16F (TRAA).  Discarded pixels keep the previous contents of out (SURVEY.md A2). */
rfx_status rfx_temporal_reproject_launch(rfx_ctx* ctx, void* stream, const rfx_temporal_params* p,
                                         const rfx_plane* input, const rfx_plane* velocity,
                                         const rfx_plane* history0, const rfx_plane* history1,
                                         const rfx_plane* out0, const rfx_plane* out1,
                                         uint32_t row0, uint32_t row1);

/* K3. gbuffer_or_normal: packed gBuffer (gbuffer_texture=1) or velocity-layout plane.
 * in: RGBA32F or RGBA16F; out: RGBA16F.  With input_linear set, in0/in1 (one size) may differ in size from out: they are
 * sampled by uv (the AO denoiser's first pass upsamples a reduced-resolution AO target); NEAREST inputs have out's size. */
rfx_status rfx_poisson_denoise_launch(rfx_ctx* ctx, void* stream, const rfx_poisson_params* p,
                                      const rfx_plane* depth, const rfx_plane* gbuffer_or_normal,
                                      const rfx_plane* in0, const rfx_plane* in1,
                                      const rfx_plane* out0, const rfx_plane* out1,
                                      uint32_t row0, uint32_t row1);

/* K4. diffuse_gi / specular_gi: RGBA16F Poisson targets; out: RGBA32F.  input_type selects the bindings of
 * DenoiserComposePass.js:23-33: DIFFUSE_SPECULAR both, DIFFUSE only diffuse_gi, SPECULAR (SSR) only specular_gi plus
 * `scene` = the composer input buffer (RGBA16F, sampled LINEAR; src/denoise/Denoiser.js:100-102); unbound ones are NULL. */
rfx_status rfx_gi_compose_launch(rfx_ctx* ctx, void* stream, const rfx_compose_params* p,
                                 const rfx_plane* depth, const rfx_plane* gbuffer,
                                 const rfx_plane* diffuse_gi, const rfx_plane* specular_gi, const rfx_plane* scene,
                                 const rfx_plane* out, uint32_t row0, uint32_t row1);

/* K5. src/ssgi/shader/ssgi_compose.frag:20-44.  gi RGBA32F, scene RGBA16F, out RGBA16F.  `p` may be NULL (no fog, no debug).
 * Fog = three.js <fog_fragment> as patched by src/ssgi/SSGIEffect.js:34-43 on vFogDepth = -getViewZ(depth) * 0.4:
 * FogExp2: 1 - exp(-density^2 * d^2); Fog: smoothstep(near, far, d); uniforms from scene.fog (SSGIEffect.js:404-412).
 * p->is_debug = 1 (ssgi_compose.frag:21-24, outputColor = textureLod(inputTexture, uv, 0.)): `gi` is the debug view and may be any
 * plane of any size, fetched at the pixel centre with its own sampler: RGBA32F NEAREST (composed, the SSGI target, trOut, velocity,
 * the G-buffer, the G-buffer debug target), RGBA16F LINEAR (dnB), R32F a depth texture, which reads (d, 0, 0, 1).  depth and
 * scene are not read then and may be NULL. */
typedef struct rfx_ssgi_compose_params {
  int32_t use_fog;      /* #define USE_FOG  (scene.fog != null)            */
  int32_t fog_exp2;     /* #define FOG_EXP2 (scene.fog.isFogExp2)          */
  float fog_color[3];
  float fog_near, fog_far, fog_density;
  float camera_near, camera_far;
  int32_t perspective;  /* PERSPECTIVE_CAMERA                              */
  int32_t is_debug;     /* uniform isDebug: pass the GI texture through    */
} rfx_ssgi_compose_params;
rfx_status rfx_ssgi_compose_launch(rfx_ctx* ctx, void* stream, const rfx_ssgi_compose_params* p, const rfx_plane* depth,
                                   const rfx_plane* gi, const rfx_plane* scene,
                                   const rfx_plane* out, uint32_t row0, uint32_t row1);

/* K6. out RGBA16F (rgb = world normal, a = ao); background pixels are not written.  `out` may be smaller than `depth`
 * (AOEffect's resolutionScale < 1: the AO target is (int)(width * scale) x (int)(height * scale), src/ao/AOEffect.js:126-146),
 * never larger: its pixels fetch depth NEAREST by uv and rebuild the normal in depth texels.
 * rfx_hbao_launch = rfx_hbao_launch_ex with normal = NULL and resolution {0, 0}. */
rfx_status rfx_hbao_launch(rfx_ctx* ctx, void* stream, const rfx_hbao_params* p,
                           const rfx_plane* depth, const rfx_plane* out,
                           uint32_t row0, uint32_t row1);
/* normal: NULL (the normal is rebuilt from 9 depth taps) or an RGBA8 plane of any size holding the VIEW-space normal packed as
 * rgb = n * 0.5 + 0.5 (postprocessing's NormalPass target), sampled NEAREST by uv: AOEffect's useNormalPass / normalTexture
 * (src/ao/AOEffect.js:48-55, hbao_utils.glsl:70-79). */
rfx_status rfx_hbao_launch_ex(rfx_ctx* ctx, void* stream, const rfx_hbao_params* p,
                              const rfx_plane* depth, const rfx_plane* normal, const rfx_plane* out,
                              uint32_t row0, uint32_t row1);

/* K6h. Horizon-march AO.  No reference draw exists for it: the reference's hbao.frag has no direction x step loop (SURVEY.md D1),
 * so this pass is an extension, written to the definition in DESIGN.md §1 (K6h) and pinned by tests/horizon_oracle.cpp.
 * Inputs and output are K6's: depth R32F; out RGBA16F (rgb = world normal, a = ao), no larger than depth, background pixels not
 * written; normal NULL (rebuilt from 9 depth taps) or an RGBA8 view-space normal plane of depth's size.  Per pixel: D directions
 * theta_d = 2 pi (d + blue.r / 255) / D, S steps of r / (S + 1) texels (r = the projected `distance`, clamped to max_radius_pixels)
 * jittered by blue.g / 255, one NEAREST depth tap each; ao = clamp(1 - intensity * mean(term), 0, 1).
 * RFX_ERR_BAD_FORMAT / RFX_ERR_SIZE_MISMATCH for the planes, RFX_ERR_INVALID_ARG for a parameter outside its documented range,
 * RFX_ERR_UNSUPPORTED for blue_noise_index 0 (as K6). */
rfx_status rfx_hbao_horizon_launch(rfx_ctx* ctx, void* stream, const rfx_hbao_horizon_params* p,
                                   const rfx_plane* depth, const rfx_plane* out, const rfx_plane* normal);
/* K6h's direction table for `directions` (1..32), built on the host: out[2 * (d * 256 + b) + {0, 1}] = (cos, sin) of
 * theta = 2 pi (d + b / 255) / directions, evaluated in double and rounded to float.  256 * directions pairs. */
rfx_status rfx_hbao_horizon_directions(int32_t directions, float* out);

/* K7. ao RGBA16F (.a; any size: sampled LINEAR by uv, e.g. a reduced-resolution AO target), input/out RGBA16F */
rfx_status rfx_ao_compose_launch(rfx_ctx* ctx, void* stream, const rfx_ao_compose_params* p,
                                 const rfx_plane* depth, const rfx_plane* ao,
                                 const rfx_plane* input, const rfx_plane* out,
                                 uint32_t row0, uint32_t row1);

/* K8. velocity RGBA32F, input/out RGBA16F (input sampled LINEAR) */
rfx_status rfx_motion_blur_launch(rfx_ctx* ctx, void* stream, const rfx_motion_blur_params* p,
                                  const rfx_plane* velocity, const rfx_plane* input,
                                  const rfx_plane* out, uint32_t row0, uint32_t row1);

/* G-buffer ingest.  albedo RGBA8 | RGBA16F (rgb = diffuse colour, a = opacity); normal RGBA16F | RGBA32F (xyz = world normal);
 * material RGBA8 | RGBA16F (r = roughness, g = metalness); emissive RGBA16F (rgb; may be NULL = black); motion RGBA16F | RGBA32F
 * (xy; may be NULL = static); depth R32F.  out_gbuffer / out_velocity RGBA32F (either may be NULL). */
rfx_status rfx_gbuffer_ingest_launch(rfx_ctx* ctx, void* stream, const rfx_ingest_params* p, const rfx_plane* albedo,
                                     const rfx_plane* normal, const rfx_plane* material, const rfx_plane* emissive,
                                     const rfx_plane* motion, const rfx_plane* depth, const rfx_plane* out_gbuffer,
                                     const rfx_plane* out_velocity, uint32_t row0, uint32_t row1);

/* Merged cosmetic effects.  input RGBA16F (sampled LINEAR, clamp), depth R32F (gradual background; else may be NULL), velocity RGBA32F
 * (sparkle; else may be NULL), out RGBA16F (may not alias input). */
rfx_status rfx_effects_launch(rfx_ctx* ctx, void* stream, const rfx_effects_params* p, const rfx_plane* input, const rfx_plane* depth,
                              const rfx_plane* velocity, const rfx_plane* out, uint32_t row0, uint32_t row1);

/* TAAPass.  input RGBA16F, history RGBA8 (the FramebufferTexture copy of the canvas; may alias out: each pixel reads only itself),
 * out RGBA8 (the canvas: clamp, round to nearest) */
rfx_status rfx_taa_launch(rfx_ctx* ctx, void* stream, const rfx_taa_params* p, const rfx_plane* input, const rfx_plane* history,
                          const rfx_plane* out, uint32_t row0, uint32_t row1);

/* GBufferDebugPass (src/gbuffer/debug/GBufferDebugPass.js): one channel of the packed G-buffer decoded by getMaterial
 * (gbuffer_packing.glsl), rgb = the channel, a = 1.  gbuffer and out RGBA32F of the same size.  mode = the index of the channel in
 * ["diffuse", "alpha", "normal", "roughness", "metalness", "emissive"] (SSGIEffect.js:237-239); any other value (an unknown string
 * gives -1 there) shows emissive, the shader's `else` branch.  The pass's `depthTexture` sampler is never bound (it is missing from
 * the material's uniforms, so it keeps unit 0, which is gBufferTexture's): a texel whose gBuffer.r compares equal to 0 - packed
 * albedo bits 0x00000000 or 0x80000000, i.e. the background clear texel and transparent-black albedo - is written (0, 0, 0, 0). */
rfx_status rfx_gbuffer_debug_launch(rfx_ctx* ctx, void* stream, int32_t mode, const rfx_plane* gbuffer, const rfx_plane* out,
                                    uint32_t row0, uint32_t row1);

/* K9. src/traa/shader/traa_compose.frag:3-6  accumulated RGBA16F -> out RGBA16F (a = 1) */
rfx_status rfx_traa_compose_launch(rfx_ctx* ctx, void* stream, const rfx_plane* accumulated,
                                   const rfx_plane* out, uint32_t row0, uint32_t row1);

/* ---- SSGI chain (native mirror of SSGIEffect.update, src/ssgi/SSGIEffect.js:372-404 +
 *      src/denoise/Denoiser.js:97-107): owns ssgiOut / trOut / dnA / dnB / composed and the
 *      cross-frame state (prev matrices, keepData, history). ---------------------------- */
typedef struct rfx_ssgi_chain rfx_ssgi_chain;

/* option denoiseMode of the Denoiser (src/denoise/Denoiser.js:7):
 *   "full"          K2 -> K3 x 2*iterations -> K4; history = the Poisson targets (default)
 *   "full_temporal" K2 -> K4 on the temporal textures; no Poisson pass, so both accumulated textures are the one FramebufferTexture
 *                   copy of the temporal target's first attachment (RGBA32F, LINEAR) — what preset "low" selects (SSGIEffect.js:82-86)
 *   "temporal"      K2 only; output 0 and K1's accumulatedTexture are the temporal pass's first texture
 *   ("denoised" binds an ARRAY of textures to K1's sampler in the reference and cannot run there: rejected with RFX_ERR_UNSUPPORTED) */
#define RFX_DENOISE_FULL 0
#define RFX_DENOISE_FULL_TEMPORAL 1
#define RFX_DENOISE_TEMPORAL 2

typedef struct rfx_ssgi_chain_options {
  uint32_t width, height;
  int32_t denoise_iterations;  /* option denoiseIterations (=> 2*iterations K3 passes) */
  int32_t steps, refine_steps;
  float distance, thickness, env_blur;
  float radius, phi, luma_phi, depth_phi, normal_phi, roughness_phi, specular_phi;
  uint32_t ssgi_flags;         /* RFX_SSGI_* */
  int32_t mode;                /* RFX_MODE_* */
  int32_t blue_noise_start;    /* startIndex of BlueNoiseUtils.js:19 (pinned)          */
  int32_t denoise_mode;        /* RFX_DENOISE_*: option denoiseMode (Denoiser.js:7,45-78); constructor-time, like mode   */
  float resolution_scale;      /* option resolutionScale (SSGIPass.js:52-57): the SSGI target is (int)(width*scale) x (int)(height*scale),
                                  everything else stays at full size; 0 or 1 = full size.  Constructor-time (a size change).      */
  int32_t _pad;
} rfx_ssgi_chain_options;

typedef struct rfx_ssgi_frame {
  rfx_camera cam;              /* current camera (un-jittered)                          */
  const rfx_plane* depth;
  const rfx_plane* gbuffer;
  const rfx_plane* velocity;   /* VelocityDepthNormalPass layout                        */
  const rfx_plane* direct_light; /* may be NULL                                         */
  float camera_pos[3];
  int32_t camera_moved;        /* didCameraMove(...) (src/utils/SceneUtils.js:17-27)    */
} rfx_ssgi_frame;

rfx_status rfx_ssgi_chain_create(rfx_ctx* ctx, const rfx_ssgi_chain_options* opt, rfx_ssgi_chain** out);
void rfx_ssgi_chain_destroy(rfx_ssgi_chain* chain);
rfx_status rfx_ssgi_chain_reset(rfx_ssgi_chain* chain);
/* reactive options (SSGIEffect.makeOptionsReactive, src/ssgi/SSGIEffect.js:157-268): replaces every option except
 * width/height (use a new chain to resize) and resets the temporal history like the reference's setters do. */
rfx_status rfx_ssgi_chain_set_options(rfx_ssgi_chain* chain, const rfx_ssgi_chain_options* opt);
rfx_status rfx_ssgi_chain_render(rfx_ssgi_chain* chain, void* stream, const rfx_ssgi_frame* frame);
/* TRAA frame tail: the second EffectPass of the reference demo's SSGI + TRAA frame (example/main.js:525-532) rendered by the chain
 * after K4 on every frame:  K5 ssgi_compose (of `composed`, depth and frame->direct_light, the composer input buffer SSGIEffect.update
 * binds) rounded to RGBA16F -> K2 in its TRAA form (temporal_reproject.frag with textureCount 1, inputType "diffuse", RGBA16F history
 * sampled LINEAR; src/traa/TRAAEffect.js:21-31) -> K9 traa_compose.  The TRAA pass uses the frame's un-jittered camera and the chain's
 * previous-frame matrices; jittering the rasteriser (TAAUtils.js) stays the host's job.  The fast chain runs the three passes as ONE
 * kernel (the K5 plane never reaches memory); every other chain runs rfx_ssgi_compose_launch -> rfx_temporal_reproject_launch ->
 * rfx_traa_compose_launch.  Both write the same bytes. */
typedef struct rfx_traa_tail_options {
  rfx_ssgi_compose_params compose;    /* K5: fog / isDebug (ssgi_compose.frag:20-44)                                           */
  float max_blend;                    /* TRAAEffect forces 0.9                                                                   */
  float neighborhood_clamp_intensity; /* 1                                                                                   */
  float confidence_power;             /* 4                                                                                   */
  int32_t log_transform;              /* 1                                                                                   */
  int32_t full_accumulate;            /* option fullAccumulate (0); AND-ed with !frame->camera_moved                          */
  int32_t _pad;
} rfx_traa_tail_options;
/* Allocates the tail's planes (TRAA accumulated RGBA16F x 2 by frame parity, K9 output RGBA16F) and renders the tail from the next
 * frame on.  On a chain whose tail is on it replaces the options and resets the TRAA history (keepData 0 on the next frame:
 * TemporalReprojectPass.reset()).  opt == NULL turns the tail off and frees its planes.  With the tail on, a frame without
 * direct_light is RFX_ERR_INVALID_ARG; rfx_ssgi_chain_reset resets the TRAA history too.  A chain attached to a group
 * (rfx_group_attach_chain*) cannot change its tail: RFX_ERR_UNSUPPORTED. */
rfx_status rfx_ssgi_chain_enable_traa(rfx_ssgi_chain* chain, const rfx_traa_tail_options* opt);
/* which: 0 composed (RGBA32F), 1 ssgiOut, 2/3 trOut[0/1], 4/5 dnB[0/1]; with the TRAA tail on: 6 the K9 output (RGBA16F), 7 the TRAA
 * accumulated plane of the latest frame (RGBA16F; next frame's history).  6 / 7 with the tail off: RFX_ERR_NOT_READY. */
rfx_status rfx_ssgi_chain_output(rfx_ssgi_chain* chain, int32_t which, rfx_plane* out);
/* Debug view of the TRAA tail: SSGIEffect's `outputTexture` (src/ssgi/SSGIEffect.js:228-251, picked from the "Debug" list of
 * example/SSGIDebugGUI.js:78-114).  With a view selected, the tail's K5 runs with isDebug and samples the view instead of `composed`
 * (ssgi_compose.frag:21-24), and that image goes through the TRAA pass and K9 as in the demo's frame.  Views:
 *   RFX_DEBUG_VIEW_NONE                    today's tail; also what RFX_DEBUG_VIEW_OUTPUT + 0 (denoiser.texture) selects, since
 *                                          isDebug = outputTexture !== denoiser.texture (SSGIEffect.js:249)
 *   RFX_DEBUG_VIEW_OUTPUT + 1..5           rfx_ssgi_chain_output's planes 1..5 (ssgiOut, trOut[0/1], dnB[0/1]); a plane the
 *                                          configuration does not have is refused with rfx_ssgi_chain_output's status
 *   RFX_DEBUG_VIEW_DEPTH / _VELOCITY / _GBUFFER   the frame's depth, velocity or packed G-buffer plane
 *   RFX_DEBUG_VIEW_GBUFFER_CHANNEL + m     GBufferDebugPass mode m (0..5, see rfx_gbuffer_debug_launch) of the frame's G-buffer,
 *                                          rendered into a chain-owned RGBA32F target every frame before the tail
 * While a view is selected the fast chain runs its tail as the three per-pass launches.  Selecting a view does not reset any
 * history (the reference's outputTexture setter calls no reset()).  A chain in a group of n > 1 takes no view: RFX_ERR_UNSUPPORTED. */
#define RFX_DEBUG_VIEW_NONE (-1)
#define RFX_DEBUG_VIEW_OUTPUT 0
#define RFX_DEBUG_VIEW_DEPTH 8
#define RFX_DEBUG_VIEW_VELOCITY 9
#define RFX_DEBUG_VIEW_GBUFFER 10
#define RFX_DEBUG_VIEW_GBUFFER_CHANNEL 16
rfx_status rfx_ssgi_chain_set_debug_view(rfx_ssgi_chain* chain, int32_t view);
/* host-buffer frame: uploads the four input planes from (pinned) host memory, renders,
 * downloads `composed` into out_host.  This is the call `bench.py`'s e2e leg times. */
typedef struct rfx_ssgi_host_frame {
  rfx_camera cam;
  const float* depth;             /* W*H      fp32 */
  const float* gbuffer;           /* W*H*4    fp32 */
  const float* velocity;          /* W*H*4    fp32 */
  const uint16_t* direct_light;   /* W*H*4    fp16, may be NULL */
  float camera_pos[3];
  int32_t camera_moved;
  float* out_composed;            /* W*H*4    fp32 */
} rfx_ssgi_host_frame;
rfx_status rfx_ssgi_chain_render_host(rfx_ssgi_chain* chain, const rfx_ssgi_host_frame* frame);
/* Pipelined form of the same path (what a per-frame caller such as EffectComposer.render would drive): submit enqueues the
 * frame's H2D copies (copy stream, staging set frame&1), its kernels (context stream) and the D2H of `composed` (third stream),
 * ordered by events only, and returns without waiting; frame i+1 uploads while frame i renders and frame i-1 downloads.
 * wait_host blocks until at most max_in_flight (0 or 1) submitted frames are incomplete.  A frame's host input buffers and
 * out_composed must stay untouched until it is complete, so a caller alternates two host buffer sets:
 *     submit(frame i, set i&1);  wait_host(chain, 1);   // frame i-1 is complete, its set is free for frame i+1
 * render_host(f) == submit_host(f) + wait_host(chain, 0).  Results are bit-identical to rfx_ssgi_chain_render. */
rfx_status rfx_ssgi_chain_submit_host(rfx_ssgi_chain* chain, const rfx_ssgi_host_frame* frame);
rfx_status rfx_ssgi_chain_wait_host(rfx_ssgi_chain* chain, int32_t max_in_flight);

/* ---- row-sharded multi-GPU groups (SURVEY.md §8e; one process per GPU) ------------------------------------------------
 * The path shards by output row band.  Bounded stencils (K2's 5x5 window, the Poisson taps, K4) are RECOMPUTED on row ranges
 * widened by rfx_shard_ranges, so no pass exchanges a halo; the two produced planes the next frame samples at arbitrary uv
 * (`composed` for K1's hit colour, `dn` for K2's history — src/ssgi/pass/SSGIPass.js:88, src/denoise/Denoiser.js:51) are read
 * IN PLACE on the rank that owns the row, through CUDA-IPC peer mappings over NVLink, instead of being replicated.  The group
 * owns an NCCL communicator for its one collective per frame (an all-gather of every rank's device-timed kernel cost, which is
 * also the frame barrier) and the band table with its cost-driven rebalancing.  Results are bit-identical to the single-GPU
 * chain.  NCCL is loaded at run time (libnccl.so.2); without it every entry below returns RFX_ERR_NCCL.
 * A group takes chains created with fast_math on and resolution_scale 1, in every mode and denoise_mode: the fast SSGI chain, and the
 * per-pass chain (mode SSR; denoise_mode full_temporal / temporal).  In a group of n > 1 the per-pass chain double-buffers every plane
 * it keeps across frames by frame parity (at attach time), reads last frame's rows on their owners (K1, K2 and the TRAA history) and
 * carries the texel of a discarded pixel from the owner (K2, K3, K4).  fast_math off or resolution_scale < 1: RFX_ERR_UNSUPPORTED,
 * returned on the refusing rank before any collective, so every rank must pass chains the group takes. */
typedef struct rfx_group rfx_group;
#define RFX_GROUP_ID_BYTES 128
rfx_status rfx_group_get_unique_id(void* id128);   /* rank 0; hand the 128 bytes to the other ranks by any means */
rfx_status rfx_group_create(rfx_ctx* ctx, const void* id128, int32_t rank, int32_t world, rfx_group** out);  /* collective */
/* The same group without NCCL / CUDA IPC: `world` members that live in ONE process (one context each — on one device or on several
 * devices with peer access — or all on the same context).  Create every member with rfx_group_create_inprocess, give every member a
 * chain with identical options (a chain the group does not take - fast_math off, resolution_scale < 1 - is RFX_ERR_UNSUPPORTED; members
 * whose mode, denoise_mode or chain path differ: RFX_ERR_INVALID_ARG), then attach them all at
 * once: the members read each other's history planes through plain
 * device pointers.  The host renders a frame by calling rfx_ssgi_chain_render_sharded for every member (any order, same stream or
 * streams it orders itself) before any member starts the next frame.  Bands are static unless moved with rfx_group_set_bounds.
 * Besides single-process multi-GPU hosts, this is what lets a 1-GPU box exercise the N-band logic (tests/test_gpu_chain.py). */
rfx_status rfx_group_create_inprocess(rfx_ctx* ctx, int32_t rank, int32_t world, rfx_group** out);
rfx_status rfx_group_attach_chains_inprocess(rfx_group* const* groups, rfx_ssgi_chain* const* chains, int32_t world);
void rfx_group_destroy(rfx_group* group);
int32_t rfx_group_rank(const rfx_group* group);
int32_t rfx_group_world(const rfx_group* group);
/* collective: maps every rank's history planes of `chain` (the same options on every rank: a mode, denoise_mode, fast_math or TRAA
 * tail that differs between ranks is RFX_ERR_INVALID_ARG on every rank) */
rfx_status rfx_group_attach_chain(rfx_group* group, rfx_ssgi_chain* chain);
/* band borders: world + 1 ascending rows, bounds[0] = 0, bounds[world] = height; rank r owns rows [bounds[r], bounds[r+1]) */
rfx_status rfx_group_get_bounds(const rfx_group* group, uint32_t* bounds);
rfx_status rfx_group_set_bounds(rfx_group* group, const uint32_t* bounds);   /* same values on every rank; next frame on */
/* every > 0: move the borders towards equal device-timed kernel cost every `every` frames, from times `lag` frames old */
rfx_status rfx_group_set_rebalance(rfx_group* group, int32_t every, int32_t lag);
rfx_status rfx_group_last_costs(const rfx_group* group, float* ms_per_rank);  /* the times the last rebalance used */
/* 1: history rows are read in place on their owner (CUDA IPC peer mappings); 0: the mappings could not be opened on some rank (or
 * RFX_GROUP_EXCHANGE=allgather is set) and the group replicates the history planes with an NCCL exchange after every frame */
int32_t rfx_group_uses_peer_reads(const rfx_group* group);
/* in lockstep on every rank, no communication: applies the border move that is due and returns the borders of the NEXT frame
 * (render_sharded calls it implicitly; a host path calls it first to size its uploads) */
rfx_status rfx_group_begin_frame(rfx_group* group, uint32_t* bounds_out);
rfx_status rfx_group_get_last_bounds(const rfx_group* group, uint32_t* bounds);  /* borders of the most recent frame */
/* collective: completes a full-frame INPUT plane of which every rank uploaded only rows [bounds[r], bounds[r+1]) — one NCCL
 * group of per-rank broadcasts over NVLink (depth / velocity are sampled at arbitrary screen positions by every rank) */
rfx_status rfx_group_allgather_rows(rfx_group* group, void* stream, const rfx_plane* plane, const uint32_t* bounds);
/* collective: one frame; this rank renders its band from full-frame input planes and joins the frame's collective on `stream` */
rfx_status rfx_ssgi_chain_render_sharded(rfx_ssgi_chain* chain, void* stream, const rfx_ssgi_frame* frame);
/* pure host arithmetic, exported for hosts that plan their bands with it (and for the CPU tests): the ranges render_sharded uses,
 * rows [ranges[2k], ranges[2k+1]) of launch k (K1, K2, K3 pass 0.., K4) for the band [own0, own1); n_launches = 3 + n_poisson_passes.
 * n_launches = 4 + n_poisson_passes: the same with the TRAA tail as the last launch; it runs on the band and K4 on the band widened
 * by RFX_TRAA_TAIL_ROWS (every earlier launch widens with it).
 * denoise_mode full_temporal / temporal run no Poisson pass: render_sharded plans them with n_poisson_passes = 0 (K1, K2, K4 and the
 * tail, 3 or 4 launches), so K1 / K2 widen only by K2's window, and maps the chain's launches onto them (K1, K2, then K4 and the tail
 * after the 2 * denoise_iterations Poisson slots, which are not launched).  "temporal" launches no K4 either; its range is K2's. */
#define RFX_TRAA_TAIL_ROWS 4  /* 2: the 5x5 clamp window; 1: its LINEAR fetches at texel centres touch row y +- 1; 1: K9's LINEAR fetch
                                 of the accumulated plane at the pixel centre (same reason).  The TRAA form takes no derivative,
                                 so no quad row is added. */
rfx_status rfx_shard_ranges(uint32_t width, uint32_t height, uint32_t own0, uint32_t own1, int32_t n_poisson_passes, float radius,
                            int32_t ssgi_mode, uint32_t* ranges, uint32_t n_launches);
rfx_status rfx_shard_rebalance(const uint32_t* bounds, const uint32_t* measured_bounds, const float* costs, int32_t n, uint32_t* out);

/* ---- AO chain (native mirror of HBAOEffect.update / HorizonAOEffect.update, src/ao/AOEffect.js:148-178): K6 or K6h into the AO
 *      target -> 2 * iterations Poisson passes (one plane, velocity-layout normals) -> K7 ao_compose, in one call.  Owns the AO target
 *      and the Poisson targets A / B, and the two blue-noise counters (the AO pass's and the denoiser's, each advanced on every read
 *      in that order).  The launches and their bytes are exactly those of the per-pass effect classes. -------------------------- */
typedef struct rfx_ao_chain rfx_ao_chain;
#define RFX_AO_HBAO 0     /* K6: hbao.frag's spp-sample form */
#define RFX_AO_HORIZON 1  /* K6h: the horizon march (directions x steps) */
typedef struct rfx_ao_chain_options {
  uint32_t width, height;         /* output size = depth / velocity / input / output planes                                    */
  int32_t algorithm;              /* RFX_AO_*; constructor-time                                                                 */
  float resolution_scale;         /* (0, 1], 0 = 1: the AO target is (int)(width*s) x (int)(height*s), its `resolution` the
                                     unrounded product (AOEffect.setSize); constructor-time                                     */
  int32_t use_normal_plane;       /* 1: frame->normal (RGBA8 view-space normals) replaces the normal rebuilt from depth         */
  /* K6 (RFX_AO_HBAO) */
  int32_t spp;
  float distance;                 /* K6's aoDistance and K6h's world-space radius                                               */
  float distance_power, bias, thickness;
  /* K6h (RFX_AO_HORIZON): ranges of rfx_hbao_horizon_params */
  int32_t directions, steps;
  float angle_bias, intensity, max_radius_pixels;
  /* Poisson denoise (PoissonDenoisePass with AOEffect's options) */
  int32_t iterations;             /* >= 0; 0: K7 composes the AO target                                                         */
  float radius, phi, luma_phi, depth_phi, normal_phi;
  /* K7 */
  float power, color[3];
  int32_t blue_noise_start;       /* the AO pass's BlueNoiseIndex start                                                         */
  int32_t denoise_blue_noise_start; /* the denoiser's (PoissonDenoisePass's) start                                              */
  int32_t _pad;
} rfx_ao_chain_options;
typedef struct rfx_ao_frame {
  float projection[16], projection_inverse[16], camera_matrix_world[16], view_matrix[16];
  const rfx_plane* depth;         /* R32F, width x height                                                                       */
  const rfx_plane* velocity;      /* RGBA32F VelocityDepthNormalPass layout: the Poisson taps' normals and depths               */
  const rfx_plane* normal;        /* RGBA8 view-space normals when use_normal_plane, else ignored                               */
  const rfx_plane* input;         /* RGBA16F scene colour K7 darkens                                                            */
  const rfx_plane* output;        /* RGBA16F; NULL skips K7 (and `input` is not read)                                            */
} rfx_ao_frame;
rfx_status rfx_ao_chain_create(rfx_ctx* ctx, const rfx_ao_chain_options* opt, rfx_ao_chain** out);
void rfx_ao_chain_destroy(rfx_ao_chain* chain);
/* Replaces the per-frame options.  luma_phi / depth_phi / normal_phi that differ from the current option are clamped to >= 1e-4, as
 * HBAOEffect's setters do (AOEffect.js:106-110); values given at creation are taken as they are.  width, height and resolution_scale
 * (a size change): RFX_ERR_SIZE_MISMATCH; algorithm: RFX_ERR_UNSUPPORTED (create a new chain). */
rfx_status rfx_ao_chain_set_options(rfx_ao_chain* chain, const rfx_ao_chain_options* opt);
/* Back to the state of a new chain: the kept planes are cleared and both blue-noise counters restart (every rank of a group together). */
rfx_status rfx_ao_chain_reset(rfx_ao_chain* chain);
rfx_status rfx_ao_chain_render(rfx_ao_chain* chain, void* stream, const rfx_ao_frame* frame);
/* which: 0 the AO target (RGBA16F, the scaled size), 1 the denoised plane K7 composes (Poisson target B; the AO target with
 * iterations 0), of the latest frame */
rfx_status rfx_ao_chain_output(rfx_ao_chain* chain, int32_t which, rfx_plane* out);
/* Row-sharded AO.  A group takes an AO chain or an SSGI chain, never both (RFX_ERR_INVALID_ARG).  No AO pass reads a produced plane at
 * an arbitrary uv: K6 / K6h read the caller's depth, the Poisson taps and K7 are bounded stencils, recomputed on widened ranges
 * (rfx_ao_shard_ranges).  In a group of n > 1 the AO target and Poisson targets A / B are double-buffered by frame parity and
 * peer-mapped at attach time, and a discarded (background) pixel of K6 / K6h / K3 carries last frame's texel from the rank that owns the
 * row.  Both algorithms, every iteration count, with or without a normal plane, fast_math on or off.  resolution_scale < 1 (the rows
 * of a smaller AO target do not map 1:1 onto output rows) and fewer than 64 rows per rank: RFX_ERR_UNSUPPORTED; members whose
 * algorithm or iterations differ: RFX_ERR_INVALID_ARG.  Results are bit-identical to one rfx_ao_chain. */
rfx_status rfx_group_attach_ao_chain(rfx_group* group, rfx_ao_chain* chain);  /* collective */
rfx_status rfx_group_attach_ao_chains_inprocess(rfx_group* const* groups, rfx_ao_chain* const* chains, int32_t world);
rfx_status rfx_ao_chain_render_sharded(rfx_ao_chain* chain, void* stream, const rfx_ao_frame* frame);  /* collective */
/* pure host arithmetic: rows [ranges[2k], ranges[2k+1]) of launch k (K6 / K6h, Poisson pass 0 .. 2*iterations-1, K7) for the band
 * [own0, own1); n_launches = 2 + 2 * iterations.  K7 runs on the band, the last Poisson pass on the band +- 1 row (K7's LINEAR fetch at
 * the pixel centre; with iterations 0 K6 gets those rows), and every earlier launch on the next one's range widened by the Poisson halo
 * ceil(|radius| * max(1, height / width)) + 1. */
rfx_status rfx_ao_shard_ranges(uint32_t width, uint32_t height, uint32_t own0, uint32_t own1, int32_t iterations, float radius,
                               uint32_t* ranges, uint32_t n_launches);

/* Per-pass device timing (CUDA events recorded on the launching stream around every kernel of
 * the chain).  Slots: 0 K1 trace, 1 K2 temporal, 2 K3 pass 0, 3 K3 passes >= 1, 4 K4 compose.
 * get_profile synchronises the stream, adds the elapsed milliseconds / launch counts of all
 * frames rendered since the last call into ms[5] / launches[5] and clears the record. */
#define RFX_CHAIN_PROFILE_SLOTS 5
rfx_status rfx_ssgi_chain_set_profiling(rfx_ssgi_chain* chain, int32_t enable);
rfx_status rfx_ssgi_chain_get_profile(rfx_ssgi_chain* chain, double* ms, uint64_t* launches);

#ifdef __cplusplus
}
#endif
#endif /* RFX_H */
