// rfx_api.cu — implementation of the C ABI declared in include/rfx.h.
//
// Host-side responsibilities: argument validation, plane bookkeeping, the small per-context
// tables the kernels index by 8-bit blue-noise values, the env-map mip chain, and the native
// SSGI chain (the mirror of SSGIEffect.update / Denoiser.render frame logic).  No torch types, no
// exceptions across the boundary, no CPU fallback: every compute entry point launches a kernel.
#include <algorithm>
#include <array>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "rfx_kernels.h"

using namespace rfx;

struct rfx_ctx {
  int device = 0;
  cudaStream_t stream = nullptr;
  std::string err;
  uint64_t launches = 0;
  // blue noise
  uchar4* blue = nullptr;
  int blue_size = 0;
  // tables
  float2* rot_table = nullptr;  // [256]
  float* step_table = nullptr;  // [steps-1][256]
  int step_table_steps = 0;
  float2* horizon_dirs[33] = {};  // K6h direction table per `directions` value, built on first use and kept (never rewritten)
  // env
  bool env_set = false;
  double env_total = 0.0;  // totalSumValue of the device-built tables (rfx_env_build)
  EnvD env{};
  std::vector<void*> env_allocs;
  // fast-math kernel variants (SFU lg2/ex2 instead of libm polynomials); 0 selects the exact-libm variants
  int fast_math = 1;
  // scratch: decoded G-buffer (float4 normal.xyz + roughness) for the fast Poisson kernel
  void* nrd = nullptr;
  int nrd_w = 0, nrd_h = 0;
  size_t nrd_pitch = 0;
  // scratch: view-space z plane for the SSGI march
  void* viewz = nullptr;
  int viewz_w = 0, viewz_h = 0;
  size_t viewz_pitch = 0;
  // default measured on H100 at 4K with tools/sweep_k1.sh
  int k3_tma = 1;     // RFX_K3_TMA=0 disables the TMA-staged tap tiles of the Poisson passes >= 1 (same bytes out; ~6 % slower per pass)
};

static rfx_status fail(rfx_ctx* c, rfx_status st, const char* fmt, ...) {
  if (c) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    c->err = buf;
  }
  return st;
}
#define CU(call)                                                                                        \
  do {                                                                                                  \
    cudaError_t e_ = (call);                                                                            \
    if (e_ != cudaSuccess) return fail(ctx, RFX_ERR_CUDA, "%s failed: %s", #call, cudaGetErrorString(e_)); \
  } while (0)

static const float kPi = 3.1415926535897932384626433832795f;

extern "C" {

int rfx_version(void) { return RFX_VERSION; }
uint32_t rfx_format_bytes(int32_t f) { return f == RFX_FMT_R32F ? 4u : f == RFX_FMT_RGBA32F ? 16u : f == RFX_FMT_RGBA16F ? 8u : f == RFX_FMT_RGBA8 ? 4u : 0u; }

rfx_status rfx_ctx_create(int device, rfx_ctx** out) {
  if (!out) return RFX_ERR_INVALID_ARG;
  *out = nullptr;
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || device < 0 || device >= n) return RFX_ERR_CUDA;
  rfx_ctx* ctx = new rfx_ctx();
  ctx->device = device;
  if (const char* e = getenv("RFX_K3_TMA")) ctx->k3_tma = atoi(e);
  if (cudaSetDevice(device) != cudaSuccess || cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) != cudaSuccess) {
    delete ctx;
    return RFX_ERR_CUDA;
  }
  // (sin, cos) of the fp32 angle (k/255)*2*pi, correctly rounded: the 256 values blueNoise().r/.g can take
  float2 rot[256];
  for (int k = 0; k < 256; k++) {
    volatile float r = (float)k / 255.0f;
    volatile float r2 = r * 2.0f;
    volatile float ang = r2 * kPi;
    rot[k].x = (float)std::sin((double)ang);
    rot[k].y = (float)std::cos((double)ang);
  }
  if (cudaMalloc(&ctx->rot_table, sizeof rot) != cudaSuccess || cudaMemcpy(ctx->rot_table, rot, sizeof rot, cudaMemcpyHostToDevice) != cudaSuccess) {
    cudaStreamDestroy(ctx->stream);
    delete ctx;
    return RFX_ERR_CUDA;
  }
  *out = ctx;
  return RFX_OK;
}

static void free_env(rfx_ctx* ctx) {
  for (void* p : ctx->env_allocs) cudaFree(p);
  ctx->env_allocs.clear();
  ctx->env_set = false;
  ctx->env = EnvD{};
}

void rfx_ctx_destroy(rfx_ctx* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  cudaStreamSynchronize(ctx->stream);
  free_env(ctx);
  cudaFree(ctx->blue);
  cudaFree(ctx->rot_table);
  cudaFree(ctx->step_table);
  for (float2* t : ctx->horizon_dirs) cudaFree(t);
  cudaFree(ctx->nrd);
  cudaFree(ctx->viewz);
  cudaStreamDestroy(ctx->stream);
  delete ctx;
}
rfx_status rfx_ctx_set_fast_math(rfx_ctx* ctx, int32_t enable) {
  if (!ctx) return RFX_ERR_INVALID_ARG;
  ctx->fast_math = enable ? 1 : 0;
  return RFX_OK;
}
const char* rfx_last_error(const rfx_ctx* ctx) { return ctx ? ctx->err.c_str() : "null context"; }
void* rfx_ctx_stream(rfx_ctx* ctx) { return ctx ? (void*)ctx->stream : nullptr; }
rfx_status rfx_ctx_sync(rfx_ctx* ctx) {
  if (!ctx) return RFX_ERR_INVALID_ARG;
  CU(cudaStreamSynchronize(ctx->stream));
  return RFX_OK;
}
uint64_t rfx_launch_count(const rfx_ctx* ctx) { return ctx ? ctx->launches : 0; }

rfx_status rfx_blue_noise_set(rfx_ctx* ctx, const uint8_t* rgba8, uint32_t w, uint32_t h) {
  if (!ctx || !rgba8 || w != h || w == 0) return fail(ctx, RFX_ERR_INVALID_ARG, "blue noise must be a square RGBA8 image");
  CU(cudaSetDevice(ctx->device));
  cudaFree(ctx->blue);
  ctx->blue = nullptr;
  CU(cudaMalloc(&ctx->blue, (size_t)w * h * 4));
  CU(cudaMemcpy(ctx->blue, rgba8, (size_t)w * h * 4, cudaMemcpyHostToDevice));
  ctx->blue_size = (int)w;
  return RFX_OK;
}

// ---- planes -----------------------------------------------------------------------------
rfx_status rfx_plane_alloc(rfx_ctx* ctx, int32_t format, uint32_t w, uint32_t h, rfx_plane* out) {
  if (!ctx || !out || w == 0 || h == 0 || rfx_format_bytes(format) == 0) return fail(ctx, RFX_ERR_INVALID_ARG, "plane_alloc: bad arguments");
  CU(cudaSetDevice(ctx->device));
  size_t pitch = ((size_t)w * rfx_format_bytes(format) + 255) & ~(size_t)255;
  void* p = nullptr;
  CU(cudaMalloc(&p, pitch * h));
  CU(cudaMemsetAsync(p, 0, pitch * h, ctx->stream));  // targets are zero after allocation (SURVEY.md A2)
  CU(cudaStreamSynchronize(ctx->stream));
  out->ptr = p; out->width = w; out->height = h; out->pitch = pitch; out->format = format; out->_reserved = 0;
  return RFX_OK;
}
rfx_status rfx_plane_free(rfx_ctx* ctx, rfx_plane* p) {
  if (!ctx || !p) return RFX_ERR_INVALID_ARG;
  CU(cudaSetDevice(ctx->device));
  CU(cudaFree(p->ptr));
  p->ptr = nullptr;
  return RFX_OK;
}
static cudaStream_t pick(rfx_ctx* ctx, void* s) { return s ? (cudaStream_t)s : ctx->stream; }
rfx_status rfx_plane_clear(rfx_ctx* ctx, void* stream, const rfx_plane* p) {
  if (!ctx || !p || !p->ptr) return RFX_ERR_INVALID_ARG;
  CU(cudaMemsetAsync(p->ptr, 0, p->pitch * p->height, pick(ctx, stream)));
  return RFX_OK;
}
rfx_status rfx_plane_upload(rfx_ctx* ctx, void* stream, const rfx_plane* dst, const void* host, uint64_t host_pitch) {
  if (!ctx || !dst || !dst->ptr || !host) return RFX_ERR_INVALID_ARG;
  size_t row = (size_t)dst->width * rfx_format_bytes(dst->format);
  if (host_pitch == 0) host_pitch = row;
  if (host_pitch == row && dst->pitch == row) CU(cudaMemcpyAsync(dst->ptr, host, row * dst->height, cudaMemcpyHostToDevice, pick(ctx, stream)));  // one contiguous DMA
  else CU(cudaMemcpy2DAsync(dst->ptr, dst->pitch, host, host_pitch, row, dst->height, cudaMemcpyHostToDevice, pick(ctx, stream)));
  return RFX_OK;
}
rfx_status rfx_plane_download(rfx_ctx* ctx, void* stream, const rfx_plane* src, void* host, uint64_t host_pitch) {
  if (!ctx || !src || !src->ptr || !host) return RFX_ERR_INVALID_ARG;
  size_t row = (size_t)src->width * rfx_format_bytes(src->format);
  if (host_pitch == 0) host_pitch = row;
  if (host_pitch == row && src->pitch == row) CU(cudaMemcpyAsync(host, src->ptr, row * src->height, cudaMemcpyDeviceToHost, pick(ctx, stream)));
  else CU(cudaMemcpy2DAsync(host, host_pitch, src->ptr, src->pitch, row, src->height, cudaMemcpyDeviceToHost, pick(ctx, stream)));
  return RFX_OK;
}
rfx_status rfx_plane_download_rows(rfx_ctx* ctx, void* stream, const rfx_plane* src, void* host, uint32_t row0, uint32_t row1) {
  if (!ctx || !src || !src->ptr || !host || row0 >= row1 || row1 > src->height) return RFX_ERR_INVALID_ARG;
  const size_t row = (size_t)src->width * rfx_format_bytes(src->format);
  const unsigned char* p = (const unsigned char*)src->ptr + (size_t)row0 * src->pitch;
  if (src->pitch == row) CU(cudaMemcpyAsync(host, p, row * (row1 - row0), cudaMemcpyDeviceToHost, pick(ctx, stream)));
  else CU(cudaMemcpy2DAsync(host, row, p, src->pitch, row, row1 - row0, cudaMemcpyDeviceToHost, pick(ctx, stream)));
  return RFX_OK;
}
rfx_status rfx_host_alloc(rfx_ctx* ctx, uint64_t bytes, void** out) {
  if (!ctx || !out) return RFX_ERR_INVALID_ARG;
  CU(cudaSetDevice(ctx->device));
  CU(cudaHostAlloc(out, bytes, cudaHostAllocDefault));
  return RFX_OK;
}
rfx_status rfx_host_free(rfx_ctx* ctx, void* p) {
  if (!ctx) return RFX_ERR_INVALID_ARG;
  CU(cudaFreeHost(p));
  return RFX_OK;
}

// ---- env map ----------------------------------------------------------------------------
rfx_status rfx_env_clear(rfx_ctx* ctx) {
  if (!ctx) return RFX_ERR_INVALID_ARG;
  cudaSetDevice(ctx->device);
  cudaStreamSynchronize(ctx->stream);
  free_env(ctx);
  return RFX_OK;
}
rfx_status rfx_env_set(rfx_ctx* ctx, const rfx_env_desc* e) {
  if (!ctx || !e || !e->map_rgba16f || e->width == 0 || e->height == 0) return fail(ctx, RFX_ERR_INVALID_ARG, "env_set: bad arguments");
  CU(cudaSetDevice(ctx->device));
  CU(cudaStreamSynchronize(ctx->stream));
  free_env(ctx);
  int w = (int)e->width, h = (int)e->height, l = 0;
  EnvD d{};
  for (;;) {
    if (l >= 16) return fail(ctx, RFX_ERR_UNSUPPORTED, "env map too large");
    size_t pitch = ((size_t)w * 8 + 255) & ~(size_t)255;
    void* p = nullptr;
    CU(cudaMalloc(&p, pitch * h));
    ctx->env_allocs.push_back(p);
    d.mip[l] = PV{(const unsigned char*)p, w, h, (long long)pitch};
    if (l == 0) {
      CU(cudaMemcpy2DAsync(p, pitch, e->map_rgba16f, (size_t)w * 8, (size_t)w * 8, h, cudaMemcpyHostToDevice, ctx->stream));
    } else {
      cudaError_t ce = launch_env_downsample(d.mip[l - 1], OutV{(unsigned char*)p, (long long)pitch}, w, h, ctx->stream);
      if (ce != cudaSuccess) return fail(ctx, RFX_ERR_CUDA, "env downsample: %s", cudaGetErrorString(ce));
      ctx->launches++;
    }
    l++;
    if (w == 1 && h == 1) break;
    w = w > 1 ? w >> 1 : 1;
    h = h > 1 ? h >> 1 : 1;
  }
  d.levels = l;
  d.size_x = (float)e->width;
  d.size_y = (float)e->height;
  d.total_sum_whole = e->total_sum_whole;
  d.total_sum_decimal = e->total_sum_decimal;
  ctx->env_total = (double)e->total_sum_whole + (double)e->total_sum_decimal;
  if (e->marginal && e->conditional) {
    float *m = nullptr, *c = nullptr;
    CU(cudaMalloc(&m, (size_t)e->height * 4));
    ctx->env_allocs.push_back(m);
    CU(cudaMalloc(&c, (size_t)e->width * e->height * 4));
    ctx->env_allocs.push_back(c);
    CU(cudaMemcpyAsync(m, e->marginal, (size_t)e->height * 4, cudaMemcpyHostToDevice, ctx->stream));
    CU(cudaMemcpyAsync(c, e->conditional, (size_t)e->width * e->height * 4, cudaMemcpyHostToDevice, ctx->stream));
    d.marginal = PV{(const unsigned char*)m, (int)e->height, 1, (long long)e->height * 4};  // image {width: height, height: 1}
    d.conditional = PV{(const unsigned char*)c, (int)e->width, (int)e->height, (long long)e->width * 4};
  }
  CU(cudaStreamSynchronize(ctx->stream));
  ctx->env = d;
  ctx->env_set = true;
  return RFX_OK;
}

// Env map + importance-sampling tables built ON THE DEVICE (SURVEY.md §8f row 1; replaces the reference's Web Worker,
// src/ssgi/utils/EquirectHdrInfoUniform.js:323-358 -> gatherData :149-245): uploads mip 0, builds the mip chain, the per-row
// cumulative distributions and the two inverse-CDF tables with the JS loops' summation order (bit-identical tables).
rfx_status rfx_env_build(rfx_ctx* ctx, const void* map_rgba16f, uint32_t width, uint32_t height, int32_t flip_y) {
  if (!ctx || !map_rgba16f || width == 0 || height == 0) return fail(ctx, RFX_ERR_INVALID_ARG, "env_build: bad arguments");
  rfx_env_desc e{};
  e.map_rgba16f = map_rgba16f; e.width = width; e.height = height;
  rfx_status st = rfx_env_set(ctx, &e);  // mip chain; no tables yet
  if (st != RFX_OK) return st;
  const size_t n = (size_t)width * height;
  float *cdf_c = nullptr, *cdf_m = nullptr, *marg = nullptr, *cond = nullptr;
  double *row_sum = nullptr, *total = nullptr;
  CU(cudaMalloc(&cdf_c, n * 4)); CU(cudaMalloc(&cdf_m, (size_t)height * 4)); CU(cudaMalloc(&row_sum, (size_t)height * 8)); CU(cudaMalloc(&total, 8));
  CU(cudaMalloc(&marg, (size_t)height * 4)); ctx->env_allocs.push_back(marg);
  CU(cudaMalloc(&cond, n * 4)); ctx->env_allocs.push_back(cond);
  cudaError_t ce = launch_env_cdf(ctx->env.mip[0], flip_y ? 1 : 0, cdf_c, cdf_m, row_sum, total, marg, cond, ctx->stream);
  ctx->launches += 3;
  double t = 0.0;
  if (ce == cudaSuccess) ce = cudaMemcpyAsync(&t, total, 8, cudaMemcpyDeviceToHost, ctx->stream);
  if (ce == cudaSuccess) ce = cudaStreamSynchronize(ctx->stream);
  cudaFree(cdf_c); cudaFree(cdf_m); cudaFree(row_sum); cudaFree(total);
  if (ce != cudaSuccess) return fail(ctx, RFX_ERR_CUDA, "env_build: %s", cudaGetErrorString(ce));
  ctx->env.marginal = PV{(const unsigned char*)marg, (int)height, 1, (long long)height * 4};
  ctx->env.conditional = PV{(const unsigned char*)cond, (int)width, (int)height, (long long)width * 4};
  const double whole = (double)(int32_t)t;  // ~~totalSumValue (EquirectHdrInfoUniform.js:346-349)
  ctx->env.total_sum_whole = (float)whole;
  ctx->env.total_sum_decimal = (float)(t - whole);
  ctx->env_total = t;
  return RFX_OK;
}
// the tables of the current environment (host copies): marginal[height], conditional[width*height], totalSum; any pointer may be NULL
rfx_status rfx_env_tables_download(rfx_ctx* ctx, float* marginal, float* conditional, double* total_sum) {
  if (!ctx) return RFX_ERR_INVALID_ARG;
  if (!ctx->env_set || !ctx->env.marginal.p) return fail(ctx, RFX_ERR_NOT_READY, "env_tables_download: no importance-sampling tables");
  CU(cudaStreamSynchronize(ctx->stream));
  if (marginal) CU(cudaMemcpy(marginal, ctx->env.marginal.p, (size_t)ctx->env.marginal.w * 4, cudaMemcpyDeviceToHost));
  if (conditional) CU(cudaMemcpy(conditional, ctx->env.conditional.p, (size_t)ctx->env.conditional.w * ctx->env.conditional.h * 4, cudaMemcpyDeviceToHost));
  if (total_sum) *total_sum = ctx->env_total;
  return RFX_OK;
}

}  // extern "C"

// ---- helpers ------------------------------------------------------------------------------
static bool plane_ok(const rfx_plane* p, int fmt) {  // kernels address planes with 32-bit byte offsets
  return p && p->ptr && p->format == fmt && p->pitch * (uint64_t)p->height < (1ull << 32) && (p->pitch % rfx_format_bytes(fmt)) == 0;
}
static bool pv(const rfx_plane* p, int fmt, PV& out) {
  if (!plane_ok(p, fmt)) return false;
  out = PV{(const unsigned char*)p->ptr, (int)p->width, (int)p->height, (long long)p->pitch};
  return true;
}
static bool ov(const rfx_plane* p, int fmt, OutV& out) {
  if (!plane_ok(p, fmt)) return false;
  out = OutV{(unsigned char*)p->ptr, (long long)p->pitch};
  return true;
}
static void cam_to_dev(const rfx_camera& c, CamD& d) {
  memcpy(d.projection.m, c.projection, 64);
  memcpy(d.projection_inverse.m, c.projection_inverse, 64);
  memcpy(d.camera_matrix_world.m, c.camera_matrix_world, 64);
  memcpy(d.view_matrix.m, c.view_matrix, 64);
  d.near_plane = c.near_plane;
  d.far_plane = c.far_plane;
  d.perspective = c.perspective;
}
// pcg4d  (reference src/utils/shader/blue_noise.glsl:17-28), integer, bit-exact
static void pcg4d(uint32_t v[4]) {
  for (int i = 0; i < 4; i++) v[i] = v[i] * 1664525u + 1013904223u;
  v[0] += v[1] * v[3]; v[1] += v[2] * v[0]; v[2] += v[0] * v[1]; v[3] += v[1] * v[2];
  for (int i = 0; i < 4; i++) v[i] ^= v[i] >> 16;
  v[0] += v[1] * v[3]; v[1] += v[2] * v[0]; v[2] += v[0] * v[1]; v[3] += v[1] * v[2];
}
static rfx_status blue_for(rfx_ctx* ctx, int index, BlueD& b) {
  if (!ctx->blue) return fail(ctx, RFX_ERR_NOT_READY, "blue noise texture not set (rfx_blue_noise_set)");
  uint32_t ui = (uint32_t)index;
  uint32_t s1[4] = {ui, ui * 15843u, ui * 31u + 4566u, ui * 2345u + 58585u};  // rng_initialize :13
  pcg4d(s1);
  b.tex = ctx->blue;
  b.size = ctx->blue_size;
  b.shift.sx = (int)((s1[0] % 0x0fffffffu) % (uint32_t)ctx->blue_size);  // shift2 :31-34
  b.shift.sy = (int)((s1[1] % 0x0fffffffu) % (uint32_t)ctx->blue_size);
  b.index = index;
  b.mask = (ctx->blue_size & (ctx->blue_size - 1)) == 0 ? ctx->blue_size - 1 : 0;
  return RFX_OK;
}
static void rows(uint32_t row0, uint32_t row1, uint32_t H, int& r0, int& r1) {
  if (row0 == 0 && row1 == 0) { r0 = 0; r1 = (int)H; }
  else { r0 = (int)row0; r1 = (int)(row1 > H ? H : row1); }
}
// mat4 * mat4 with the oracle's lowering: s = ((a0*b0 + a1*b1) + a2*b2) + a3*b3, no contraction
static void matmul(const float* A, const float* B, float* R) {
  for (int c = 0; c < 4; c++)
    for (int r = 0; r < 4; r++) {
      volatile float s = 0.0f;
      for (int k = 0; k < 4; k++) {
        volatile float p = A[k * 4 + r] * B[c * 4 + k];
        s = s + p;
      }
      R[c * 4 + r] = s;
    }
}
static rfx_status ensure_step_table(rfx_ctx* ctx, int steps) {
  if (ctx->step_table && ctx->step_table_steps == steps) return RFX_OK;
  if (steps < 1 || steps > 4096) return fail(ctx, RFX_ERR_INVALID_ARG, "steps out of range");
  CU(cudaStreamSynchronize(ctx->stream));
  cudaFree(ctx->step_table);
  ctx->step_table = nullptr;
  int rows_n = steps + 4;  // rows 0..steps-2 hold cs(1..steps-1, b); spare zero rows: the fast march reads up to 3 steps ahead
  std::vector<float> t((size_t)rows_n * 256, 0.0f);
  for (int i = 1; i < steps; i++)
    for (int k = 0; k < 256; k++) {  // ssgi.frag:453   cs = 1. - exp(-0.25 * pow(float(i) + random.b - 0.5, 2.))
      volatile float b = (float)k / 255.0f;
      volatile float u = (float)i + b;
      volatile float v = u - 0.5f;
      volatile float p = (float)std::pow((double)v, 2.0);
      volatile float q = -0.25f * p;
      volatile float e = (float)std::exp((double)q);
      t[(size_t)(i - 1) * 256 + k] = 1.0f - e;
    }
  CU(cudaMalloc(&ctx->step_table, t.size() * 4));
  CU(cudaMemcpy(ctx->step_table, t.data(), t.size() * 4, cudaMemcpyHostToDevice));
  ctx->step_table_steps = steps;
  return RFX_OK;
}
// K2's uniforms for an a.W x a.H target
static void temporal_uniforms(const rfx_ctx* ctx, const rfx_temporal_params* p, TemporalArgs& a) {
  cam_to_dev(p->cam, a.cam);
  memcpy(a.prev_view.m, p->prev_view_matrix, 64);
  memcpy(a.prev_world.m, p->prev_camera_matrix_world, 64);
  memcpy(a.prev_proj.m, p->prev_projection, 64);
  memcpy(a.prev_proj_inv.m, p->prev_projection_inverse, 64);
  matmul(p->prev_projection, p->prev_view_matrix, a.prev_proj_view.m);
  memcpy(a.camera_pos, p->camera_pos, 12);
  a.max_blend = p->max_blend; a.clamp_intensity = p->neighborhood_clamp_intensity; a.keep_data = p->keep_data; a.confidence_power = p->confidence_power;
  a.inv_w = (float)(1.0 / (double)a.W);  // TemporalReprojectPass.js:135: JS doubles, uploaded as float32
  a.inv_h = (float)(1.0 / (double)a.H);
  a.full_accumulate = p->full_accumulate; a.texture_count = p->texture_count; a.input_type = p->input_type; a.log_transform = p->log_transform;
  a.rs0 = p->reproject_specular[0]; a.rs1 = p->reproject_specular[1]; a.history_linear = p->history_linear;
  a.fast = ctx->fast_math;
}
#define LAUNCHED(expr)                                                                                   \
  do {                                                                                                   \
    cudaError_t e_ = (expr);                                                                             \
    if (e_ != cudaSuccess) return fail(ctx, RFX_ERR_CUDA, "%s: %s", #expr, cudaGetErrorString(e_));      \
    ctx->launches++;                                                                                     \
  } while (0)

extern "C" {

// The four per-pass entry points the native chain drives are split in two: the extern "C" wrapper checks its pointers and resolves
// the row arguments (row0 == row1 == 0: every row); the static implementation validates the planes and launches over output rows
// [r0, r1), with what only the chain knows passed explicitly.

// K1.  acc_peer: K1's `accumulated` in a row-sharded group, whose rows live on their owners (nullptr: the local plane)
static rfx_status ssgi_trace(rfx_ctx* ctx, void* stream, const rfx_ssgi_params* p, const rfx_plane* depth, const rfx_plane* gbuffer, const rfx_plane* velocity,
                             const rfx_plane* direct_light, const rfx_plane* accumulated, const rfx_plane* out, int r0, int r1, const PeerPV* acc_peer) {
  SsgiArgs a{};
  if (!pv(depth, RFX_FMT_R32F, a.depth) || !pv(gbuffer, RFX_FMT_RGBA32F, a.gb) || !ov(out, RFX_FMT_RGBA32F, a.out))
    return fail(ctx, RFX_ERR_BAD_FORMAT, "ssgi_trace: depth must be R32F, gbuffer/out RGBA32F");
  if (velocity && !pv(velocity, RFX_FMT_RGBA32F, a.velocity)) return fail(ctx, RFX_ERR_BAD_FORMAT, "ssgi_trace: velocity must be RGBA32F");
  if (direct_light && !pv(direct_light, RFX_FMT_RGBA16F, a.direct)) return fail(ctx, RFX_ERR_BAD_FORMAT, "ssgi_trace: direct light must be RGBA16F");
  if (accumulated && !pv(accumulated, RFX_FMT_RGBA32F, a.accumulated)) return fail(ctx, RFX_ERR_BAD_FORMAT, "ssgi_trace: accumulated must be RGBA32F");
  a.W = (int)out->width; a.H = (int)out->height;
  const int TW = a.depth.w, TH = a.depth.h;  // the input planes share one size; the render target may be smaller (resolutionScale < 1, SSGIPass.js:52-57)
  if (a.gb.w != TW || a.gb.h != TH || (a.velocity.p && (a.velocity.w != TW || a.velocity.h != TH)) ||
      (a.direct.p && (a.direct.w != TW || a.direct.h != TH)) || (a.accumulated.p && (a.accumulated.w != TW || a.accumulated.h != TH)))
    return fail(ctx, RFX_ERR_SIZE_MISMATCH, "ssgi_trace: depth / gbuffer / velocity / direct light / accumulated must have one size");
  if (a.W > TW || a.H > TH) return fail(ctx, RFX_ERR_SIZE_MISMATCH, "ssgi_trace: the output may be smaller than the input planes (resolutionScale <= 1), not larger");
  a.scaled = a.W != TW || a.H != TH;
  if (p->steps < 1 || p->refine_steps < 0 || (p->mode != RFX_MODE_SSGI && p->mode != RFX_MODE_SSR)) return fail(ctx, RFX_ERR_INVALID_ARG, "ssgi_trace: bad steps/mode");
  a.row0 = r0; a.row1 = r1;
  cam_to_dev(p->cam, a.cam);
  a.ray_distance = p->ray_distance; a.thickness = p->thickness; a.env_blur = p->env_blur; a.max_env_mip = p->max_env_map_mip_level;
  a.near_minus_far = p->cam.near_plane - p->cam.far_plane;  // SSGIPass.js:85-87
  a.far_minus_near = p->cam.far_plane - p->cam.near_plane;
  a.near_mul_far = p->cam.near_plane * p->cam.far_plane;
  a.steps = p->steps; a.refine_steps = p->refine_steps; a.mode = p->mode; a.flags = p->flags;
  if (p->flags & (RFX_SSGI_USE_ENVMAP | RFX_SSGI_IMPORTANCE_SAMPLING)) {
    if (!ctx->env_set) return fail(ctx, RFX_ERR_NOT_READY, "ssgi_trace: env map requested but rfx_env_set was not called");
    if ((p->flags & RFX_SSGI_IMPORTANCE_SAMPLING) && !ctx->env.marginal.p) return fail(ctx, RFX_ERR_NOT_READY, "ssgi_trace: importance sampling needs CDF tables");
    a.env = ctx->env;
  }
  rfx_status st = blue_for(ctx, p->blue_noise_index, a.blue);
  if (st != RFX_OK) return st;
  if (p->blue_noise_index == 0) return fail(ctx, RFX_ERR_UNSUPPORTED, "ssgi_trace: blue_noise_index 0 (tiled lookup) is not used by this pass");
  st = ensure_step_table(ctx, p->steps);
  if (st != RFX_OK) return st;
  a.rot_table = ctx->rot_table;
  a.step_table = ctx->step_table;
  a.fast = ctx->fast_math;
  {  // perspective sparsity pattern: [P00 0 P20 0; 0 P11 P21 0; 0 0 P22 P32; 0 0 -1 0] (column-major m[col*4+row])
    const float* M = p->cam.projection;
    a.proj_sparse = M[1] == 0.0f && M[2] == 0.0f && M[3] == 0.0f && M[4] == 0.0f && M[6] == 0.0f && M[7] == 0.0f && M[11] == -1.0f &&
                    M[12] == 0.0f && M[13] == 0.0f && M[15] == 0.0f;
  }
  // view-space z plane (scratch): the march taps read it instead of converting depth -> viewZ per tap
  if (!ctx->viewz || ctx->viewz_w != TW || ctx->viewz_h != TH) {
    CU(cudaStreamSynchronize(ctx->stream));
    cudaFree(ctx->viewz);
    ctx->viewz = nullptr;
    ctx->viewz_pitch = ((size_t)TW * 4 + 255) & ~(size_t)255;
    CU(cudaMalloc(&ctx->viewz, ctx->viewz_pitch * TH));
    ctx->viewz_w = TW; ctx->viewz_h = TH;
  }
  {  // fast fused kernel: projection rows in texel units (0.5 W P00, 0.5 W P20, 0.5 H P11, 0.5 H P21), word pitch of the viewZ plane
    const float* M = p->cam.projection;
    const float hw = 0.5f * (float)a.W, hh = 0.5f * (float)a.H;
    a.ps_x0 = hw * M[0]; a.ps_x2 = hw * M[8]; a.ps_y1 = hh * M[5]; a.ps_y2 = hh * M[9]; a.ps_hw = hw; a.ps_hh = hh;
    a.vz_pitchw = (int)(ctx->viewz_pitch / 4);
    if (acc_peer) a.acc_peer = *acc_peer;
  }
  LAUNCHED(launch_viewz(a, OutV{(unsigned char*)ctx->viewz, (long long)ctx->viewz_pitch}, pick(ctx, stream)));
  a.viewz = PV{(const unsigned char*)ctx->viewz, TW, TH, (long long)ctx->viewz_pitch};
  LAUNCHED(launch_ssgi(a, pick(ctx, stream)));
  return RFX_OK;
}
rfx_status rfx_ssgi_trace_launch(rfx_ctx* ctx, void* stream, const rfx_ssgi_params* p, const rfx_plane* depth, const rfx_plane* gbuffer,
                                 const rfx_plane* velocity, const rfx_plane* direct_light, const rfx_plane* accumulated, const rfx_plane* out,
                                 uint32_t row0, uint32_t row1) {
  if (!ctx || !p || !out) return fail(ctx, RFX_ERR_INVALID_ARG, "ssgi_trace: null argument");
  int r0, r1;
  rows(row0, row1, out->height, r0, r1);
  return ssgi_trace(ctx, stream, p, depth, gbuffer, velocity, direct_light, accumulated, out, r0, r1, nullptr);
}

// K2
static rfx_status temporal_reproject(rfx_ctx* ctx, void* stream, const rfx_temporal_params* p, const rfx_plane* input, const rfx_plane* velocity,
                                     const rfx_plane* history0, const rfx_plane* history1, const rfx_plane* out0, const rfx_plane* out1, int r0, int r1,
                                     const TemporalPeer* peer = nullptr) {  // peer: history on the owners + carry (launch_temporal_peer)
  TemporalArgs a{};
  if (p->texture_count != 1 && p->texture_count != 2) return fail(ctx, RFX_ERR_INVALID_ARG, "temporal: texture_count must be 1 or 2");
  a.input_half = input->format == RFX_FMT_RGBA16F;
  if (!pv(input, a.input_half ? RFX_FMT_RGBA16F : RFX_FMT_RGBA32F, a.input)) return fail(ctx, RFX_ERR_BAD_FORMAT, "temporal: input must be RGBA32F or RGBA16F");
  if (p->input_type != RFX_INPUT_DIFFUSE && a.input_half) return fail(ctx, RFX_ERR_BAD_FORMAT, "temporal: packed inputs must be RGBA32F");
  if (!pv(velocity, RFX_FMT_RGBA32F, a.velocity)) return fail(ctx, RFX_ERR_BAD_FORMAT, "temporal: velocity must be RGBA32F");
  a.hist_f32 = history0 && history0->format == RFX_FMT_RGBA32F;  // the FloatType FramebufferTexture history of denoiseMode "full_temporal" / "temporal"
  const int hfmt = a.hist_f32 ? RFX_FMT_RGBA32F : RFX_FMT_RGBA16F;
  if (!pv(history0, hfmt, a.hist0)) return fail(ctx, RFX_ERR_BAD_FORMAT, "temporal: history must be RGBA16F or RGBA32F");
  a.out_half = out0->format == RFX_FMT_RGBA16F;
  if (!ov(out0, a.out_half ? RFX_FMT_RGBA16F : RFX_FMT_RGBA32F, a.out0)) return fail(ctx, RFX_ERR_BAD_FORMAT, "temporal: out must be RGBA32F or RGBA16F");
  if (p->texture_count == 2) {
    if (!pv(history1, hfmt, a.hist1) || !ov(out1, out0->format, a.out1)) return fail(ctx, RFX_ERR_BAD_FORMAT, "temporal: second plane missing / wrong format");
  }
  a.W = (int)out0->width; a.H = (int)out0->height;
  if (a.velocity.w != a.W || a.velocity.h != a.H || a.hist0.w != a.W || a.hist0.h != a.H || a.input.w > a.W || a.input.h > a.H)
    return fail(ctx, RFX_ERR_SIZE_MISMATCH, "temporal: plane sizes differ (only the input may be smaller: resolutionScale < 1)");
  a.in_scaled = a.input.w != a.W || a.input.h != a.H;
  if (a.in_scaled && a.input_half) return fail(ctx, RFX_ERR_UNSUPPORTED, "temporal: a scaled input is the RGBA32F SSGI target");
  a.row0 = r0; a.row1 = r1;
  temporal_uniforms(ctx, p, a);
  if (peer) LAUNCHED(launch_temporal_peer(a, *peer, pick(ctx, stream)));
  else LAUNCHED(launch_temporal(a, pick(ctx, stream)));
  return RFX_OK;
}
rfx_status rfx_temporal_reproject_launch(rfx_ctx* ctx, void* stream, const rfx_temporal_params* p, const rfx_plane* input, const rfx_plane* velocity,
                                         const rfx_plane* history0, const rfx_plane* history1, const rfx_plane* out0, const rfx_plane* out1,
                                         uint32_t row0, uint32_t row1) {
  if (!ctx || !p || !input || !out0) return fail(ctx, RFX_ERR_INVALID_ARG, "temporal: null argument");
  int r0, r1;
  rows(row0, row1, out0->height, r0, r1);
  return temporal_reproject(ctx, stream, p, input, velocity, history0, history1, out0, out1, r0, r1);
}

// K3.  decoded: the context's G-buffer scratch already holds this frame's decode (the chain decodes once per frame)
static rfx_status poisson_denoise(rfx_ctx* ctx, void* stream, const rfx_poisson_params* p, const rfx_plane* depth, const rfx_plane* gb, const rfx_plane* in0,
                                  const rfx_plane* in1, const rfx_plane* out0, const rfx_plane* out1, int r0, int r1, bool decoded,
                                  const PeerCarry* carry = nullptr) {
  if (p->texture_count != 1 && p->texture_count != 2) return fail(ctx, RFX_ERR_INVALID_ARG, "poisson: texture_count must be 1 or 2");
  PoissonArgs a{};
  if (!pv(depth, RFX_FMT_R32F, a.depth) || !pv(gb, RFX_FMT_RGBA32F, a.gb)) return fail(ctx, RFX_ERR_BAD_FORMAT, "poisson: depth R32F + gbuffer/normal RGBA32F required");
  a.in_half = in0->format == RFX_FMT_RGBA16F;
  if (!pv(in0, a.in_half ? RFX_FMT_RGBA16F : RFX_FMT_RGBA32F, a.in0)) return fail(ctx, RFX_ERR_BAD_FORMAT, "poisson: in0 must be RGBA32F or RGBA16F");
  if (!ov(out0, RFX_FMT_RGBA16F, a.out0)) return fail(ctx, RFX_ERR_BAD_FORMAT, "poisson: out must be RGBA16F");
  if (p->texture_count == 2) {
    if (!pv(in1, in0->format, a.in1) || !ov(out1, RFX_FMT_RGBA16F, a.out1)) return fail(ctx, RFX_ERR_BAD_FORMAT, "poisson: second plane missing / wrong format");
  } else {
    a.in1 = a.in0;
  }
  if (p->input_linear && !a.in_half) return fail(ctx, RFX_ERR_UNSUPPORTED, "poisson: LINEAR inputs must be RGBA16F");
  a.W = (int)out0->width; a.H = (int)out0->height;
  if (a.depth.w != a.W || a.depth.h != a.H || a.gb.w != a.W || a.gb.h != a.H || a.in1.w != a.in0.w || a.in1.h != a.in0.h)
    return fail(ctx, RFX_ERR_SIZE_MISMATCH, "poisson: plane sizes differ");
  // LINEAR inputs are sampled by uv and may have any size (the AO denoiser's first pass reads a reduced-resolution AO target)
  if (!p->input_linear && (a.in0.w != a.W || a.in0.h != a.H)) return fail(ctx, RFX_ERR_SIZE_MISMATCH, "poisson: NEAREST inputs must have the output's size");
  if (out0->ptr == in0->ptr || (out1 && in1 && out1->ptr == in1->ptr)) return fail(ctx, RFX_ERR_INVALID_ARG, "poisson: in-place filtering is not allowed");
  a.row0 = r0; a.row1 = r1;
  a.radius = p->radius; a.phi = p->phi; a.luma_phi = p->luma_phi; a.depth_phi = p->depth_phi; a.normal_phi = p->normal_phi;
  a.roughness_phi = p->roughness_phi; a.specular_phi = p->specular_phi;
  a.texture_count = p->texture_count; a.spec0 = p->is_texture_specular[0]; a.spec1 = p->is_texture_specular[1];
  a.gbuffer_texture = p->gbuffer_texture; a.input_linear = p->input_linear;
  rfx_status st = blue_for(ctx, p->blue_noise_index, a.blue);
  if (st != RFX_OK) return st;
  if (p->blue_noise_index == 0) return fail(ctx, RFX_ERR_UNSUPPORTED, "poisson: blue_noise_index 0 is not used by this pass");
  a.rot_table = ctx->rot_table;
  const bool fast = ctx->fast_math && ((p->input_linear && a.in_half) || (!p->input_linear && !a.in_half));
  if (!fast) {
    LAUNCHED(launch_poisson(a, pick(ctx, stream), carry));
    return RFX_OK;
  }
  // fast variant: decode the G-buffer once into the context scratch (the native chain reuses it across the passes of a frame)
  if (!ctx->nrd || ctx->nrd_w != a.W || ctx->nrd_h != a.H) {
    CU(cudaStreamSynchronize(ctx->stream));
    cudaFree(ctx->nrd);
    ctx->nrd = nullptr;
    ctx->nrd_pitch = ((size_t)a.W * 16 + 255) & ~(size_t)255;
    CU(cudaMalloc(&ctx->nrd, ctx->nrd_pitch * a.H));
    ctx->nrd_w = a.W; ctx->nrd_h = a.H;
    decoded = false;
  }
  if (!decoded)  // (the chain's first pass of a frame has the widest rows of all its passes, so its decode serves the later ones)
    LAUNCHED(launch_gbuffer_decode(a.gb, OutV{(unsigned char*)ctx->nrd, (long long)ctx->nrd_pitch}, a.W, a.H, p->gbuffer_texture ? 1 : 0, a.row0, a.row1,
                                   (int)std::ceil(p->radius * std::max(1.0f, (float)a.H / (float)a.W)) + 1, pick(ctx, stream)));
  a.nrd = PV{(const unsigned char*)ctx->nrd, a.W, a.H, (long long)ctx->nrd_pitch};
  {
    const float SQ = 1.41421356237f;
    const float px[8] = {-1.0f, 0.0f, 1.0f, 0.0f, -0.25f * SQ, 0.25f * SQ, 0.25f * SQ, -0.25f * SQ};
    const float py[8] = {0.0f, -1.0f, 0.0f, 1.0f, -0.25f * SQ, -0.25f * SQ, 0.25f * SQ, 0.25f * SQ};
    for (int i = 0; i < 8; i++) { a.tap_ox[i] = px[i] / (float)a.W; a.tap_oy[i] = py[i] / (float)a.H; }  // offset / resolution
  }
  LAUNCHED(launch_poisson_fast(a, pick(ctx, stream), carry));
  return RFX_OK;
}
rfx_status rfx_poisson_denoise_launch(rfx_ctx* ctx, void* stream, const rfx_poisson_params* p, const rfx_plane* depth, const rfx_plane* gb,
                                      const rfx_plane* in0, const rfx_plane* in1, const rfx_plane* out0, const rfx_plane* out1, uint32_t row0,
                                      uint32_t row1) {
  if (!ctx || !p || !in0 || !out0) return fail(ctx, RFX_ERR_INVALID_ARG, "poisson: null argument");
  int r0, r1;
  rows(row0, row1, out0->height, r0, r1);
  return poisson_denoise(ctx, stream, p, depth, gb, in0, in1, out0, out1, r0, r1, false);
}

// K4
static rfx_status gi_compose(rfx_ctx* ctx, void* stream, const rfx_compose_params* p, const rfx_plane* depth, const rfx_plane* gb, const rfx_plane* dgi,
                             const rfx_plane* sgi, const rfx_plane* scene, const rfx_plane* out, int r0, int r1, const PeerPV* carry = nullptr) {
  ComposeArgs a{};
  if (!pv(depth, RFX_FMT_R32F, a.depth) || !pv(gb, RFX_FMT_RGBA32F, a.gb) || !ov(out, RFX_FMT_RGBA32F, a.out))
    return fail(ctx, RFX_ERR_BAD_FORMAT, "gi_compose: depth R32F, gbuffer RGBA32F, out RGBA32F required");
  if (p->input_type != RFX_INPUT_DIFFUSE_SPECULAR && p->input_type != RFX_INPUT_DIFFUSE && p->input_type != RFX_INPUT_SPECULAR)
    return fail(ctx, RFX_ERR_INVALID_ARG, "gi_compose: bad input_type");
  // DenoiserComposePass.js:23-33: diffuseSpecular binds both GI textures, diffuse only the first, specular only the second
  const bool need_d = p->input_type != RFX_INPUT_SPECULAR, need_s = p->input_type != RFX_INPUT_DIFFUSE;
  const rfx_plane* first = need_d ? dgi : sgi;
  a.gi_f32 = first && first->format == RFX_FMT_RGBA32F;  // denoiseMode "full_temporal": the temporal pass's FloatType NEAREST targets
  const int gfmt = a.gi_f32 ? RFX_FMT_RGBA32F : RFX_FMT_RGBA16F;
  if (need_d && !pv(dgi, gfmt, a.diffuse)) return fail(ctx, RFX_ERR_BAD_FORMAT, "gi_compose: diffuse GI must be RGBA16F (or both RGBA32F)");
  if (need_s && !pv(sgi, gfmt, a.specular)) return fail(ctx, RFX_ERR_BAD_FORMAT, "gi_compose: specular GI must be RGBA16F (or both RGBA32F)");
  if (p->input_type == RFX_INPUT_SPECULAR && scene && !pv(scene, RFX_FMT_RGBA16F, a.scene)) return fail(ctx, RFX_ERR_BAD_FORMAT, "gi_compose: scene must be RGBA16F");
  a.W = (int)out->width; a.H = (int)out->height;
  if (a.depth.w != a.W || a.depth.h != a.H || a.gb.w != a.W || a.gb.h != a.H || (a.diffuse.p && (a.diffuse.w != a.W || a.diffuse.h != a.H)) ||
      (a.specular.p && (a.specular.w != a.W || a.specular.h != a.H)) || (a.scene.p && (a.scene.w != a.W || a.scene.h != a.H)))
    return fail(ctx, RFX_ERR_SIZE_MISMATCH, "gi_compose: plane sizes differ");
  a.row0 = r0; a.row1 = r1;
  cam_to_dev(p->cam, a.cam);
  a.input_type = p->input_type;
  a.fast = ctx->fast_math;
  LAUNCHED(launch_gi_compose(a, pick(ctx, stream), carry));
  return RFX_OK;
}
rfx_status rfx_gi_compose_launch(rfx_ctx* ctx, void* stream, const rfx_compose_params* p, const rfx_plane* depth, const rfx_plane* gb,
                                 const rfx_plane* dgi, const rfx_plane* sgi, const rfx_plane* scene, const rfx_plane* out, uint32_t row0, uint32_t row1) {
  if (!ctx || !p || !out) return fail(ctx, RFX_ERR_INVALID_ARG, "gi_compose: null argument");
  int r0, r1;
  rows(row0, row1, out->height, r0, r1);
  return gi_compose(ctx, stream, p, depth, gb, dgi, sgi, scene, out, r0, r1);
}

// K5's uniforms from the C ABI's parameters (fog, camera, isDebug)
static void compose_uniforms(const rfx_ssgi_compose_params& p, SsgiComposeArgs& a) {
  a.use_fog = p.use_fog; a.fog_exp2 = p.fog_exp2; a.perspective = p.perspective; a.is_debug = p.is_debug;
  memcpy(a.fog_color, p.fog_color, 12);
  a.fog_near = p.fog_near; a.fog_far = p.fog_far; a.fog_density = p.fog_density; a.camera_near = p.camera_near; a.camera_far = p.camera_far;
}
// K5 with isDebug for a view ssgi_compose_kernel does not fetch (another format or size): depth and scene are not read
static rfx_status ssgi_compose_debug(rfx_ctx* ctx, void* stream, const rfx_plane* gi, const rfx_plane* out, uint32_t row0, uint32_t row1) {
  SsgiComposeDebugArgs a{};
  a.gi_fmt = (int)gi->format;
  if ((a.gi_fmt != RFX_FMT_R32F && a.gi_fmt != RFX_FMT_RGBA16F && a.gi_fmt != RFX_FMT_RGBA32F) || !pv(gi, a.gi_fmt, a.gi) || !ov(out, RFX_FMT_RGBA16F, a.out))
    return fail(ctx, RFX_ERR_BAD_FORMAT, "ssgi_compose: a debug view must be R32F, RGBA16F or RGBA32F and out RGBA16F");
  a.W = (int)out->width; a.H = (int)out->height;
  rows(row0, row1, out->height, a.row0, a.row1);
  LAUNCHED(launch_ssgi_compose_debug(a, pick(ctx, stream)));
  return RFX_OK;
}
rfx_status rfx_ssgi_compose_launch(rfx_ctx* ctx, void* stream, const rfx_ssgi_compose_params* p, const rfx_plane* depth, const rfx_plane* gi, const rfx_plane* scene,
                                   const rfx_plane* out, uint32_t row0, uint32_t row1) {
  if (!ctx || !out) return fail(ctx, RFX_ERR_INVALID_ARG, "ssgi_compose: null argument");
  if (p && p->is_debug && gi && (!depth || !scene || !(gi->format == RFX_FMT_RGBA32F && gi->width == out->width && gi->height == out->height)))
    return ssgi_compose_debug(ctx, stream, gi, out, row0, row1);
  SsgiComposeArgs a{};
  if (!pv(depth, RFX_FMT_R32F, a.depth) || !pv(gi, RFX_FMT_RGBA32F, a.gi) || !pv(scene, RFX_FMT_RGBA16F, a.scene) || !ov(out, RFX_FMT_RGBA16F, a.out))
    return fail(ctx, RFX_ERR_BAD_FORMAT, "ssgi_compose: depth R32F, gi RGBA32F, scene/out RGBA16F required");
  a.W = (int)out->width; a.H = (int)out->height;
  if (a.depth.w != a.W || a.depth.h != a.H || a.gi.w != a.W || a.scene.w != a.W) return fail(ctx, RFX_ERR_SIZE_MISMATCH, "ssgi_compose: plane sizes differ");
  rows(row0, row1, out->height, a.row0, a.row1);
  if (p) compose_uniforms(*p, a);
  LAUNCHED(launch_ssgi_compose(a, pick(ctx, stream)));
  return RFX_OK;
}

}  // extern "C"

// K6 over output rows [r0, r1); carry: as poisson_denoise's, `out` (the AO chain in a row-sharded group)
static rfx_status hbao(rfx_ctx* ctx, void* stream, const rfx_hbao_params* p, const rfx_plane* depth, const rfx_plane* normal, const rfx_plane* out,
                       uint32_t row0, uint32_t row1, const PeerPV* carry = nullptr) {
  HbaoArgs a{};
  if (!pv(depth, RFX_FMT_R32F, a.depth) || !ov(out, RFX_FMT_RGBA16F, a.out)) return fail(ctx, RFX_ERR_BAD_FORMAT, "hbao: depth R32F, out RGBA16F required");
  if (normal && !pv(normal, RFX_FMT_RGBA8, a.normal)) return fail(ctx, RFX_ERR_BAD_FORMAT, "hbao: the normal plane must be RGBA8");
  a.W = (int)out->width; a.H = (int)out->height;
  if (a.W > a.depth.w || a.H > a.depth.h)
    return fail(ctx, RFX_ERR_SIZE_MISMATCH, "hbao: the output may be smaller than the depth plane (resolutionScale <= 1), not larger");
  if (p->spp < 0) return fail(ctx, RFX_ERR_INVALID_ARG, "hbao: spp < 0");
  const bool res_default = p->resolution[0] == 0.0f && p->resolution[1] == 0.0f;
  if (!res_default && !(p->resolution[0] > 0.0f && p->resolution[1] > 0.0f)) return fail(ctx, RFX_ERR_INVALID_ARG, "hbao: resolution must be positive or {0, 0}");
  a.res_x = res_default ? (float)a.W : p->resolution[0];
  a.res_y = res_default ? (float)a.H : p->resolution[1];
  a.general = a.W != a.depth.w || a.H != a.depth.h || a.normal.p || a.res_x != (float)a.W || a.res_y != (float)a.H;
  rows(row0, row1, out->height, a.row0, a.row1);
  memcpy(a.projection_view.m, p->projection_view, 64);
  memcpy(a.projection_inverse.m, p->projection_inverse, 64);
  memcpy(a.camera_matrix_world.m, p->camera_matrix_world, 64);
  memcpy(a.view_matrix.m, p->view_matrix, 64);
  a.ao_distance = p->ao_distance; a.distance_power = p->distance_power; a.bias = p->bias; a.thickness = p->thickness; a.spp = p->spp;
  rfx_status st = blue_for(ctx, p->blue_noise_index, a.blue);
  if (st != RFX_OK) return st;
  if (p->blue_noise_index == 0) return fail(ctx, RFX_ERR_UNSUPPORTED, "hbao: blue_noise_index 0 is not used by this pass");
  a.rot_table = ctx->rot_table;
  LAUNCHED(launch_hbao(a, pick(ctx, stream), carry));
  return RFX_OK;
}

extern "C" {

rfx_status rfx_hbao_launch_ex(rfx_ctx* ctx, void* stream, const rfx_hbao_params* p, const rfx_plane* depth, const rfx_plane* normal, const rfx_plane* out,
                              uint32_t row0, uint32_t row1) {
  if (!ctx || !p || !out) return fail(ctx, RFX_ERR_INVALID_ARG, "hbao: null argument");
  return hbao(ctx, stream, p, depth, normal, out, row0, row1);
}

rfx_status rfx_hbao_launch(rfx_ctx* ctx, void* stream, const rfx_hbao_params* p, const rfx_plane* depth, const rfx_plane* out, uint32_t row0, uint32_t row1) {
  if (!ctx || !p) return fail(ctx, RFX_ERR_INVALID_ARG, "hbao: null argument");
  rfx_hbao_params q{};  // the fields before view_matrix only: callers built against the shorter struct pass no more than those
  memcpy(&q, p, offsetof(rfx_hbao_params, view_matrix));
  return rfx_hbao_launch_ex(ctx, stream, &q, depth, nullptr, out, row0, row1);
}

rfx_status rfx_hbao_horizon_directions(int32_t directions, float* out) {
  if (directions < 1 || directions > 32 || !out) return RFX_ERR_INVALID_ARG;
  for (int d = 0; d < directions; d++)
    for (int b = 0; b < 256; b++) {
      const double theta = 2.0 * 3.14159265358979323846 * ((double)d + (double)b / 255.0) / (double)directions;
      out[2 * (d * 256 + b)] = (float)std::cos(theta);
      out[2 * (d * 256 + b) + 1] = (float)std::sin(theta);
    }
  return RFX_OK;
}

}  // extern "C"

// K6h: horizon-march AO (an extension; no reference draw exists, SURVEY.md D1) over output rows [r0, r1) (0, 0: all); carry: as hbao's
static rfx_status hbao_horizon(rfx_ctx* ctx, void* stream, const rfx_hbao_horizon_params* p, const rfx_plane* depth, const rfx_plane* out,
                               const rfx_plane* normal, uint32_t row0, uint32_t row1, const PeerPV* carry = nullptr) {
  HbaoHorizonArgs a{};
  if (!pv(depth, RFX_FMT_R32F, a.depth) || !ov(out, RFX_FMT_RGBA16F, a.out))
    return fail(ctx, RFX_ERR_BAD_FORMAT, "hbao_horizon: depth R32F, out RGBA16F required");
  if (normal && !pv(normal, RFX_FMT_RGBA8, a.normal)) return fail(ctx, RFX_ERR_BAD_FORMAT, "hbao_horizon: the normal plane must be RGBA8");
  a.W = (int)out->width; a.H = (int)out->height;
  if (a.W > a.depth.w || a.H > a.depth.h)
    return fail(ctx, RFX_ERR_SIZE_MISMATCH, "hbao_horizon: the output may be smaller than the depth plane, not larger");
  if (a.normal.p && (a.normal.w != a.depth.w || a.normal.h != a.depth.h))
    return fail(ctx, RFX_ERR_SIZE_MISMATCH, "hbao_horizon: the normal plane must have the depth plane's size");
  if (p->directions < 1 || p->directions > 32) return fail(ctx, RFX_ERR_INVALID_ARG, "hbao_horizon: directions must lie in 1..32");
  if (p->steps < 1 || p->steps > 64) return fail(ctx, RFX_ERR_INVALID_ARG, "hbao_horizon: steps must lie in 1..64");
  if (!(p->distance > 0.0f) || !std::isfinite(p->distance)) return fail(ctx, RFX_ERR_INVALID_ARG, "hbao_horizon: distance must be > 0");
  if (!(p->max_radius_pixels >= 1.0f)) return fail(ctx, RFX_ERR_INVALID_ARG, "hbao_horizon: max_radius_pixels must be >= 1");
  if (!(p->intensity >= 0.0f) || !std::isfinite(p->intensity)) return fail(ctx, RFX_ERR_INVALID_ARG, "hbao_horizon: intensity must be >= 0");
  if (!(p->angle_bias >= 0.0f && p->angle_bias < 1.0f)) return fail(ctx, RFX_ERR_INVALID_ARG, "hbao_horizon: angle_bias must lie in [0, 1)");
  const bool res_default = p->resolution[0] == 0.0f && p->resolution[1] == 0.0f;
  if (!res_default && !(p->resolution[0] > 0.0f && p->resolution[1] > 0.0f))
    return fail(ctx, RFX_ERR_INVALID_ARG, "hbao_horizon: resolution must be positive or {0, 0}");
  a.res_x = res_default ? (float)a.W : p->resolution[0];
  a.res_y = res_default ? (float)a.H : p->resolution[1];
  memcpy(a.projection.m, p->projection, 64);
  memcpy(a.projection_inverse.m, p->projection_inverse, 64);
  memcpy(a.camera_matrix_world.m, p->camera_matrix_world, 64);
  memcpy(a.view_matrix.m, p->view_matrix, 64);
  a.distance = p->distance;
  a.dist2 = p->distance * p->distance;
  a.inv_dist2 = 1.0f / a.dist2;
  a.angle_bias = p->angle_bias; a.intensity = p->intensity; a.max_radius_pixels = p->max_radius_pixels;
  a.directions = p->directions; a.steps = p->steps;
  rows(row0, row1, out->height, a.row0, a.row1);
  a.fast = ctx->fast_math;
  if (p->blue_noise_index == 0) return fail(ctx, RFX_ERR_UNSUPPORTED, "hbao_horizon: blue_noise_index 0 is not used by this pass");
  rfx_status st = blue_for(ctx, p->blue_noise_index, a.blue);
  if (st != RFX_OK) return st;
  float2*& dirs = ctx->horizon_dirs[p->directions];
  if (!dirs) {  // a fresh allocation no launch has read yet, filled synchronously; kept only once filled
    std::vector<float> host((size_t)p->directions * 512);
    rfx_hbao_horizon_directions(p->directions, host.data());
    float2* t = nullptr;
    CU(cudaMalloc(&t, host.size() * sizeof(float)));
    const cudaError_t e = cudaMemcpy(t, host.data(), host.size() * sizeof(float), cudaMemcpyHostToDevice);
    if (e != cudaSuccess) {
      cudaFree(t);
      return fail(ctx, RFX_ERR_CUDA, "hbao_horizon: direction table upload failed: %s", cudaGetErrorString(e));
    }
    dirs = t;
  }
  a.dirs = dirs;
  LAUNCHED(launch_hbao_horizon(a, pick(ctx, stream), carry));
  return RFX_OK;
}

// K7 over output rows [r0, r1) (0, 0: all)
static rfx_status ao_compose(rfx_ctx* ctx, void* stream, const rfx_ao_compose_params* p, const rfx_plane* depth, const rfx_plane* ao,
                             const rfx_plane* input, const rfx_plane* out, uint32_t row0, uint32_t row1) {
  AoComposeArgs a{};
  if (!pv(depth, RFX_FMT_R32F, a.depth) || !pv(ao, RFX_FMT_RGBA16F, a.ao) || !pv(input, RFX_FMT_RGBA16F, a.input) || !ov(out, RFX_FMT_RGBA16F, a.out))
    return fail(ctx, RFX_ERR_BAD_FORMAT, "ao_compose: depth R32F, ao/input/out RGBA16F required");
  a.W = (int)out->width; a.H = (int)out->height;
  // `ao` is sampled LINEAR by uv: any size (a reduced-resolution AO target when the denoiser runs no iteration, AOEffect.js:148-154)
  if (a.depth.w != a.W || a.depth.h != a.H || a.input.w != a.W || a.input.h != a.H) return fail(ctx, RFX_ERR_SIZE_MISMATCH, "ao_compose: depth / input / out sizes differ");
  rows(row0, row1, out->height, a.row0, a.row1);
  a.power = p->power;
  memcpy(a.color, p->color, 12);
  LAUNCHED(launch_ao_compose(a, pick(ctx, stream)));
  return RFX_OK;
}

extern "C" {

rfx_status rfx_hbao_horizon_launch(rfx_ctx* ctx, void* stream, const rfx_hbao_horizon_params* p, const rfx_plane* depth, const rfx_plane* out,
                                   const rfx_plane* normal) {
  if (!ctx || !p || !out) return fail(ctx, RFX_ERR_INVALID_ARG, "hbao_horizon: null argument");
  return hbao_horizon(ctx, stream, p, depth, out, normal, 0, 0);
}

rfx_status rfx_ao_compose_launch(rfx_ctx* ctx, void* stream, const rfx_ao_compose_params* p, const rfx_plane* depth, const rfx_plane* ao,
                                 const rfx_plane* input, const rfx_plane* out, uint32_t row0, uint32_t row1) {
  if (!ctx || !p || !out) return fail(ctx, RFX_ERR_INVALID_ARG, "ao_compose: null argument");
  return ao_compose(ctx, stream, p, depth, ao, input, out, row0, row1);
}

}  // extern "C"

// K8's arguments (rfx_motion_blur_launch and the merged TRAA + motion-blur pass): the planes, the rows and the uniforms
static rfx_status motion_blur_args(rfx_ctx* ctx, const char* who, const rfx_motion_blur_params* p, const rfx_plane* velocity, const rfx_plane* input,
                                   const rfx_plane* out, uint32_t row0, uint32_t row1, MotionBlurArgs& a) {
  if (!pv(velocity, RFX_FMT_RGBA32F, a.velocity) || !pv(input, RFX_FMT_RGBA16F, a.input) || !ov(out, RFX_FMT_RGBA16F, a.out))
    return fail(ctx, RFX_ERR_BAD_FORMAT, "%s: velocity RGBA32F, input/out RGBA16F required", who);
  a.W = (int)out->width; a.H = (int)out->height;
  if (a.velocity.w != a.W || a.velocity.h != a.H || a.input.w != a.W || a.input.h != a.H) return fail(ctx, RFX_ERR_SIZE_MISMATCH, "%s: plane sizes differ", who);
  if (input->ptr == out->ptr) return fail(ctx, RFX_ERR_INVALID_ARG, "%s: in-place is not allowed", who);
  if (p->samples < 1) return fail(ctx, RFX_ERR_INVALID_ARG, "%s: samples < 1", who);
  rows(row0, row1, out->height, a.row0, a.row1);
  a.intensity = p->intensity; a.jitter = p->jitter; a.delta_time = p->delta_time; a.res_x = p->resolution[0]; a.res_y = p->resolution[1];
  a.samples = p->samples;
  return blue_for(ctx, p->frame, a.blue);
}

// The merged TRAA + motion-blur pass over output rows [row0, row1) (0, 0: all).  peer: the input buffer's rows live on their owners
// (a row-sharded group of n > 1); its local plane is `input`.
static rfx_status traa_motion_blur(rfx_ctx* ctx, void* stream, const rfx_motion_blur_params* p, const rfx_plane* velocity, const rfx_plane* acc,
                                   const rfx_plane* input, const rfx_plane* out, uint32_t row0, uint32_t row1, const PeerPV* peer) {
  TraaMotionBlurArgs a{};
  rfx_status st = motion_blur_args(ctx, "traa_motion_blur", p, velocity, input, out, row0, row1, a.mb);
  if (st != RFX_OK) return st;
  if (!pv(acc, RFX_FMT_RGBA16F, a.acc)) return fail(ctx, RFX_ERR_BAD_FORMAT, "traa_motion_blur: accumulated RGBA16F required");
  if (a.acc.w != a.mb.W || a.acc.h != a.mb.H) return fail(ctx, RFX_ERR_SIZE_MISMATCH, "traa_motion_blur: plane sizes differ");
  if (acc->ptr == out->ptr) return fail(ctx, RFX_ERR_INVALID_ARG, "traa_motion_blur: out may not alias accumulated");
  LAUNCHED(launch_traa_motion_blur(a, pick(ctx, stream), peer));
  return RFX_OK;
}

extern "C" {

rfx_status rfx_motion_blur_launch(rfx_ctx* ctx, void* stream, const rfx_motion_blur_params* p, const rfx_plane* velocity, const rfx_plane* input,
                                  const rfx_plane* out, uint32_t row0, uint32_t row1) {
  if (!ctx || !p || !out) return fail(ctx, RFX_ERR_INVALID_ARG, "motion_blur: null argument");
  MotionBlurArgs a{};
  rfx_status st = motion_blur_args(ctx, "motion_blur", p, velocity, input, out, row0, row1, a);
  if (st != RFX_OK) return st;
  LAUNCHED(launch_motion_blur(a, pick(ctx, stream)));
  return RFX_OK;
}

rfx_status rfx_traa_motion_blur_launch(rfx_ctx* ctx, void* stream, const rfx_motion_blur_params* p, const rfx_plane* velocity, const rfx_plane* acc,
                                       const rfx_plane* input, const rfx_plane* out, uint32_t row0, uint32_t row1) {
  if (!ctx || !p || !acc || !out) return fail(ctx, RFX_ERR_INVALID_ARG, "traa_motion_blur: null argument");
  return traa_motion_blur(ctx, stream, p, velocity, acc, input, out, row0, row1, nullptr);
}

rfx_status rfx_gbuffer_debug_launch(rfx_ctx* ctx, void* stream, int32_t mode, const rfx_plane* gbuffer, const rfx_plane* out, uint32_t row0, uint32_t row1) {
  if (!ctx || !out) return fail(ctx, RFX_ERR_INVALID_ARG, "gbuffer_debug: null argument");
  GbufferDebugArgs a{};
  if (!pv(gbuffer, RFX_FMT_RGBA32F, a.gb) || !ov(out, RFX_FMT_RGBA32F, a.out)) return fail(ctx, RFX_ERR_BAD_FORMAT, "gbuffer_debug: RGBA32F planes required");
  a.W = (int)out->width; a.H = (int)out->height;
  if (a.gb.w != a.W || a.gb.h != a.H) return fail(ctx, RFX_ERR_SIZE_MISMATCH, "gbuffer_debug: plane sizes differ");
  a.mode = mode >= 0 && mode <= 5 ? mode : 5;  // the shader's `else` branch: emissive
  rows(row0, row1, out->height, a.row0, a.row1);
  LAUNCHED(launch_gbuffer_debug(a, pick(ctx, stream)));
  return RFX_OK;
}

rfx_status rfx_traa_compose_launch(rfx_ctx* ctx, void* stream, const rfx_plane* acc, const rfx_plane* out, uint32_t row0, uint32_t row1) {
  if (!ctx || !out) return fail(ctx, RFX_ERR_INVALID_ARG, "traa_compose: null argument");
  TraaComposeArgs a{};
  if (!pv(acc, RFX_FMT_RGBA16F, a.acc) || !ov(out, RFX_FMT_RGBA16F, a.out)) return fail(ctx, RFX_ERR_BAD_FORMAT, "traa_compose: RGBA16F planes required");
  a.W = (int)out->width; a.H = (int)out->height;
  if (a.acc.w != a.W || a.acc.h != a.H) return fail(ctx, RFX_ERR_SIZE_MISMATCH, "traa_compose: plane sizes differ");
  rows(row0, row1, out->height, a.row0, a.row1);
  LAUNCHED(launch_traa_compose(a, pick(ctx, stream)));
  return RFX_OK;
}

rfx_status rfx_effects_launch(rfx_ctx* ctx, void* stream, const rfx_effects_params* p, const rfx_plane* input, const rfx_plane* depth, const rfx_plane* velocity,
                              const rfx_plane* out, uint32_t row0, uint32_t row1) {
  if (!ctx || !p || !input || !out) return fail(ctx, RFX_ERR_INVALID_ARG, "effects: null argument");
  if (p->n_effects < 1 || p->n_effects > 4) return fail(ctx, RFX_ERR_INVALID_ARG, "effects: n_effects must be 1..4");
  EffectsArgs a{};
  if (!pv(input, RFX_FMT_RGBA16F, a.input) || !ov(out, RFX_FMT_RGBA16F, a.out)) return fail(ctx, RFX_ERR_BAD_FORMAT, "effects: input / out must be RGBA16F");
  if (input->ptr == out->ptr) return fail(ctx, RFX_ERR_INVALID_ARG, "effects: out may not alias input (neighbour taps)");
  a.W = (int)out->width; a.H = (int)out->height;
  if (a.input.w != a.W || a.input.h != a.H) return fail(ctx, RFX_ERR_SIZE_MISMATCH, "effects: plane sizes differ");
  for (int i = 0; i < p->n_effects; i++) {
    const int e = p->effects[i];
    a.effects[i] = e;
    if (e < RFX_FX_SHARPNESS || e > RFX_FX_SPARKLE) return fail(ctx, RFX_ERR_INVALID_ARG, "effects: unknown effect id %d", e);
    if (e == RFX_FX_GRADUAL_BACKGROUND && (!pv(depth, RFX_FMT_R32F, a.depth) || a.depth.w != a.W || a.depth.h != a.H))
      return fail(ctx, RFX_ERR_BAD_FORMAT, "effects: GradualBackground needs an R32F depth plane of the output size");
    if (e == RFX_FX_SPARKLE && (!pv(velocity, RFX_FMT_RGBA32F, a.velocity) || a.velocity.w != a.W || a.velocity.h != a.H))
      return fail(ctx, RFX_ERR_BAD_FORMAT, "effects: Sparkle needs an RGBA32F velocity plane of the output size");
  }
  a.n_effects = p->n_effects;
  cam_to_dev(p->cam, a.cam);
  a.texel_x = (float)(1.0 / a.W); a.texel_y = (float)(1.0 / a.H);
  a.sharpness = p->sharpness; a.alphax = p->alphax; a.alphay = p->alphay; a.aberration = p->aberration;
  memcpy(a.bg, p->background_color, 12);
  a.max_distance = p->max_distance; a.spread = p->spread; a.intensity = p->intensity; a.sparkle_perspective = p->sparkle_perspective;
  rows(row0, row1, out->height, a.row0, a.row1);
  LAUNCHED(launch_effects(a, pick(ctx, stream)));
  return RFX_OK;
}

rfx_status rfx_taa_launch(rfx_ctx* ctx, void* stream, const rfx_taa_params* p, const rfx_plane* input, const rfx_plane* history, const rfx_plane* out,
                          uint32_t row0, uint32_t row1) {
  if (!ctx || !p || !input || !out) return fail(ctx, RFX_ERR_INVALID_ARG, "taa: null argument");
  TaaArgs a{};
  if (!pv(input, RFX_FMT_RGBA16F, a.input) || !ov(out, RFX_FMT_RGBA8, a.out)) return fail(ctx, RFX_ERR_BAD_FORMAT, "taa: input RGBA16F, out RGBA8");
  a.W = (int)out->width; a.H = (int)out->height;
  if (a.input.w != a.W || a.input.h != a.H) return fail(ctx, RFX_ERR_SIZE_MISMATCH, "taa: plane sizes differ");
  if (p->camera_not_moved_frames != 0.0f && (!pv(history, RFX_FMT_RGBA8, a.history) || a.history.w != a.W || a.history.h != a.H))
    return fail(ctx, RFX_ERR_BAD_FORMAT, "taa: an RGBA8 history plane of the output size is needed once the camera stands still");
  a.camera_not_moved_frames = p->camera_not_moved_frames; a.srgb_output = p->srgb_output;
  rows(row0, row1, out->height, a.row0, a.row1);
  LAUNCHED(launch_taa(a, pick(ctx, stream)));
  return RFX_OK;
}

rfx_status rfx_gbuffer_ingest_launch(rfx_ctx* ctx, void* stream, const rfx_ingest_params* p, const rfx_plane* albedo, const rfx_plane* normal,
                                     const rfx_plane* material, const rfx_plane* emissive, const rfx_plane* motion, const rfx_plane* depth,
                                     const rfx_plane* out_gbuffer, const rfx_plane* out_velocity, uint32_t row0, uint32_t row1) {
  if (!ctx || !p || !albedo || !normal || !material || !depth || (!out_gbuffer && !out_velocity)) return fail(ctx, RFX_ERR_INVALID_ARG, "gbuffer_ingest: null argument");
  IngestArgs a{};
  auto one_of = [](const rfx_plane* pl, int f0, int f1, PV& out, int& is_second) {
    if (pl && pl->format == f1) { is_second = 1; return pv(pl, f1, out); }
    is_second = 0;
    return pv(pl, f0, out);
  };
  if (!one_of(albedo, RFX_FMT_RGBA8, RFX_FMT_RGBA16F, a.albedo, a.albedo_half) || !one_of(material, RFX_FMT_RGBA8, RFX_FMT_RGBA16F, a.material, a.material_half) ||
      !one_of(normal, RFX_FMT_RGBA16F, RFX_FMT_RGBA32F, a.normal, a.normal_f32) || !pv(depth, RFX_FMT_R32F, a.depth) ||
      (emissive && !pv(emissive, RFX_FMT_RGBA16F, a.emissive)) || (motion && !one_of(motion, RFX_FMT_RGBA16F, RFX_FMT_RGBA32F, a.motion, a.motion_f32)) ||
      (out_gbuffer && !ov(out_gbuffer, RFX_FMT_RGBA32F, a.out_gb)) || (out_velocity && !ov(out_velocity, RFX_FMT_RGBA32F, a.out_vel)))
    return fail(ctx, RFX_ERR_BAD_FORMAT, "gbuffer_ingest: albedo / material RGBA8|RGBA16F, normal / motion RGBA16F|RGBA32F, emissive RGBA16F, depth R32F, outputs RGBA32F");
  a.W = (int)depth->width; a.H = (int)depth->height;
  for (const rfx_plane* pl : {albedo, normal, material, emissive, motion, out_gbuffer, out_velocity})
    if (pl && ((int)pl->width != a.W || (int)pl->height != a.H)) return fail(ctx, RFX_ERR_SIZE_MISMATCH, "gbuffer_ingest: plane sizes differ");
  a.normalize_normals = p->normalize_normals;
  a.motion_sx = p->motion_scale[0]; a.motion_sy = p->motion_scale[1];
  rows(row0, row1, depth->height, a.row0, a.row1);
  LAUNCHED(launch_gbuffer_ingest(a, pick(ctx, stream)));
  return RFX_OK;
}

}  // extern "C"

// ==========================================================================================
// native SSGI chain
// ==========================================================================================
struct IPlane {  // chain-internal plane (formats of k_chain.cu): raw pitched allocation
  void* p = nullptr;
  size_t pitch = 0;
};
// A plane the chain may keep from one frame to the next (hist_planes lists the ones its configuration keeps).  Such a plane is
// double-buffered by a frame parity so that, in a row-sharded group, no rank overwrites rows a peer may still be reading; view[b]
// reads buffer b, each row on the rank that owns it.  Alone, view[b] is the n = 1 view of the local buffer.
struct HistPlane {
  rfx_plane buf[2]{};
  PeerPV view[2]{};
};
// The TRAA frame tail a chain can end with (rfx_*_chain_enable_traa): TRAAEffect's temporal pass over `mid` into the accumulated plane,
// then K9.  `mid` is the composer buffer before the TRAA EffectPass: the SSGI chain's K5 output, the AO chain's K7 output.  With the
// motion-blur stage on (rfx_*_chain_set_motion_blur), the merged TRAA + motion-blur pass replaces K9; its taps read all of `mid`.  `mid` is single-buffered (buffer 0) unless a row-sharded group with the stage gave it buffer 1:
// then it goes by tail parity like `acc`, so that a rank's next frame never writes rows a slower peer's merged pass still reads.
struct TraaTail {
  bool on = false;
  rfx_traa_tail_options opt{};
  HistPlane acc;        // accumulated plane by tail parity (buf[prev] is the history)
  HistPlane mid;
  rfx_plane out{};      // K9 output (SSGI; the AO tail writes frame->output)
  bool blur = false;    // the motion-blur stage
  rfx_motion_blur_params blur_p{};  // this frame's MotionBlurEffect uniforms
  // In a row-sharded group of n > 1 with the stage on, a frame has two phases (rfx_*_chain_render_sharded, then _finish): the merged pass
  // reads this frame's `mid` rows on their owners, so it waits for the frame's barrier.  `pending`: phase 1 ran, the merged pass did not.
  bool split = false;
  bool pending = false;
  rfx_plane p2_velocity{}, p2_out{};  // what phase 2 launches on: the frame's velocity plane and output
  int p2_r0 = 0, p2_r1 = 0;           // ... and the rows (the band, or with the cosmetic stage on its input rows)
  // The cosmetic stage (rfx_*_chain_set_effects): one effects launch over the tail's image after the tail's last pass.  `fx_plane` is the
  // SSGI chain's stage output (output 6) and the AO chain's stage input (the tail writes it instead of frame->output).  `fx_job` is this
  // frame's launch, set by the chain before its tail and run by tail_end (in phase 2 of a split frame).
  bool fx = false;
  rfx_effects_params fx_p{};
  rfx_plane fx_plane{};
  struct { rfx_plane in, depth, velocity, out; int r0, r1; } fx_job{};
  uint64_t frames = 0;  // tails rendered; acc.buf[frames & 1] is written next
  float keep = 0.0f;    // keepData of the TRAA pass
  int cur() const { return (int)(frames & 1); }
  int mid_cur() const { return mid.buf[1].ptr ? cur() : 0; }
  rfx_plane& mid_w() { return mid.buf[mid_cur()]; }  // this frame's `mid`
  const rfx_plane& latest() const { return acc.buf[(frames + 1) & 1]; }  // the accumulated plane of the latest frame
  const rfx_plane& mid_latest() const { return mid.buf[mid.buf[1].ptr ? (int)((frames + 1) & 1) : 0]; }  // `mid` of the latest frame
  void advance() { keep = 1.0f; frames++; }  // after a frame's tail: keep the history from now on
};
// What a row-sharded group (rfx_group.inl) needs of a member chain; both chain kinds derive from it.
struct GroupMember {
  rfx_ctx* ctx = nullptr;
  struct rfx_group* group = nullptr;  // row-sharded group the chain is attached to (rfx_group_attach_*)
  // attached to a group of n > 1 (the SSGI fast chain excepted): the peer / carry instantiations and both buffers of every plane the chain
  // keeps are in use.  A frame's kernels read last frame's rows on their owners and carry the texels of discarded pixels from there.
  bool group_peer = false;
  TraaTail tail;
};
// The copy pipeline of a chain's host-buffer path (rfx_*_chain_submit_host): two staging sets, so frame i+1 uploads while frame i
// renders; H2D, kernels and D2H each get their own stream and are ordered by events only.  Frame i uses set i & 1: ev_up[set] fires
// after its upload, ev_rendered[set] after its kernels, ev_dn[set] after its download.  Created at the first submit.
struct HostPipe {
  bool ready = false;
  cudaStream_t s_up = nullptr, s_dn = nullptr;
  cudaEvent_t ev_up[2]{}, ev_rendered[2]{}, ev_dn[2]{};
  uint64_t submitted = 0;  // frames submitted
  int set() const { return (int)(submitted & 1); }
};
static rfx_status host_pipe_init(rfx_ctx* ctx, HostPipe& p) {
  if (p.ready) return RFX_OK;
  CU(cudaStreamCreateWithFlags(&p.s_up, cudaStreamNonBlocking));
  CU(cudaStreamCreateWithFlags(&p.s_dn, cudaStreamNonBlocking));
  for (int i = 0; i < 2; i++) {
    CU(cudaEventCreateWithFlags(&p.ev_up[i], cudaEventDisableTiming));
    CU(cudaEventCreateWithFlags(&p.ev_rendered[i], cudaEventDisableTiming));
    CU(cudaEventCreateWithFlags(&p.ev_dn[i], cudaEventDisableTiming));
  }
  p.ready = true;
  return RFX_OK;
}
static void host_pipe_destroy(HostPipe& p) {  // after the chain's last frame: waits for its copies
  if (p.s_up) cudaStreamSynchronize(p.s_up);
  if (p.s_dn) cudaStreamSynchronize(p.s_dn);
  for (int i = 0; i < 2; i++) for (cudaEvent_t e : {p.ev_up[i], p.ev_rendered[i], p.ev_dn[i]}) if (e) cudaEventDestroy(e);
  if (p.s_up) cudaStreamDestroy(p.s_up);
  if (p.s_dn) cudaStreamDestroy(p.s_dn);
}
// Blocks until at most `max_in_flight` (0 or 1; larger values do not wait) submitted frames are incomplete.  Frames complete in
// submission order: a complete frame's downloads are filled and its host input buffers may be overwritten.
static rfx_status host_pipe_wait(rfx_ctx* ctx, const HostPipe& p, int32_t max_in_flight) {
  if (p.submitted == 0 || !p.ready) return RFX_OK;
  if (max_in_flight == 0) { CU(cudaEventSynchronize(p.ev_dn[(p.submitted - 1) & 1])); }
  else if (max_in_flight == 1 && p.submitted >= 2) { CU(cudaEventSynchronize(p.ev_dn[(p.submitted - 2) & 1])); }
  return RFX_OK;
}
struct rfx_ssgi_chain : GroupMember {
  rfx_ssgi_chain_options opt;
  rfx_plane ssgi_out{};
  // per-pass chain: single-buffered alone (buffer 0, rendered in place); buffer 1 of each plane the chain keeps is added by a group of
  // n > 1 (group_alloc_history).  The fast chain uses buffer 0 of tr[] and dnB[] for the reference-format views of chain_output,
  // and `composed` double-buffered by frame parity (composed.buf[cur] is output 0).
  HistPlane composed, tr[2], dnA[2], dnB[2];
  rfx_plane fb{};  // denoise_mode != full: the FramebufferTexture copy of the temporal target's attachment 0 (TemporalReprojectPass.js:134-152,197-200)
  // fast chain (fast_math on at creation, mode SSGI): interleaved internal planes
  bool fastpath = false;
  IPlane nrdz, tr32;
  // the Poisson targets A / B of the fast chain, both planes of a target interleaved in one 16-byte texel (typed RGBA32F for their
  // size).  fdnA.buf[1] is used by row-sharded groups only (the A target double-buffered like B, see chain_render_fast).
  HistPlane fdnA, fdnB;
  uint64_t frame_idx = 0;    // frames completed (advances with the frame's last launch)
  bool views_valid = false;  // tr[]/dnB[] hold the split views of the current frame's interleaved planes
  // host-buffer entry points: the staging sets of the four input planes and their copy pipeline (see rfx_ssgi_chain_submit_host)
  rfx_plane in_depth[2]{}, in_gb[2]{}, in_vel[2]{}, in_direct[2]{};
  HostPipe host;
  int dn_buf[2] = {-1, -1};  // fast chain: which composed buffer the D2H of staging set 0 / 1 reads
  // cross-frame state (TemporalReprojectPass.js:203-213)
  bool have_prev = false;
  float prev_view[16], prev_world[16], prev_proj[16], prev_proj_inv[16], prev_pos[3];
  float keep_data = 0.0f;  // SSGIEffect's constructor resets the denoiser (makeOptionsReactive -> reset())
  // blue-noise counters: one closure per material (BlueNoiseUtils.js:17-33)
  int32_t bn_trace = 0, bn_poisson = 0;
  // the TRAA tail (`tail`, after K4) reads the frame's camera and the previous-frame matrices its K2 used
  rfx_temporal_params traa_tp{};
  // debug view of the tail's K5 (rfx_ssgi_chain_set_debug_view); RFX_DEBUG_VIEW_NONE: composed, isDebug off
  int32_t debug_view = RFX_DEBUG_VIEW_NONE;
  rfx_plane debug_gb{};                 // GBufferDebugPass target of the G-buffer channel views
  // the compose stage (rfx_ssgi_chain_set_compose): K5 of output 0 into `image` (output 9).  The fast chain writes image[frame parity]
  // (as `composed`, so that a host-path download of frame i-1 never races frame i); the per-pass chain writes image[0].
  bool compose_on = false;
  rfx_ssgi_compose_params compose_p{};
  rfx_plane image[2]{};
  // optional per-pass event timing
  bool profiling = false;
  struct Span { cudaEvent_t a, b; int slot; };
  std::vector<Span> spans;
  std::vector<cudaEvent_t> event_pool;
};

static PV rpv(const rfx_plane& p) { return PV{(const unsigned char*)p.ptr, (int)p.width, (int)p.height, (long long)p.pitch}; }
static OutV rov(const rfx_plane& p) { return OutV{(unsigned char*)p.ptr, (long long)p.pitch}; }
// view[b] of `h` in a group of n ranks; base[r]: rank r's buffer b.  n = 1 with this rank's buffer: the view a chain reads alone.
static void set_view(HistPlane& h, int b, const void* const* base, int n) {
  PeerPV& v = h.view[b];
  v = PeerPV{};
  v.local = rpv(h.buf[b]);
  v.n = n;
  for (int r = 0; r < n; r++) v.base[r] = (const unsigned char*)base[r];
  v.own0 = 0; v.own1 = v.local.h;
}
static void local_views(HistPlane& h) {
  for (int b = 0; b < 2; b++) set_view(h, b, &h.buf[b].ptr, 1);
}
static std::array<HistPlane*, 9> every_hist_plane(rfx_ssgi_chain* ch) {  // whether the chain's configuration keeps it or not (the tail's aside)
  return {&ch->composed, &ch->tr[0], &ch->tr[1], &ch->dnA[0], &ch->dnA[1], &ch->dnB[0], &ch->dnB[1], &ch->fdnA, &ch->fdnB};
}
// per-pass chain and AO chain: the buffer of every plane they keep that holds the latest frame (rfx_group.inl)
static int pass_latest(const GroupMember* ch);

static void traa_free(rfx_ctx* ctx, TraaTail& t) {
  for (rfx_plane* p : {&t.acc.buf[0], &t.acc.buf[1], &t.out, &t.mid.buf[0], &t.mid.buf[1], &t.fx_plane}) if (p->ptr) rfx_plane_free(ctx, p);
}
// rfx_*_chain_enable_traa once the chain kind's own checks passed: NULL frees the tail's planes.  Otherwise the planes are allocated on
// first use (`out` where the chain asks for it; nothing is left allocated on failure), and the options replace the old ones.
static rfx_status traa_enable(rfx_ctx* ctx, TraaTail& t, const rfx_traa_tail_options* opt, uint32_t W, uint32_t H, bool with_out) {
  if (!opt) {
    CU(cudaStreamSynchronize(ctx->stream));
    traa_free(ctx, t);
    t.on = false;
    t.blur = false;  // the stages end the tail: they go with it
    t.fx = false;
    return RFX_OK;
  }
  if (!t.acc.buf[0].ptr) {
    rfx_status st = RFX_OK;
    for (rfx_plane* p : {&t.acc.buf[0], &t.acc.buf[1], with_out ? &t.out : nullptr, &t.mid.buf[0]})
      if (p && st == RFX_OK) st = rfx_plane_alloc(ctx, RFX_FMT_RGBA16F, W, H, p);
    if (st != RFX_OK) { traa_free(ctx, t); return st; }
    local_views(t.acc);
    local_views(t.mid);
  }
  t.opt = *opt;
  t.on = true;
  t.keep = 0.0f;  // a new TemporalReprojectPass, or TemporalReprojectPass.reset()
  return RFX_OK;
}
// rfx_*_chain_set_motion_blur: `fixed` = the chain's tail cannot change (it is attached to a group), so neither can the stage; its values can.
static rfx_status traa_set_blur(rfx_ctx* ctx, TraaTail& t, const rfx_motion_blur_params* p, bool fixed) {
  if (!t.on) return fail(ctx, RFX_ERR_NOT_READY, "set_motion_blur: the motion-blur stage shares the TRAA tail's pass, and the tail is off");
  if (fixed && (p != nullptr) != t.blur)
    return fail(ctx, RFX_ERR_UNSUPPORTED, "set_motion_blur: the chain is attached to a group, whose planes are fixed at attach time: the stage cannot be turned on or off");
  if (p && p->samples < 1) return fail(ctx, RFX_ERR_INVALID_ARG, "set_motion_blur: samples < 1");
  t.blur = p != nullptr;
  if (p) t.blur_p = *p;
  return RFX_OK;
}
// The checks of an effects list shared by rfx_effects_launch's callers on the host (rfx_*_chain_set_effects, rfx_fx_stage_rows).
static bool fx_list_ok(const rfx_effects_params* p) {
  if (!p || p->n_effects < 1 || p->n_effects > 4) return false;
  for (int i = 0; i < p->n_effects; i++)
    if (p->effects[i] < RFX_FX_SHARPNESS || p->effects[i] > RFX_FX_SPARKLE) return false;
  return true;
}
// rfx_*_chain_set_effects: the stage needs the tail; turning it on allocates its plane, turning it off frees it.  It keeps nothing across
// frames and no peer reads it, so a chain in a group may change it between frames, but not between the two phases of a split frame.
static rfx_status traa_set_fx(rfx_ctx* ctx, TraaTail& t, const rfx_effects_params* p, uint32_t W, uint32_t H) {
  if (!t.on) return fail(ctx, RFX_ERR_NOT_READY, "set_effects: the cosmetic stage runs over the TRAA tail's image, and the tail is off");
  if (t.pending) return fail(ctx, RFX_ERR_NOT_READY, "set_effects: the last row-sharded frame waits for its second phase (render_sharded_finish)");
  if (p && !fx_list_ok(p)) return fail(ctx, RFX_ERR_INVALID_ARG, "set_effects: n_effects must be 1..4 and every effect an RFX_FX_* id");
  if (!p) {
    if (t.fx_plane.ptr) {
      CU(cudaStreamSynchronize(ctx->stream));
      rfx_plane_free(ctx, &t.fx_plane);
      t.fx_plane = rfx_plane{};
    }
    t.fx = false;
    return RFX_OK;
  }
  if (!t.fx_plane.ptr) {
    rfx_status st = rfx_plane_alloc(ctx, RFX_FMT_RGBA16F, W, H, &t.fx_plane);
    if (st != RFX_OK) return st;
  }
  t.fx_p = *p;
  t.fx = true;
  return RFX_OK;
}
// The end of a frame's tail, after its last pass (K9 or the merged TRAA + motion-blur pass): the cosmetic stage's launch
// when it is on.  The tail advances first: its TRAA planes are complete whatever the stage returns.
static rfx_status tail_end(rfx_ctx* ctx, void* stream, TraaTail& t) {
  t.advance();
  if (!t.fx) return RFX_OK;
  const auto& j = t.fx_job;
  return rfx_effects_launch(ctx, stream, &t.fx_p, &j.in, &j.depth, &j.velocity, &j.out, (uint32_t)j.r0, (uint32_t)j.r1);
}

static cudaEvent_t chain_event(rfx_ssgi_chain* ch) {
  if (!ch->event_pool.empty()) { cudaEvent_t e = ch->event_pool.back(); ch->event_pool.pop_back(); return e; }
  cudaEvent_t e = nullptr;
  cudaEventCreate(&e);
  return e;
}
struct SpanGuard {  // records an event pair around one launch when profiling is on
  rfx_ssgi_chain* ch; cudaStream_t s; cudaEvent_t a = nullptr; int slot;
  SpanGuard(rfx_ssgi_chain* c, cudaStream_t st, int sl) : ch(c), s(st), slot(sl) { if (ch->profiling) { a = chain_event(ch); cudaEventRecord(a, s); } }
  ~SpanGuard() { if (a) { cudaEvent_t b = chain_event(ch); cudaEventRecord(b, s); ch->spans.push_back({a, b, slot}); } }
};

static int32_t next_blue(int32_t start, int32_t& counter) {  // BlueNoiseUtils.js:25-28
  const int64_t highest = 0x7fffffff;
  counter = (int32_t)(((int64_t)start + (int64_t)counter + 1) % highest);
  return counter;
}

extern "C" {

rfx_status rfx_ssgi_chain_create(rfx_ctx* ctx, const rfx_ssgi_chain_options* opt, rfx_ssgi_chain** out) {
  if (!ctx || !opt || !out || opt->width == 0 || opt->height == 0 || opt->denoise_iterations < 0) return fail(ctx, RFX_ERR_INVALID_ARG, "chain_create: bad arguments");
  rfx_ssgi_chain* ch = new rfx_ssgi_chain();
  ch->ctx = ctx;
  ch->opt = *opt;
  rfx_status st = RFX_OK;
  auto alloc = [&](int fmt, rfx_plane* p) { if (st == RFX_OK) st = rfx_plane_alloc(ctx, fmt, opt->width, opt->height, p); };
  auto ialloc = [&](size_t texel, IPlane* p) {
    if (st != RFX_OK) return;
    p->pitch = ((size_t)opt->width * texel + 255) & ~(size_t)255;
    if (p->pitch * opt->height >= (1ull << 32)) { st = fail(ctx, RFX_ERR_UNSUPPORTED, "chain_create: internal plane exceeds 4 GiB"); return; }
    if (cudaMalloc(&p->p, p->pitch * opt->height) != cudaSuccess || cudaMemset(p->p, 0, p->pitch * opt->height) != cudaSuccess) st = fail(ctx, RFX_ERR_CUDA, "chain_create: cudaMalloc failed");
  };
  CU(cudaSetDevice(ctx->device));
  if (opt->denoise_mode < RFX_DENOISE_FULL || opt->denoise_mode > RFX_DENOISE_TEMPORAL) {
    delete ch;
    return fail(ctx, RFX_ERR_UNSUPPORTED, "chain_create: denoise_mode must be full / full_temporal / temporal (\"denoised\" hands an array of textures to a sampler in the reference and cannot run there either)");
  }
  const bool scaled = opt->resolution_scale != 0.0f && opt->resolution_scale != 1.0f;
  if (scaled && !(opt->resolution_scale > 0.0f && opt->resolution_scale < 1.0f)) { delete ch; return fail(ctx, RFX_ERR_INVALID_ARG, "chain_create: resolution_scale must be in (0, 1]"); }
  const uint32_t sw = scaled ? (uint32_t)((double)opt->width * (double)opt->resolution_scale) : opt->width;   // renderTarget.setSize(width * scale, height * scale)
  const uint32_t sh = scaled ? (uint32_t)((double)opt->height * (double)opt->resolution_scale) : opt->height;
  if (sw == 0 || sh == 0) { delete ch; return fail(ctx, RFX_ERR_INVALID_ARG, "chain_create: resolution_scale leaves an empty SSGI target"); }
  // latched: the history formats differ between the paths; the fused fast chain needs the full-size SSGI target and the Poisson history
  ch->fastpath = ctx->fast_math && opt->mode == RFX_MODE_SSGI && opt->denoise_mode == RFX_DENOISE_FULL && !scaled;
  if (st == RFX_OK) st = rfx_plane_alloc(ctx, RFX_FMT_RGBA32F, sw, sh, &ch->ssgi_out);
  if (opt->denoise_mode != RFX_DENOISE_FULL) alloc(RFX_FMT_RGBA32F, &ch->fb);
  if (ch->fastpath) {
    ialloc(16, &ch->nrdz); ialloc(32, &ch->tr32);
    for (HistPlane* h : {&ch->fdnA, &ch->fdnB, &ch->composed})
      for (rfx_plane& b : h->buf) alloc(RFX_FMT_RGBA32F, &b);
  } else {
    for (int i = 0; i < 2; i++) { alloc(RFX_FMT_RGBA32F, &ch->tr[i].buf[0]); alloc(RFX_FMT_RGBA16F, &ch->dnA[i].buf[0]); alloc(RFX_FMT_RGBA16F, &ch->dnB[i].buf[0]); }
    alloc(RFX_FMT_RGBA32F, &ch->composed.buf[0]);
  }
  if (st != RFX_OK) { rfx_ssgi_chain_destroy(ch); return st; }
  for (HistPlane* h : every_hist_plane(ch)) local_views(*h);
  *out = ch;
  return RFX_OK;
}

void rfx_ssgi_chain_destroy(rfx_ssgi_chain* ch) {
  if (!ch) return;
  rfx_ctx* ctx = ch->ctx;
  cudaStreamSynchronize(ctx->stream);
  host_pipe_destroy(ch->host);
  for (HistPlane* h : every_hist_plane(ch))
    for (rfx_plane& p : h->buf) if (p.ptr) rfx_plane_free(ctx, &p);
  traa_free(ctx, ch->tail);
  rfx_plane* all[] = {&ch->fb, &ch->ssgi_out, &ch->debug_gb, &ch->image[0], &ch->image[1],
                      &ch->in_depth[0], &ch->in_gb[0], &ch->in_vel[0], &ch->in_direct[0], &ch->in_depth[1], &ch->in_gb[1], &ch->in_vel[1], &ch->in_direct[1]};
  for (rfx_plane* p : all) if (p->ptr) rfx_plane_free(ctx, p);
  for (IPlane* p : {&ch->nrdz, &ch->tr32}) if (p->p) cudaFree(p->p);
  for (auto& sp : ch->spans) { cudaEventDestroy(sp.a); cudaEventDestroy(sp.b); }
  for (cudaEvent_t e : ch->event_pool) cudaEventDestroy(e);
  delete ch;
}

rfx_status rfx_ssgi_chain_set_profiling(rfx_ssgi_chain* ch, int32_t enable) {
  if (!ch) return RFX_ERR_INVALID_ARG;
  ch->profiling = enable != 0;
  return RFX_OK;
}
rfx_status rfx_ssgi_chain_get_profile(rfx_ssgi_chain* ch, double* ms, uint64_t* launches) {
  if (!ch || !ms || !launches) return RFX_ERR_INVALID_ARG;
  rfx_ctx* ctx = ch->ctx;
  CU(cudaDeviceSynchronize());
  for (auto& sp : ch->spans) {
    float t = 0.0f;
    CU(cudaEventElapsedTime(&t, sp.a, sp.b));
    ms[sp.slot] += (double)t;
    launches[sp.slot] += 1;
    ch->event_pool.push_back(sp.a);
    ch->event_pool.push_back(sp.b);
  }
  ch->spans.clear();
  return RFX_OK;
}

rfx_status rfx_ssgi_chain_set_options(rfx_ssgi_chain* ch, const rfx_ssgi_chain_options* opt) {
  if (!ch || !opt) return RFX_ERR_INVALID_ARG;
  if (opt->width != ch->opt.width || opt->height != ch->opt.height) return fail(ch->ctx, RFX_ERR_SIZE_MISMATCH, "chain_set_options: size change needs a new chain");
  if (opt->denoise_iterations < 0 || opt->steps < 1 || opt->refine_steps < 0) return fail(ch->ctx, RFX_ERR_INVALID_ARG, "chain_set_options: bad option value");
  if (opt->denoise_mode != ch->opt.denoise_mode || opt->mode != ch->opt.mode) return fail(ch->ctx, RFX_ERR_UNSUPPORTED, "chain_set_options: mode / denoise_mode are constructor options (Denoiser.js:17-64): create a new chain");
  if (opt->resolution_scale != ch->opt.resolution_scale) return fail(ch->ctx, RFX_ERR_SIZE_MISMATCH, "chain_set_options: resolution_scale resizes the SSGI target (SSGIEffect.js:193-196 calls setSize): create a new chain");
  const int32_t start = ch->opt.blue_noise_start;
  ch->opt = *opt;
  ch->opt.blue_noise_start = start;  // the blue-noise closures keep their start index for the life of the material
  ch->keep_data = 0.0f;              // every reference setter ends with this.reset()
  return RFX_OK;
}

rfx_status rfx_ssgi_chain_reset(rfx_ssgi_chain* ch) {
  if (!ch) return RFX_ERR_INVALID_ARG;
  ch->keep_data = 0.0f;  // TemporalReprojectPass.reset()  :158-160
  ch->tail.keep = 0.0f;  // the TRAA pass's too (TRAAEffect.reset)
  return RFX_OK;
}

rfx_status rfx_ssgi_chain_enable_traa(rfx_ssgi_chain* ch, const rfx_traa_tail_options* opt) {
  if (!ch) return RFX_ERR_INVALID_ARG;
  if (ch->group) return fail(ch->ctx, RFX_ERR_UNSUPPORTED, "chain_enable_traa: the chain is attached to a group, whose peer mappings are fixed at attach time");
  if (opt && ch->compose_on) return fail(ch->ctx, RFX_ERR_INVALID_ARG, "chain_enable_traa: the compose stage is on, and the tail runs K5 itself (turn the stage off first)");
  return traa_enable(ch->ctx, ch->tail, opt, ch->opt.width, ch->opt.height, true);
}

rfx_status rfx_ssgi_chain_set_compose(rfx_ssgi_chain* ch, const rfx_ssgi_compose_params* p) {
  if (!ch) return RFX_ERR_INVALID_ARG;
  rfx_ctx* ctx = ch->ctx;
  if (!p) {
    if (ch->image[0].ptr) {  // no launch or download may still use the planes
      CU(cudaStreamSynchronize(ctx->stream));
      rfx_status st = host_pipe_wait(ctx, ch->host, 0);
      if (st != RFX_OK) return st;
      for (rfx_plane& b : ch->image)
        if (b.ptr) { rfx_plane_free(ctx, &b); b = rfx_plane{}; }
    }
    ch->compose_on = false;
    return RFX_OK;
  }
  if (p->is_debug) return fail(ctx, RFX_ERR_INVALID_ARG, "chain_set_compose: is_debug is not a stage option (select a view with rfx_ssgi_chain_set_debug_view)");
  if (ch->tail.on) return fail(ctx, RFX_ERR_INVALID_ARG, "chain_set_compose: the TRAA tail is on, and it runs K5 itself");
  for (int b = 0; b < (ch->fastpath ? 2 : 1); b++)
    if (!ch->image[b].ptr) {
      rfx_status st = rfx_plane_alloc(ctx, RFX_FMT_RGBA16F, ch->opt.width, ch->opt.height, &ch->image[b]);
      if (st != RFX_OK) return st;
    }
  ch->compose_p = *p;
  ch->compose_on = true;
  return RFX_OK;
}

rfx_status rfx_ssgi_chain_set_motion_blur(rfx_ssgi_chain* ch, const rfx_motion_blur_params* p) {
  if (!ch) return RFX_ERR_INVALID_ARG;
  return traa_set_blur(ch->ctx, ch->tail, p, ch->group != nullptr);
}

rfx_status rfx_ssgi_chain_set_effects(rfx_ssgi_chain* ch, const rfx_effects_params* p) {
  if (!ch) return RFX_ERR_INVALID_ARG;
  return traa_set_fx(ch->ctx, ch->tail, p, ch->opt.width, ch->opt.height);
}

}  // extern "C"
// fast chain: tr[]/dnB[] buffer 0 := the reference-format views of the interleaved planes, dn from fdnB.buf[parity]
static rfx_status split_views(rfx_ssgi_chain* ch, int parity, cudaStream_t s) {
  rfx_ctx* ctx = ch->ctx;
  const int W = (int)ch->opt.width, H = (int)ch->opt.height;
  LAUNCHED(launch_split_tr(PV{(const unsigned char*)ch->tr32.p, W, H, (long long)ch->tr32.pitch}, rov(ch->tr[0].buf[0]), rov(ch->tr[1].buf[0]), W, H, s));
  LAUNCHED(launch_split_dn(rpv(ch->fdnB.buf[parity]), rov(ch->dnB[0].buf[0]), rov(ch->dnB[1].buf[0]), W, H, s));
  ch->views_valid = true;
  return RFX_OK;
}
// fast chain: the reference-format planes tr[]/dnB[] buffer 0 that split_views fills (allocated once, on first use)
static rfx_status alloc_split_views(rfx_ssgi_chain* ch) {
  rfx_status st = RFX_OK;
  for (int i = 0; i < 2 && st == RFX_OK; i++) {
    if (!ch->tr[i].buf[0].ptr) st = rfx_plane_alloc(ch->ctx, RFX_FMT_RGBA32F, ch->opt.width, ch->opt.height, &ch->tr[i].buf[0]);
    if (st == RFX_OK && !ch->dnB[i].buf[0].ptr) st = rfx_plane_alloc(ch->ctx, RFX_FMT_RGBA16F, ch->opt.width, ch->opt.height, &ch->dnB[i].buf[0]);
  }
  return st;
}
extern "C" {

rfx_status rfx_ssgi_chain_output(rfx_ssgi_chain* ch, int32_t which, rfx_plane* out) {
  if (!ch || !out) return RFX_ERR_INVALID_ARG;
  rfx_ctx* ctx = ch->ctx;
  if (which < 0 || which > 9) return fail(ctx, RFX_ERR_INVALID_ARG, "chain_output: which must be 0..9");
  if (which == 9) {
    if (!ch->compose_on) return fail(ctx, RFX_ERR_INVALID_ARG, "chain_output: output 9 needs the compose stage (rfx_ssgi_chain_set_compose)");
    *out = ch->image[ch->fastpath ? (int)((ch->frame_idx + 1) & 1) : 0];  // the fast chain's by the parity of the latest frame
    return RFX_OK;
  }
  if (which >= 6) {
    if (!ch->tail.on) return fail(ctx, RFX_ERR_NOT_READY, "chain_output: outputs 6 / 7 / 8 need the TRAA tail (rfx_ssgi_chain_enable_traa)");
    if (which == 8 && !ch->tail.fx) return fail(ctx, RFX_ERR_NOT_READY, "chain_output: output 8 needs the cosmetic stage (rfx_ssgi_chain_set_effects)");
    // with the cosmetic stage on, output 6 is its image and 8 the tail's image it reads
    *out = which == 7 ? ch->tail.latest() : which == 6 && ch->tail.fx ? ch->tail.fx_plane : ch->tail.out;
    return RFX_OK;
  }
  if (ch->fastpath) {
    const int last = (int)((ch->frame_idx + 1) & 1);  // parity of the most recently completed frame
    if (which == 0) { *out = ch->composed.buf[last]; return RFX_OK; }
    if (which == 1) { *out = ch->ssgi_out; return RFX_OK; }
    // views of the interleaved planes in the reference's formats, refreshed on the context stream
    rfx_plane *tr0 = &ch->tr[0].buf[0], *tr1 = &ch->tr[1].buf[0], *dn0 = &ch->dnB[0].buf[0], *dn1 = &ch->dnB[1].buf[0];
    if (!tr0->ptr || !dn1->ptr) {
      rfx_status st = alloc_split_views(ch);
      if (st != RFX_OK) return st;
    }
    if (!ch->views_valid) {
      rfx_status st = split_views(ch, last, ctx->stream);
      if (st != RFX_OK) return st;
    }
    *out = which == 2 ? *tr0 : which == 3 ? *tr1 : which == 4 ? *dn0 : *dn1;
    return RFX_OK;
  }
  // a plane the chain keeps holds the latest frame in buffer pass_latest; the others are single-buffered
  const int b = pass_latest(ch);
  auto latest = [&](const HistPlane& h) { return h.buf[h.buf[1].ptr ? b : 0]; };
  switch (which) {
    case 0: *out = latest(ch->opt.denoise_mode == RFX_DENOISE_TEMPORAL ? ch->tr[0] : ch->composed); break;  // denoiser.texture (Denoiser.js:67-78)
    case 1: *out = ch->ssgi_out; break;
    case 2: *out = latest(ch->tr[0]); break;
    case 3: *out = latest(ch->tr[1]); break;
    case 4: *out = latest(ch->dnB[0]); break;
    default: *out = latest(ch->dnB[1]); break;
  }
  return RFX_OK;
}

rfx_status rfx_ssgi_chain_set_debug_view(rfx_ssgi_chain* ch, int32_t view) {
  if (!ch) return RFX_ERR_INVALID_ARG;
  rfx_ctx* ctx = ch->ctx;
  if (view == RFX_DEBUG_VIEW_OUTPUT) view = RFX_DEBUG_VIEW_NONE;  // denoiser.texture: isDebug is false (SSGIEffect.js:249)
  const bool plane = view > RFX_DEBUG_VIEW_OUTPUT && view <= RFX_DEBUG_VIEW_OUTPUT + 5;
  const bool channel = view >= RFX_DEBUG_VIEW_GBUFFER_CHANNEL && view <= RFX_DEBUG_VIEW_GBUFFER_CHANNEL + 5;
  if (!(view == RFX_DEBUG_VIEW_NONE || plane || channel || view == RFX_DEBUG_VIEW_DEPTH || view == RFX_DEBUG_VIEW_VELOCITY || view == RFX_DEBUG_VIEW_GBUFFER))
    return fail(ctx, RFX_ERR_INVALID_ARG, "chain_set_debug_view: unknown view %d", view);
  if (view != RFX_DEBUG_VIEW_NONE && ch->group && rfx_group_world(ch->group) > 1)
    return fail(ctx, RFX_ERR_UNSUPPORTED, "chain_set_debug_view: a chain in a row-sharded group takes no debug view");
  // Every plane a view needs is allocated here, and nothing is launched: the frame that shows the view fills them on its own stream.
  // Every configuration has planes 1..5 (the per-pass chain allocates them all; the fast chain splits its interleaved ones).
  rfx_status st = RFX_OK;
  if (ch->fastpath && plane && view >= RFX_DEBUG_VIEW_OUTPUT + 2) st = alloc_split_views(ch);
  if (st == RFX_OK && channel && !ch->debug_gb.ptr) st = rfx_plane_alloc(ctx, RFX_FMT_RGBA32F, ch->opt.width, ch->opt.height, &ch->debug_gb);
  if (st != RFX_OK) return st;
  ch->debug_view = view;
  return RFX_OK;
}

// Output rows [r0, r1) of chain launch k: ranges[2k], ranges[2k+1] in a row-sharded frame (rfx_shard_ranges), else all H rows
struct Rows { int r0, r1; };
static Rows launch_rows(const uint32_t* ranges, uint32_t k, int H) { return ranges ? Rows{(int)ranges[2 * k], (int)ranges[2 * k + 1]} : Rows{0, H}; }

// ------------------------------------------------------------------------------------------
// fast chain (k_chain.cu): same frame logic as chain_render_impl below, interleaved internal planes, compose fused into the
// last Poisson pass.  Launch indices k (for `ranges` and [k_begin, k_end)) are those of the reference chain — K1, K2, K3 pass
// 0..2n-1, K4 — the K4 range selects the rows the last pass composes.
// ------------------------------------------------------------------------------------------
static PV ipv(const IPlane& p, int w, int h) { return PV{(const unsigned char*)p.p, w, h, (long long)p.pitch}; }
static OutV iov(const IPlane& p) { return OutV{(unsigned char*)p.p, (long long)p.pitch}; }

// K1's uniforms of this frame (SSGIPass.render, src/ssgi/pass/SSGIPass.js:68-95)
static rfx_ssgi_params trace_params(rfx_ssgi_chain* ch, const rfx_ssgi_frame* f) {
  const rfx_ctx* ctx = ch->ctx;
  const rfx_ssgi_chain_options& o = ch->opt;
  rfx_ssgi_params sp{};
  sp.cam = f->cam;
  sp.ray_distance = o.distance; sp.thickness = o.thickness; sp.env_blur = o.env_blur;
  sp.max_env_map_mip_level = ctx->env_set ? (float)((int)std::floor(std::log2((double)std::max(ctx->env.size_x, ctx->env.size_y))) + 1) : 0.0f;  // Utils.js:30-34
  sp.steps = o.steps; sp.refine_steps = o.refine_steps; sp.mode = o.mode; sp.flags = o.ssgi_flags;
  sp.blue_noise_index = next_blue(o.blue_noise_start, ch->bn_trace);
  return sp;
}

// Before K2: the first frame's previous camera is the current one (the constructor clones the current camera matrices,
// TemporalReprojectPass.js:94-97).  The current (un-jittered) camera and the previous-frame matrices are also kept for the TRAA tail
// (its TemporalReprojectPass tracks the same camera, so its previous frame is the chain's).
static void prev_camera_init(rfx_ssgi_chain* ch, const rfx_ssgi_frame* f) {
  if (!ch->have_prev) {
    memcpy(ch->prev_view, f->cam.view_matrix, 64); memcpy(ch->prev_world, f->cam.camera_matrix_world, 64);
    memcpy(ch->prev_proj, f->cam.projection, 64); memcpy(ch->prev_proj_inv, f->cam.projection_inverse, 64);
    memcpy(ch->prev_pos, f->camera_pos, 12);
    ch->have_prev = true;
  }
  rfx_temporal_params& tp = ch->traa_tp;
  tp.cam = f->cam;
  memcpy(tp.prev_view_matrix, ch->prev_view, 64); memcpy(tp.prev_camera_matrix_world, ch->prev_world, 64);
  memcpy(tp.prev_projection, ch->prev_proj, 64); memcpy(tp.prev_projection_inverse, ch->prev_proj_inv, 64);
  memcpy(tp.camera_pos, f->camera_pos, 12); memcpy(tp.prev_camera_pos, ch->prev_pos, 12);
}
// After K2 (TemporalReprojectPass.js:195,203-213): keep the history from now on, and this frame's camera is the next one's previous
static void prev_camera_roll(rfx_ssgi_chain* ch, const rfx_ssgi_frame* f) {
  ch->keep_data = 1.0f;
  memcpy(ch->prev_world, f->cam.camera_matrix_world, 64); memcpy(ch->prev_view, f->cam.view_matrix, 64);
  memcpy(ch->prev_proj, f->cam.projection, 64); memcpy(ch->prev_proj_inv, f->cam.projection_inverse, 64);
  memcpy(ch->prev_pos, f->camera_pos, 12);
}

// The plane the tail's K5 shows for the chain's debug view in this frame (the fast chain splits this frame's interleaved planes; the
// G-buffer channel views run GBufferDebugPass, which SSGIEffect.update renders right after SSGIPass, SSGIEffect.js:398-399)
static rfx_status debug_view_plane(rfx_ssgi_chain* ch, void* stream, const rfx_ssgi_frame* f, const rfx_plane** out) {
  const int v = ch->debug_view;
  if (v == RFX_DEBUG_VIEW_DEPTH) *out = f->depth;
  else if (v == RFX_DEBUG_VIEW_VELOCITY) *out = f->velocity;
  else if (v == RFX_DEBUG_VIEW_GBUFFER) *out = f->gbuffer;
  else if (v >= RFX_DEBUG_VIEW_GBUFFER_CHANNEL) {
    rfx_status st = rfx_gbuffer_debug_launch(ch->ctx, stream, v - RFX_DEBUG_VIEW_GBUFFER_CHANNEL, f->gbuffer, &ch->debug_gb, 0, 0);
    if (st != RFX_OK) return st;
    *out = &ch->debug_gb;
  } else if (v == RFX_DEBUG_VIEW_OUTPUT + 1) {
    *out = &ch->ssgi_out;
  } else if (ch->fastpath) {
    rfx_status st = split_views(ch, (int)(ch->frame_idx & 1), pick(ch->ctx, stream));
    if (st != RFX_OK) return st;
    *out = v == 2 ? &ch->tr[0].buf[0] : v == 3 ? &ch->tr[1].buf[0] : v == 4 ? &ch->dnB[0].buf[0] : &ch->dnB[1].buf[0];
  } else {
    *out = v == 2 ? &ch->tr[0].buf[0] : v == 3 ? &ch->tr[1].buf[0] : v == 4 ? &ch->dnB[0].buf[0] : &ch->dnB[1].buf[0];  // alone: buffer 0
  }
  return RFX_OK;
}

// The TRAA pass of a chain's frame tail (TRAAEffect, shared by the SSGI and AO chains).  traa_params: K2's uniforms, TRAAEffect's forced
// options (TRAAEffect.js:21-31) over the TemporalReprojectPass defaults, on cam_tp's camera and previous-frame matrices.
static rfx_temporal_params traa_params(const TraaTail& t, const rfx_temporal_params& cam_tp, int32_t camera_moved) {
  const rfx_traa_tail_options& o = t.opt;
  rfx_temporal_params tp = cam_tp;
  tp.max_blend = o.max_blend; tp.neighborhood_clamp_intensity = o.neighborhood_clamp_intensity;
  tp.confidence_power = o.confidence_power; tp.log_transform = o.log_transform ? 1 : 0;
  tp.keep_data = t.keep;
  tp.full_accumulate = o.full_accumulate && !camera_moved ? 1 : 0;
  tp.texture_count = 1; tp.input_type = RFX_INPUT_DIFFUSE; tp.history_linear = 1;
  tp.reproject_specular[0] = tp.reproject_specular[1] = 0;
  return tp;
}
// K2 in its TRAA form over the tail's `mid` on the output rows kr +- 1 (K9's LINEAR fetch) into buffer cur() of the accumulated plane,
// reading last frame's other buffer (in a row-sharded group of n > 1, `peer`: on the rank that owns each row), then K9 from it into `out`
// on kr, or with the motion-blur stage on the merged TRAA + motion-blur pass, whose taps read all of `mid`.  `mid` must hold rows
// kr +- RFX_TRAA_TAIL_ROWS (with the stage alone: every row).  Then the tail ends (tail_end: the cosmetic stage, the advance).  With a
// split frame (t.split) the merged pass and the tail's end wait for phase 2 (traa_blur_finish): this returns with t.pending set.
static rfx_status traa_launches(rfx_ctx* ctx, void* stream, const rfx_temporal_params& tp, TraaTail& t, const rfx_plane* velocity, bool peer,
                                const rfx_plane* out, Rows kr) {
  const int cur = t.cur(), H = (int)t.acc.buf[cur].height;
  TemporalPeer tpeer{};
  tpeer.hist0 = tpeer.hist1 = t.acc.view[cur ^ 1];
  rfx_status st = temporal_reproject(ctx, stream, &tp, &t.mid_w(), velocity, &t.acc.buf[cur ^ 1], nullptr, &t.acc.buf[cur], nullptr, std::max(0, kr.r0 - 1),
                                     std::min(H, kr.r1 + 1), peer ? &tpeer : nullptr);
  if (st != RFX_OK) return st;
  if (t.blur && t.split) {
    t.p2_velocity = *velocity; t.p2_out = *out; t.p2_r0 = kr.r0; t.p2_r1 = kr.r1;
    t.pending = true;
    return RFX_OK;
  }
  if (t.blur) st = traa_motion_blur(ctx, stream, &t.blur_p, velocity, &t.acc.buf[cur], &t.mid_w(), out, (uint32_t)kr.r0, (uint32_t)kr.r1, nullptr);
  else st = rfx_traa_compose_launch(ctx, stream, &t.acc.buf[cur], out, (uint32_t)kr.r0, (uint32_t)kr.r1);
  return st != RFX_OK ? st : tail_end(ctx, stream, t);
}
// Phase 2 of a split frame, after the frame's barrier: the merged pass on the band, its taps reading this frame's `mid` through `mid_view`
// (each row on its owner, or the local plane once the rows were replicated), then the tail advances.
static rfx_status traa_blur_finish(rfx_ctx* ctx, void* stream, TraaTail& t, const PeerPV& mid_view) {
  const int cur = t.cur();
  rfx_status st = traa_motion_blur(ctx, stream, &t.blur_p, &t.p2_velocity, &t.acc.buf[cur], &t.mid_w(), &t.p2_out, (uint32_t)t.p2_r0, (uint32_t)t.p2_r1,
                                   mid_view.n > 1 ? &mid_view : nullptr);
  if (st != RFX_OK) return st;
  t.pending = false;
  return tail_end(ctx, stream, t);
}

// The compose stage as a per-pass launch on rows kr: K5 of output 0 (`out0`), or with a debug view selected K5 with isDebug of the view,
// into `out` (the per-pass chain, and the fast chain while a view is selected)
static rfx_status chain_render_stage(rfx_ssgi_chain* ch, void* stream, const rfx_ssgi_frame* f, const rfx_plane* out0, const rfx_plane* out, Rows kr) {
  rfx_ssgi_compose_params q = ch->compose_p;
  const rfx_plane* view = out0;
  if (ch->debug_view != RFX_DEBUG_VIEW_NONE) {
    q.is_debug = 1;
    rfx_status st = debug_view_plane(ch, stream, f, &view);
    if (st != RFX_OK) return st;
  }
  return rfx_ssgi_compose_launch(ch->ctx, stream, &q, f->depth, view, f->direct_light, out, (uint32_t)kr.r0, (uint32_t)kr.r1);
}
// The compose stage fused into the fast chain's K4 (cpoisson / ccompose with k5.out set): K5's planes and uniforms, `out` its image
static rfx_status stage_args(rfx_ssgi_chain* ch, const rfx_ssgi_frame* f, const rfx_plane& out, SsgiComposeArgs& c) {
  rfx_ctx* ctx = ch->ctx;
  const int W = (int)ch->opt.width, H = (int)ch->opt.height;
  if (!pv(f->depth, RFX_FMT_R32F, c.depth) || !pv(f->direct_light, RFX_FMT_RGBA16F, c.scene) || !ov(&out, RFX_FMT_RGBA16F, c.out))
    return fail(ctx, RFX_ERR_BAD_FORMAT, "chain: the compose stage needs an RGBA16F direct light plane");
  if (c.scene.w != W || c.scene.h != H) return fail(ctx, RFX_ERR_SIZE_MISMATCH, "chain: the direct light plane must match the chain size");
  c.W = W; c.H = H; c.row0 = 0; c.row1 = H;
  compose_uniforms(ch->compose_p, c);
  return RFX_OK;
}

// The TRAA tail (launch k of the frame): K5 of `composed` (or with a debug view selected, K5 with isDebug of the view) -> K2 in its TRAA
// form -> K9, as the three per-pass entry points on the rows each needs (K5 on the K9 rows +- RFX_TRAA_TAIL_ROWS, K2 on them +- 1).
static rfx_status chain_render_tail(rfx_ssgi_chain* ch, void* stream, const rfx_ssgi_frame* f, const rfx_plane* composed, const uint32_t* ranges, uint32_t k) {
  rfx_ctx* ctx = ch->ctx;
  const int H = (int)ch->opt.height, halo = RFX_TRAA_TAIL_ROWS;
  const Rows kr = launch_rows(ranges, k, H);
  TraaTail& tail = ch->tail;
  if (tail.fx) {  // the cosmetic stage: K9's plane into the stage's plane on launch k + 1's rows (the band; the tail runs on the rows it reads)
    const Rows fr = launch_rows(ranges, k + 1, H);
    tail.fx_job = {tail.out, *f->depth, *f->velocity, tail.fx_plane, fr.r0, fr.r1};
  }
  rfx_status st = RFX_OK;
  rfx_ssgi_compose_params q = tail.opt.compose;
  const rfx_plane* view = composed;
  if (ch->debug_view != RFX_DEBUG_VIEW_NONE) {
    q.is_debug = 1;
    st = debug_view_plane(ch, stream, f, &view);
  }
  if (st == RFX_OK)
    st = rfx_ssgi_compose_launch(ctx, stream, &q, f->depth, view, f->direct_light, &tail.mid_w(), (uint32_t)std::max(0, kr.r0 - halo),
                                 (uint32_t)std::min(H, kr.r1 + halo));
  // in a group of n > 1 the TRAA history rows live on their owners, whichever chain kind renders the rest of the frame
  const bool peer = ch->group && rfx_group_world(ch->group) > 1;
  if (st == RFX_OK) st = traa_launches(ctx, stream, traa_params(tail, ch->traa_tp, f->camera_moved), tail, f->velocity, peer, &tail.out, kr);
  return st;  // the tail ends in traa_launches
}

// 2-D TMA descriptor over a plane of 16-byte texels, addressed as rows of 4-byte elements (the box must pass cpoisson_tma_fits)
static bool encode_texel_map(CUtensorMap* map, const void* base, int W, int H, size_t pitch, int box_w, int box_h) {
  typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                               CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
  static EncodeFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess || !p) return false;
    fn = (EncodeFn)p;
  }
  const cuuint64_t dims[2] = {(cuuint64_t)W * 4, (cuuint64_t)H};
  const cuuint64_t strides[1] = {(cuuint64_t)pitch};
  const cuuint32_t box[2] = {(cuuint32_t)box_w * 4, (cuuint32_t)box_h};
  const cuuint32_t estr[2] = {1, 1};
  return fn(map, CU_TENSOR_MAP_DATA_TYPE_UINT32, 2, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
            CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

static rfx_status chain_render_fast(rfx_ssgi_chain* ch, void* stream, const rfx_ssgi_frame* f, const uint32_t* ranges, uint32_t k_begin, uint32_t k_end) {
  rfx_ctx* ctx = ch->ctx;
  const rfx_ssgi_chain_options& o = ch->opt;
  const int W = (int)o.width, H = (int)o.height;
  auto on = [&](uint32_t k) { return k >= k_begin && k < k_end; };
  const cudaStream_t cs = stream ? (cudaStream_t)stream : ctx->stream;
  const int cur = (int)(ch->frame_idx & 1), prev = cur ^ 1;
  rfx_status st = RFX_OK;
  PV depth, gb, vel;
  if (!pv(f->depth, RFX_FMT_R32F, depth) || !pv(f->gbuffer, RFX_FMT_RGBA32F, gb) || !pv(f->velocity, RFX_FMT_RGBA32F, vel))
    return fail(ctx, RFX_ERR_BAD_FORMAT, "chain: depth must be R32F, gbuffer / velocity RGBA32F");
  if (depth.w != W || depth.h != H || gb.w != W || gb.h != H || vel.w != W || vel.h != H) return fail(ctx, RFX_ERR_SIZE_MISMATCH, "chain: input planes must match the chain size");
  CamD cam;
  cam_to_dev(f->cam, cam);
  uint32_t k = 0;
  ch->views_valid = false;
  // ---- K1
  if (on(k)) {
    const rfx_ssgi_params sp = trace_params(ch, f);
    const Rows kr = launch_rows(ranges, k, H);
    {
      SpanGuard g(ch, cs, 0);
      st = ssgi_trace(ctx, stream, &sp, f->depth, f->gbuffer, nullptr, f->direct_light, &ch->composed.buf[prev], &ch->ssgi_out, kr.r0, kr.r1,
                      &ch->composed.view[prev]);
    }
    if (st != RFX_OK) return st;
  }
  k++;
  // ---- K2
  if (on(k)) {
    CTemporalArgs a{};
    a.input = rpv(ch->ssgi_out); a.velocity = vel;
    a.hist = ch->fdnB.view[prev];
    a.out = iov(ch->tr32);
    a.W = W; a.H = H;
    const Rows kr = launch_rows(ranges, k, H);
    a.row0 = kr.r0; a.row1 = kr.r1;
    a.cam = cam;
    prev_camera_init(ch, f);
    memcpy(a.prev_world.m, ch->prev_world, 64); memcpy(a.prev_proj_inv.m, ch->prev_proj_inv, 64);
    matmul(ch->prev_proj, ch->prev_view, a.prev_proj_view.m);
    memcpy(a.camera_pos, f->camera_pos, 12);
    a.max_blend = 1.0f; a.clamp_intensity = 0.5f; a.keep_data = ch->keep_data; a.confidence_power = 0.75f;  // Denoiser.js:26-43, TemporalReprojectPass.js:17-32
    a.inv_w = (float)(1.0 / (double)W); a.inv_h = (float)(1.0 / (double)H);
    a.full_accumulate = f->camera_moved ? 0 : 1;
    {
      SpanGuard g(ch, cs, 1);
      LAUNCHED(launch_ctemporal(a, cs));
    }
    prev_camera_roll(ch, f);
  }
  k++;
  // ---- K3 (+ fused K4)
  const int n_pass = 2 * o.denoise_iterations;
  const int halo = (int)std::ceil(o.radius * std::max(1.0f, (float)H / (float)W)) + 1;  // rows a Poisson tap can reach (the offset is rotated AFTER the division by the resolution)
  bool decoded = false;
  auto decode = [&](int row0, int row1) -> rfx_status {
    if (decoded) return RFX_OK;
    CDecodeArgs d{gb, depth, iov(ch->nrdz), W, H};
    LAUNCHED(launch_cdecode(d, row0, row1, halo, cs));
    decoded = true;
    return RFX_OK;
  };
  const uint32_t k_compose = 2u + (uint32_t)n_pass;
  // the compose stage rides on K4 unless a debug view is selected (then it is a launch of its own after K4)
  const bool fused_stage = ch->compose_on && ch->debug_view == RFX_DEBUG_VIEW_NONE;
  for (int i = 0; i < n_pass; i++, k++) {
    if (!on(k)) continue;
    const bool horizontal = (i % 2) == 0, last = i == n_pass - 1;
    CPoissonArgs a{};
    const Rows kr = launch_rows(ranges, k, H);
    a.row0 = kr.r0; a.row1 = kr.r1;
    if ((st = decode(a.row0, a.row1)) != RFX_OK) return st;  // the first pass of a frame has the widest rows of all its passes
    a.nrdz = ipv(ch->nrdz, W, H);
    a.first = i == 0;
    // Target A (even passes).  A `discard`ed pixel keeps its texel = last frame's LAST even pass there (A2), and the LINEAR taps of the next
    // pass read such texels at silhouettes.  One GPU: A is single-buffered and a discard is simply no write.  In a row-sharded group a
    // rank's A rows outside its band hold the result of whichever even pass last covered them (the ranges shrink pass by pass), not the
    // last one's, so A is double-buffered by frame parity like B and the discarded texel is carried from the rank that OWNS the row.
    const int acur = ch->group ? cur : 0;
    a.in = i == 0 ? ipv(ch->tr32, W, H) : rpv(horizontal ? ch->fdnB.buf[cur] : ch->fdnA.buf[acur]);
    a.out = rov(horizontal ? ch->fdnA.buf[acur] : ch->fdnB.buf[cur]);
    if (!horizontal) a.carry = ch->fdnB.view[prev];
    else if (ch->group) a.carry = ch->fdnA.view[prev];
    a.W = W; a.H = H;
    a.radius = o.radius; a.phi = o.phi; a.luma_phi = o.luma_phi; a.depth_phi = o.depth_phi; a.normal_phi = o.normal_phi;
    a.roughness_phi = o.roughness_phi; a.specular_phi = o.specular_phi;
    if ((st = blue_for(ctx, next_blue(o.blue_noise_start, ch->bn_poisson), a.blue)) != RFX_OK) return st;
    a.rot_table = ctx->rot_table;
    a.reach_x = (int)std::ceil(o.radius * std::max(1.0f, (float)W / (float)H)) + 2;
    a.reach_y = (int)std::ceil(o.radius * std::max(1.0f, (float)H / (float)W)) + 2;
    {
      const float SQ = 1.41421356237f;
      const float px[8] = {-1.0f, 0.0f, 1.0f, 0.0f, -0.25f * SQ, 0.25f * SQ, 0.25f * SQ, -0.25f * SQ};
      const float py[8] = {0.0f, -1.0f, 0.0f, 1.0f, -0.25f * SQ, -0.25f * SQ, 0.25f * SQ, 0.25f * SQ};
      for (int t = 0; t < 8; t++) { a.tap_ox[t] = px[t] / (float)W; a.tap_oy[t] = py[t] / (float)H; }
    }
    if (last && on(k_compose)) {
      a.compose = 1;
      const Rows cr = launch_rows(ranges, k_compose, H);
      a.crow0 = cr.r0; a.crow1 = cr.r1;
      a.gb = gb;
      a.composed = rov(ch->composed.buf[cur]);
      a.composed_carry = ch->composed.view[prev];
      a.cam = cam;
      if (fused_stage && (st = stage_args(ch, f, ch->image[cur], a.k5)) != RFX_OK) return st;
    }
    SpanGuard g(ch, cs, i == 0 ? 2 : 3);
    const int box_w = (kTileW + 2 * a.reach_x) | 1, box_h = kTileH + 2 * a.reach_y;  // odd row pitch in texels: consecutive tile rows start 4 banks apart
    if (ctx->k3_tma && i > 0 && cpoisson_tma_fits(box_w, box_h)) {  // TMA-staged tap tiles for the LINEAR passes, where the tiles fit
      CPoissonTmaArgs t{};
      t.a = a;
      t.box_w = box_w;
      t.box_h = box_h;
      if (encode_texel_map(&t.map_in, a.in.p, W, H, (size_t)a.in.pitch, t.box_w, t.box_h) && encode_texel_map(&t.map_nrdz, a.nrdz.p, W, H, (size_t)a.nrdz.pitch, t.box_w, t.box_h)) {
        LAUNCHED(launch_cpoisson_tma(t, cs));
        continue;
      }
    }
    LAUNCHED(launch_cpoisson(a, cs));
  }
  // ---- K4 stand-alone (no Poisson pass to ride on, or the caller split the frame between the last pass and K4)
  k = k_compose;
  if (on(k) && (n_pass == 0 || !on(k - 1))) {
    CComposeArgs a{};
    const Rows kr = launch_rows(ranges, k, H);
    a.row0 = kr.r0; a.row1 = kr.r1;
    if ((st = decode(a.row0, a.row1)) != RFX_OK) return st;
    a.nrdz = ipv(ch->nrdz, W, H); a.gb = gb; a.dn = rpv(ch->fdnB.buf[cur]);
    a.composed = rov(ch->composed.buf[cur]);
    a.composed_carry = ch->composed.view[prev];
    a.W = W; a.H = H; a.cam = cam;
    if (fused_stage && (st = stage_args(ch, f, ch->image[cur], a.k5)) != RFX_OK) return st;
    SpanGuard g(ch, cs, 4);
    LAUNCHED(launch_ccompose(a, cs));
  }
  if (ch->compose_on && !fused_stage && on(k) && (st = chain_render_stage(ch, stream, f, &ch->composed.buf[cur], &ch->image[cur], launch_rows(ranges, k, H))) != RFX_OK)
    return st;
  // ---- TRAA tail (reads this frame's `composed`, so it runs before the planes change parity)
  if (ch->tail.on && on(k_compose + 1) && (st = chain_render_tail(ch, stream, f, &ch->composed.buf[cur], ranges, k_compose + 1)) != RFX_OK) return st;
  if (on(ch->tail.on ? k_compose + 1 : k_compose)) ch->frame_idx++;  // the frame is complete: its planes become `prev`
  return RFX_OK;
}

// One frame of the chain.  `ranges` == nullptr: whole planes.  Otherwise ranges[2k], ranges[2k+1] = output rows [a,b) of launch k
// (chain order: K1, K2, K3 pass 0..2*iterations-1, K4, the TRAA tail) of this rank's band, widened by the halos the next launches
// recompute locally (rfx_shard_ranges).  Only launches k in [k_begin, k_end) are issued, so a caller can wait between two
// launches of a frame (rfx_ssgi_chain_submit_host waits before K4); per-frame state advances with the launch that consumes it.
static rfx_status chain_render_impl(rfx_ssgi_chain* ch, void* stream, const rfx_ssgi_frame* f, const uint32_t* ranges, uint32_t k_begin, uint32_t k_end) {
  if ((ch->tail.on || ch->compose_on) && !f->direct_light)
    return fail(ch->ctx, RFX_ERR_INVALID_ARG, "chain: the TRAA tail and the compose stage compose over the direct light plane (the composer input buffer): it may not be NULL");
  if (ch->fastpath) return chain_render_fast(ch, stream, f, ranges, k_begin, k_end);
  rfx_ctx* ctx = ch->ctx;
  const rfx_ssgi_chain_options& o = ch->opt;
  rfx_status st = RFX_OK;
  const bool dm_full = o.denoise_mode == RFX_DENOISE_FULL;
  if (ranges && ch->ssgi_out.height != o.height) return fail(ctx, RFX_ERR_UNSUPPORTED, "chain: row-range rendering is implemented for resolution_scale 1 only");
  // launches: K1, K2, K3 passes, K4 (both modes: DenoiserComposePass runs for inputType specular too), then the TRAA tail when it is on
  const int H = (int)o.height;
  // what SSGIPass samples as accumulatedTexture = denoiser.texture (Denoiser.js:67-78): the compose target, or the temporal pass's first texture
  HistPlane& accumulated = o.denoise_mode == RFX_DENOISE_TEMPORAL ? ch->tr[0] : ch->composed;
  // Alone the chain renders its planes in place.  In a row-sharded group of n > 1 (rfx_group.inl) the frame reads last frame's
  // buffer `rd` of every plane it keeps, on the rank that owns each row, and writes buffer `wr`; the peer and carry instantiations
  // are chosen for every launch of such a frame, and never otherwise.
  const bool peer = ch->group_peer;
  const int rd = pass_latest(ch), wr = peer ? rd ^ 1 : rd;
  auto carry2 = [&](const HistPlane& p0, const HistPlane& p1) { PeerCarry c{}; c.p[0] = p0.view[rd]; c.p[1] = p1.view[rd]; return c; };
  auto on = [&](uint32_t k) { return k >= k_begin && k < k_end; };
  const cudaStream_t cs = stream ? (cudaStream_t)stream : ctx->stream;
  uint32_t k = 0;
  // ---- K1  SSGIPass.render (src/ssgi/pass/SSGIPass.js:68-95)
  if (on(k)) {
    const rfx_ssgi_params sp = trace_params(ch, f);
    const Rows kr = launch_rows(ranges, k, (int)ch->ssgi_out.height);
    {
      SpanGuard g(ch, cs, 0);  // velocityTexture is a null sampler in the shipped wiring (SURVEY.md D4)
      st = ssgi_trace(ctx, stream, &sp, f->depth, f->gbuffer, nullptr, f->direct_light, &accumulated.buf[rd], &ch->ssgi_out, kr.r0, kr.r1,
                      &accumulated.view[rd]);
    }
    if (st != RFX_OK) return st;
  }
  k++;
  // ---- K2  TemporalReprojectPass.render (TemporalReprojectPass.js:162-214), options from Denoiser.js:26-43 + SSGIEffect.js:74-77
  const int tc = o.mode == RFX_MODE_SSGI ? 2 : 1;
  if (on(k)) {
    rfx_temporal_params tp{};
    tp.cam = f->cam;
    prev_camera_init(ch, f);
    memcpy(tp.prev_view_matrix, ch->prev_view, 64); memcpy(tp.prev_camera_matrix_world, ch->prev_world, 64);
    memcpy(tp.prev_projection, ch->prev_proj, 64); memcpy(tp.prev_projection_inverse, ch->prev_proj_inv, 64);
    memcpy(tp.camera_pos, f->camera_pos, 12); memcpy(tp.prev_camera_pos, ch->prev_pos, 12);
    tp.max_blend = 1.0f; tp.neighborhood_clamp_intensity = 0.5f; tp.keep_data = ch->keep_data; tp.confidence_power = 0.75f;
    tp.full_accumulate = f->camera_moved ? 0 : 1;  // options.fullAccumulate && !didCameraMove
    tp.log_transform = 1; tp.history_linear = 1;
    if (o.mode == RFX_MODE_SSGI) { tp.texture_count = 2; tp.input_type = RFX_INPUT_DIFFUSE_SPECULAR; tp.reproject_specular[0] = 0; tp.reproject_specular[1] = 1; }
    else { tp.texture_count = 1; tp.input_type = RFX_INPUT_SPECULAR; tp.reproject_specular[0] = 1; tp.reproject_specular[1] = 1; }
    {
      const Rows kr = launch_rows(ranges, k, H);
      SpanGuard g(ch, cs, 1);
      // without a denoise pass overrideAccumulatedTextures stays empty: BOTH accumulated textures are the one FramebufferTexture
      rfx_plane* h0 = dm_full ? &ch->dnB[0].buf[rd] : &ch->fb;
      rfx_plane* h1 = dm_full ? &ch->dnB[1].buf[rd] : &ch->fb;
      TemporalPeer tpeer{};
      if (peer) {  // last frame's dnB, or last frame's tr[0] (of which `fb` is a byte copy on one GPU), on the owners; tr carried
        HistPlane& p0 = dm_full ? ch->dnB[0] : ch->tr[0];
        HistPlane& p1 = tc == 2 && dm_full ? ch->dnB[1] : p0;
        h0 = &p0.buf[rd]; h1 = &p1.buf[rd];
        tpeer.hist0 = p0.view[rd]; tpeer.hist1 = p1.view[rd];
        tpeer.carry = carry2(ch->tr[0], ch->tr[tc - 1]);
      }
      const rfx_plane* out1 = tc == 2 ? &ch->tr[1].buf[wr] : nullptr;
      st = temporal_reproject(ctx, stream, &tp, &ch->ssgi_out, f->velocity, h0, tc == 2 ? h1 : nullptr, &ch->tr[0].buf[wr], out1, kr.r0, kr.r1,
                              peer ? &tpeer : nullptr);
    }
    if (st != RFX_OK) return st;
    // renderer.copyFramebufferToTexture(tmpVec2, this.framebufferTexture) after the draw (:197-200).  In a group the next frame reads
    // this frame's tr[0] buffer on its owners instead.
    const rfx_plane& t0 = ch->tr[0].buf[wr];
    if (!dm_full && !peer) CU(cudaMemcpy2DAsync(ch->fb.ptr, ch->fb.pitch, t0.ptr, t0.pitch, (size_t)t0.width * 16, t0.height, cudaMemcpyDeviceToDevice, cs));
    prev_camera_roll(ch, f);
  }
  k++;
  // ---- K3  PoissonDenoisePass.render (PoissonDenoisePass.js:135-149)
  rfx_poisson_params pp{};
  pp.radius = o.radius; pp.phi = o.phi; pp.luma_phi = o.luma_phi; pp.depth_phi = o.depth_phi; pp.normal_phi = o.normal_phi;
  pp.roughness_phi = o.roughness_phi; pp.specular_phi = o.specular_phi;
  pp.texture_count = tc; pp.gbuffer_texture = 1;
  if (o.mode == RFX_MODE_SSGI) { pp.is_texture_specular[0] = 0; pp.is_texture_specular[1] = 1; } else { pp.is_texture_specular[0] = 1; pp.is_texture_specular[1] = 1; }
  bool decoded = false;
  for (int i = 0; i < 2 * o.denoise_iterations; i++, k++) {
    if (!on(k) || !dm_full) continue;  // "full_temporal" / "temporal": no denoise pass (Denoiser.js:47-52)
    const bool horizontal = (i % 2) == 0;
    HistPlane* inp = i == 0 ? ch->tr : (horizontal ? ch->dnB : ch->dnA);
    HistPlane* outp = horizontal ? ch->dnA : ch->dnB;
    pp.input_linear = i == 0 ? 0 : 1;
    pp.blue_noise_index = next_blue(o.blue_noise_start, ch->bn_poisson);
    {
      const Rows kr = launch_rows(ranges, k, H);
      SpanGuard g(ch, cs, i == 0 ? 2 : 3);
      // the G-buffer does not change within a frame: decode it once, reuse it afterwards
      const PeerCarry pc = carry2(outp[0], outp[1]);  // the target's planes of last frame
      st = poisson_denoise(ctx, stream, &pp, f->depth, f->gbuffer, &inp[0].buf[wr], tc == 2 ? &inp[1].buf[wr] : nullptr, &outp[0].buf[wr],
                           tc == 2 ? &outp[1].buf[wr] : nullptr, kr.r0, kr.r1, decoded, peer ? &pc : nullptr);
      decoded = true;
    }
    if (st != RFX_OK) return st;
  }
  // ---- K4  DenoiserComposePass.render ("full" and "full_temporal": Denoiser.js:55-64)
  const HistPlane* gi = dm_full ? ch->dnB : ch->tr;  // composerInputTextures = denoisePass?.texture ?? the temporal textures
  if (on(k) && o.denoise_mode != RFX_DENOISE_TEMPORAL) {
    rfx_compose_params cp{};
    cp.cam = f->cam;
    cp.input_type = o.mode == RFX_MODE_SSGI ? RFX_INPUT_DIFFUSE_SPECULAR : RFX_INPUT_SPECULAR;  // SSGIEffect.js:70-77
    {
      const Rows kr = launch_rows(ranges, k, H);
      SpanGuard g(ch, cs, 4);
      const PeerPV* cc = peer ? &ch->composed.view[rd] : nullptr;  // last frame's `composed`
      rfx_plane* out = &ch->composed.buf[wr];
      if (o.mode == RFX_MODE_SSGI) st = gi_compose(ctx, stream, &cp, f->depth, f->gbuffer, &gi[0].buf[wr], &gi[1].buf[wr], nullptr, out, kr.r0, kr.r1, cc);
      else st = gi_compose(ctx, stream, &cp, f->depth, f->gbuffer, nullptr, &gi[0].buf[wr], f->direct_light, out, kr.r0, kr.r1, cc);  // scene = the composer input buffer (Denoiser.js:100-102)
    }
    if (st != RFX_OK) return st;
  }
  // ---- the compose stage over output 0 (`composed`, or the temporal texture in denoiseMode "temporal", which K2 wrote)
  if (ch->compose_on && on(k) && (st = chain_render_stage(ch, stream, f, &accumulated.buf[wr], &ch->image[0], launch_rows(ranges, k, H))) != RFX_OK) return st;
  k++;
  // ---- TRAA tail over the effect's output (`composed`, or the temporal texture in denoiseMode "temporal")
  if (ch->tail.on && on(k)) return chain_render_tail(ch, stream, f, &accumulated.buf[wr], ranges, k);
  return RFX_OK;
}

rfx_status rfx_ssgi_chain_render(rfx_ssgi_chain* ch, void* stream, const rfx_ssgi_frame* f) {
  if (!ch || !f) return RFX_ERR_INVALID_ARG;
  return chain_render_impl(ch, stream, f, nullptr, 0, 0xffffffffu);
}

// Host-buffer path.  submit enqueues one frame and returns: the four input planes go H2D on a copy stream into staging set
// (frame & 1), the chain runs on the context stream once that upload's event fires, and `composed` and / or the frame's image go D2H
// on a third stream once the frame's last kernel is done.  Frame i+1 therefore uploads (and frame i-1 downloads) while frame i renders;
// PCIe is full duplex, so steady-state time per frame is max(H2D, kernels, D2H) instead of their sum.  Hazards, all resolved on the
// device:
//   staging set reuse   - the upload of frame i+2 waits for frame i's kernels (ev_rendered);
//   downloaded planes   - fast chain: `composed` and the compose stage's image (output 9) are double-buffered by frame parity, and
//                         frame i+2's kernels wait for frame i's D2H (ev_dn); the TRAA tail's image (output 6: K9's, the merged
//                         TRAA + motion-blur pass's or the cosmetic stage's plane) is single-buffered, so frame i+1's tail waits for
//                         frame i's D2H.  Per-pass chain: every downloaded plane is written by K4, the compose stage or the tail, which
//                         all wait for frame i's D2H (ev_dn); K1 of frame i+1 only reads `composed`.
rfx_status rfx_ssgi_chain_submit_host(rfx_ssgi_chain* ch, const rfx_ssgi_host_frame* hf) {
  if (!ch || !hf || !hf->depth || !hf->gbuffer || !hf->velocity || (!hf->out_composed && !hf->out_color)) return RFX_ERR_INVALID_ARG;
  rfx_ctx* ctx = ch->ctx;
  if (hf->out_color && !ch->compose_on && !ch->tail.on)
    return fail(ctx, RFX_ERR_NOT_READY, "chain_submit_host: out_color is the compose stage's or the TRAA tail's image, and both are off");
  rfx_status st = RFX_OK;
  HostPipe& hp = ch->host;
  if (!hp.ready) {
    auto alloc = [&](int fmt, rfx_plane* p) { if (st == RFX_OK) st = rfx_plane_alloc(ctx, fmt, ch->opt.width, ch->opt.height, p); };
    for (int i = 0; i < 2; i++) {
      alloc(RFX_FMT_R32F, &ch->in_depth[i]); alloc(RFX_FMT_RGBA32F, &ch->in_gb[i]); alloc(RFX_FMT_RGBA32F, &ch->in_vel[i]); alloc(RFX_FMT_RGBA16F, &ch->in_direct[i]);
    }
    if (st != RFX_OK || (st = host_pipe_init(ctx, hp)) != RFX_OK) return st;
  }
  const int set = hp.set();
  if (hp.submitted >= 2) CU(cudaStreamWaitEvent(hp.s_up, hp.ev_rendered[set], 0));
  if ((st = rfx_plane_upload(ctx, hp.s_up, &ch->in_depth[set], hf->depth, 0)) != RFX_OK) return st;
  if ((st = rfx_plane_upload(ctx, hp.s_up, &ch->in_gb[set], hf->gbuffer, 0)) != RFX_OK) return st;
  if (hf->direct_light && (st = rfx_plane_upload(ctx, hp.s_up, &ch->in_direct[set], hf->direct_light, 0)) != RFX_OK) return st;
  if ((st = rfx_plane_upload(ctx, hp.s_up, &ch->in_vel[set], hf->velocity, 0)) != RFX_OK) return st;
  CU(cudaEventRecord(hp.ev_up[set], hp.s_up));
  CU(cudaStreamWaitEvent(ctx->stream, hp.ev_up[set], 0));
  rfx_ssgi_frame f{};
  f.cam = hf->cam;
  f.depth = &ch->in_depth[set]; f.gbuffer = &ch->in_gb[set]; f.velocity = &ch->in_vel[set]; f.direct_light = hf->direct_light ? &ch->in_direct[set] : nullptr;
  memcpy(f.camera_pos, hf->camera_pos, 12);
  f.camera_moved = hf->camera_moved;
  const rfx_plane* result = &ch->composed.buf[0];
  if (ch->fastpath) {
    // `composed` is double-buffered by frame parity: this frame writes composed.buf[cur], whose previous reader is the D2H of two
    // frames ago (long finished in steady state); frame i-1's D2H keeps running under this frame's kernels
    const int cur = (int)(ch->frame_idx & 1);
    for (int q = 0; q < 2; q++)
      if (ch->dn_buf[q] == cur) CU(cudaStreamWaitEvent(ctx->stream, hp.ev_dn[q], 0));
    // the tail (its launches after K4) writes the single-buffered image: it waits for the previous frame's D2H
    const uint32_t split = ch->tail.on ? 3u + 2u * (uint32_t)ch->opt.denoise_iterations : 0xffffffffu;
    if ((st = chain_render_impl(ch, nullptr, &f, nullptr, 0, split)) != RFX_OK) return st;
    if (ch->tail.on) {
      if (hp.submitted >= 1) CU(cudaStreamWaitEvent(ctx->stream, hp.ev_dn[set ^ 1], 0));
      if ((st = chain_render_impl(ch, nullptr, &f, nullptr, split, 0xffffffffu)) != RFX_OK) return st;
    }
    result = &ch->composed.buf[cur];
    ch->dn_buf[set] = cur;
  } else {
    const uint32_t n_launches = 3u + 2u * (uint32_t)ch->opt.denoise_iterations;
    const uint32_t split = n_launches - 1;  // K4 is the only launch that writes `composed`
    if (split && (st = chain_render_impl(ch, nullptr, &f, nullptr, 0, split)) != RFX_OK) return st;
    if (hp.submitted >= 1) CU(cudaStreamWaitEvent(ctx->stream, hp.ev_dn[set ^ 1], 0));
    if ((st = chain_render_impl(ch, nullptr, &f, nullptr, split, 0xffffffffu)) != RFX_OK) return st;
  }
  rfx_plane image{};  // the frame's image: output 9 with the compose stage, else output 6 (the tail's)
  if (hf->out_color && (st = rfx_ssgi_chain_output(ch, ch->compose_on ? 9 : 6, &image)) != RFX_OK) return st;
  CU(cudaEventRecord(hp.ev_rendered[set], ctx->stream));
  CU(cudaStreamWaitEvent(hp.s_dn, hp.ev_rendered[set], 0));
  if (hf->out_composed && (st = rfx_plane_download(ctx, hp.s_dn, result, hf->out_composed, 0)) != RFX_OK) return st;
  if (hf->out_color && (st = rfx_plane_download(ctx, hp.s_dn, &image, hf->out_color, 0)) != RFX_OK) return st;
  CU(cudaEventRecord(hp.ev_dn[set], hp.s_dn));
  hp.submitted++;
  return RFX_OK;
}

// Blocks until at most `max_in_flight` (0 or 1) of the submitted frames are still incomplete.  A complete frame's out_composed is
// filled and its input buffers may be overwritten.  Frames complete in submission order.
rfx_status rfx_ssgi_chain_wait_host(rfx_ssgi_chain* ch, int32_t max_in_flight) {
  if (!ch || max_in_flight < 0) return RFX_ERR_INVALID_ARG;
  return host_pipe_wait(ch->ctx, ch->host, max_in_flight);
}

// synchronous form: one frame in, its result out
rfx_status rfx_ssgi_chain_render_host(rfx_ssgi_chain* ch, const rfx_ssgi_host_frame* hf) {
  rfx_status st = rfx_ssgi_chain_submit_host(ch, hf);
  return st != RFX_OK ? st : rfx_ssgi_chain_wait_host(ch, 0);
}

}  // extern "C"

// ==========================================================================================
// native AO chain: HBAOEffect.update / HorizonAOEffect.update (K6 or K6h -> K3 x 2*iterations -> K7) in one call
// ==========================================================================================
struct rfx_ao_chain : GroupMember {
  rfx_ao_chain_options opt;
  float luma_phi, depth_phi, normal_phi;  // the denoiser's values: opt's, clamped where a setter changed them (AOEffect.js:106-110)
  // the planes a frame leaves for the next (a discarded pixel keeps its texel): alone single-buffered (buffer 0, rendered in place);
  // buffer 1 is added by a group of n > 1 (group_alloc_history)
  HistPlane target, dnA, dnB;
  int32_t bn_ao = 0, bn_dn = 0;  // the AO pass's and the denoiser's BlueNoiseIndex
  // the TRAA tail (`tail`: K7 into tail.mid, then the TRAA pass and K9 into frame->output) reads the previous frame's camera
  bool traa_have_prev = false;    // traa_prev holds the previous frame's camera
  rfx_ao_traa_frame traa_prev{};
  // host-buffer path (rfx_ao_chain_submit_host): per staging set the input planes and the two planes its D2H reads; each plane is
  // allocated (for both sets) by the first frame that needs it
  HostPipe host;
  rfx_plane in_depth[2]{}, in_vel[2]{}, in_normal[2]{}, in_input[2]{}, out_color[2]{}, out_ao[2]{};
};

static void ao_target_size(const rfx_ao_chain_options& o, uint32_t& w, uint32_t& h, float& rx, float& ry) {
  const double s = o.resolution_scale == 0.0f ? 1.0 : (double)o.resolution_scale;
  const double fw = (double)o.width * s, fh = (double)o.height * s;  // AOEffect.setSize: setSize(width * scale, height * scale)
  w = (uint32_t)fw; h = (uint32_t)fh;
  rx = (float)fw; ry = (float)fh;  // uniform `resolution`: the unrounded product
}

extern "C" {

rfx_status rfx_ao_chain_create(rfx_ctx* ctx, const rfx_ao_chain_options* opt, rfx_ao_chain** out) {
  if (!ctx || !opt || !out || opt->width == 0 || opt->height == 0 || opt->iterations < 0) return fail(ctx, RFX_ERR_INVALID_ARG, "ao_chain_create: bad arguments");
  if (opt->algorithm != RFX_AO_HBAO && opt->algorithm != RFX_AO_HORIZON) return fail(ctx, RFX_ERR_INVALID_ARG, "ao_chain_create: algorithm must be RFX_AO_HBAO or RFX_AO_HORIZON");
  if (opt->resolution_scale != 0.0f && !(opt->resolution_scale > 0.0f && opt->resolution_scale <= 1.0f))
    return fail(ctx, RFX_ERR_INVALID_ARG, "ao_chain_create: resolution_scale must be in (0, 1]");
  uint32_t tw, th;
  float rx, ry;
  ao_target_size(*opt, tw, th, rx, ry);
  if (tw == 0 || th == 0) return fail(ctx, RFX_ERR_INVALID_ARG, "ao_chain_create: resolution_scale leaves an empty AO target");
  CU(cudaSetDevice(ctx->device));
  rfx_ao_chain* ch = new rfx_ao_chain();
  ch->ctx = ctx;
  ch->opt = *opt;
  ch->luma_phi = opt->luma_phi; ch->depth_phi = opt->depth_phi; ch->normal_phi = opt->normal_phi;
  rfx_status st = rfx_plane_alloc(ctx, RFX_FMT_RGBA16F, tw, th, &ch->target.buf[0]);
  for (HistPlane* h : {&ch->dnA, &ch->dnB})
    if (st == RFX_OK) st = rfx_plane_alloc(ctx, RFX_FMT_RGBA16F, opt->width, opt->height, &h->buf[0]);
  if (st != RFX_OK) { rfx_ao_chain_destroy(ch); return st; }
  for (HistPlane* h : {&ch->target, &ch->dnA, &ch->dnB}) local_views(*h);
  *out = ch;
  return RFX_OK;
}

void rfx_ao_chain_destroy(rfx_ao_chain* ch) {
  if (!ch) return;
  cudaStreamSynchronize(ch->ctx->stream);
  host_pipe_destroy(ch->host);
  for (HistPlane* h : {&ch->target, &ch->dnA, &ch->dnB})
    for (rfx_plane& p : h->buf) if (p.ptr) rfx_plane_free(ch->ctx, &p);
  traa_free(ch->ctx, ch->tail);
  for (int i = 0; i < 2; i++)
    for (rfx_plane* p : {&ch->in_depth[i], &ch->in_vel[i], &ch->in_normal[i], &ch->in_input[i], &ch->out_color[i], &ch->out_ao[i]})
      if (p->ptr) rfx_plane_free(ch->ctx, p);
  delete ch;
}

rfx_status rfx_ao_chain_set_options(rfx_ao_chain* ch, const rfx_ao_chain_options* opt) {
  if (!ch || !opt) return RFX_ERR_INVALID_ARG;
  rfx_ctx* ctx = ch->ctx;
  if (opt->width != ch->opt.width || opt->height != ch->opt.height || opt->resolution_scale != ch->opt.resolution_scale)
    return fail(ctx, RFX_ERR_SIZE_MISMATCH, "ao_chain_set_options: width, height and resolution_scale size the planes: create a new chain");
  if (opt->algorithm != ch->opt.algorithm) return fail(ctx, RFX_ERR_UNSUPPORTED, "ao_chain_set_options: the algorithm is a constructor option: create a new chain");
  if (opt->iterations < 0) return fail(ctx, RFX_ERR_INVALID_ARG, "ao_chain_set_options: iterations < 0");
  if (opt->luma_phi != ch->opt.luma_phi) ch->luma_phi = std::max(opt->luma_phi, 0.0001f);
  if (opt->depth_phi != ch->opt.depth_phi) ch->depth_phi = std::max(opt->depth_phi, 0.0001f);
  if (opt->normal_phi != ch->opt.normal_phi) ch->normal_phi = std::max(opt->normal_phi, 0.0001f);
  const int32_t s0 = ch->opt.blue_noise_start, s1 = ch->opt.denoise_blue_noise_start;
  ch->opt = *opt;
  ch->opt.blue_noise_start = s0;  // the counters keep their start index for the life of the effect
  ch->opt.denoise_blue_noise_start = s1;
  return RFX_OK;
}

rfx_status rfx_ao_chain_reset(rfx_ao_chain* ch) {
  if (!ch) return RFX_ERR_INVALID_ARG;
  rfx_ctx* ctx = ch->ctx;
  for (HistPlane* h : {&ch->target, &ch->dnA, &ch->dnB, &ch->tail.acc})
    for (const rfx_plane& p : h->buf)
      if (p.ptr) CU(cudaMemset2DAsync(p.ptr, p.pitch, 0, (size_t)p.width * 8, p.height, ctx->stream));
  ch->bn_ao = ch->bn_dn = 0;
  ch->luma_phi = ch->opt.luma_phi; ch->depth_phi = ch->opt.depth_phi; ch->normal_phi = ch->opt.normal_phi;
  ch->tail.keep = 0.0f;  // a new TRAA pass: keepData 0, and the first frame's previous camera is its own
  ch->traa_have_prev = false;
  return RFX_OK;
}

rfx_status rfx_ao_chain_enable_traa(rfx_ao_chain* ch, const rfx_traa_tail_options* opt) {
  if (!ch) return RFX_ERR_INVALID_ARG;
  rfx_ctx* ctx = ch->ctx;
  if (ch->group && rfx_group_world(ch->group) > 1)
    return fail(ctx, RFX_ERR_UNSUPPORTED, "ao_chain_enable_traa: the chain is in a row-sharded group, whose peer mappings are fixed at attach time");
  static const rfx_ssgi_compose_params no_compose{};
  if (opt && memcmp(&opt->compose, &no_compose, sizeof no_compose) != 0)
    return fail(ctx, RFX_ERR_INVALID_ARG, "ao_chain_enable_traa: the AO tail has no K5: `compose` must be all zero");
  return traa_enable(ctx, ch->tail, opt, ch->opt.width, ch->opt.height, false);
}

rfx_status rfx_ao_chain_set_motion_blur(rfx_ao_chain* ch, const rfx_motion_blur_params* p) {
  if (!ch) return RFX_ERR_INVALID_ARG;
  return traa_set_blur(ch->ctx, ch->tail, p, ch->group && rfx_group_world(ch->group) > 1);
}

rfx_status rfx_ao_chain_set_effects(rfx_ao_chain* ch, const rfx_effects_params* p) {
  if (!ch) return RFX_ERR_INVALID_ARG;
  return traa_set_fx(ch->ctx, ch->tail, p, ch->opt.width, ch->opt.height);
}

rfx_status rfx_ao_chain_output(rfx_ao_chain* ch, int32_t which, rfx_plane* out) {
  if (!ch || !out) return RFX_ERR_INVALID_ARG;
  if (ch->tail.on && (which == 2 || which == 3)) {
    *out = which == 2 ? ch->tail.mid_latest() : ch->tail.latest();
    return RFX_OK;
  }
  if (which == 4) {
    if (!ch->tail.fx) return fail(ch->ctx, RFX_ERR_NOT_READY, "ao_chain_output: output 4 needs the cosmetic stage (rfx_ao_chain_set_effects)");
    *out = ch->tail.fx_plane;
    return RFX_OK;
  }
  if (which < 0 || which > 1) return fail(ch->ctx, RFX_ERR_INVALID_ARG, "ao_chain_output: which must be 0 or 1 (2 / 3 with the TRAA tail on, 4 with the cosmetic stage)");
  const HistPlane& h = which == 1 && ch->opt.iterations > 0 ? ch->dnB : ch->target;  // AOEffect's `texture`
  *out = h.buf[h.buf[1].ptr ? pass_latest(ch) : 0];
  return RFX_OK;
}

}  // extern "C"

// One frame of the AO chain.  `ranges` == nullptr: whole planes.  Otherwise ranges[2k], ranges[2k+1] = output rows [a,b) of launch k
// (K6 / K6h, K3 pass 0..2*iterations-1, K7[, the TRAA tail]) of this rank's band, widened by the halos the next launches recompute
// (rfx_ao_shard_ranges).  `t`: the TRAA tail's camera, given exactly when the tail is on (the entry points check it).
static rfx_status ao_render_impl(rfx_ao_chain* ch, void* stream, const rfx_ao_frame* f, const uint32_t* ranges, const rfx_ao_traa_frame* t) {
  rfx_ctx* ctx = ch->ctx;
  const rfx_ao_chain_options& o = ch->opt;
  if (!f->depth || !f->velocity) return fail(ctx, RFX_ERR_INVALID_ARG, "ao_chain: depth and velocity are required");
  if (o.use_normal_plane && !f->normal) return fail(ctx, RFX_ERR_INVALID_ARG, "ao_chain: use_normal_plane needs frame->normal (RGBA8 view-space normals)");
  if (f->output && !f->input) return fail(ctx, RFX_ERR_INVALID_ARG, "ao_chain: K7 composes over frame->input: it may not be NULL with an output");
  if (t && !f->output) return fail(ctx, RFX_ERR_INVALID_ARG, "ao_chain: the TRAA tail renders into frame->output: it may not be NULL");
  if (f->depth->width != o.width || f->depth->height != o.height) return fail(ctx, RFX_ERR_SIZE_MISMATCH, "ao_chain: the depth plane must have the chain's size");
  const rfx_plane* normal = o.use_normal_plane ? f->normal : nullptr;
  // Alone the chain renders in place.  In a row-sharded group of n > 1 (rfx_group.inl) it writes buffer `wr` and a discarded pixel
  // carries last frame's texel (buffer `rd`) from the rank that owns the row.
  const bool peer = ch->group_peer;
  const int rd = pass_latest(ch), wr = peer ? rd ^ 1 : rd;
  uint32_t k = 0;
  rfx_status st;
  {  // ---- K6 / K6h  AOPass.render (src/ao/AOPass.js:86-110)
    uint32_t tw, th;
    float rx, ry;
    ao_target_size(o, tw, th, rx, ry);
    const Rows kr = launch_rows(ranges, k, (int)th);
    const PeerPV* carry = peer ? &ch->target.view[rd] : nullptr;
    if (o.algorithm == RFX_AO_HBAO) {
      rfx_hbao_params p{};
      for (int c = 0; c < 4; c++)  // projectionMatrix * matrixWorldInverse in float64, rounded to fp32 (AOPass.js:93-96)
        for (int r = 0; r < 4; r++) {
          double acc = 0.0;
          for (int i = 0; i < 4; i++) acc += (double)f->projection[i * 4 + r] * (double)f->view_matrix[c * 4 + i];
          p.projection_view[c * 4 + r] = (float)acc;
        }
      memcpy(p.projection_inverse, f->projection_inverse, 64);
      memcpy(p.camera_matrix_world, f->camera_matrix_world, 64);
      memcpy(p.view_matrix, f->view_matrix, 64);
      p.resolution[0] = rx; p.resolution[1] = ry;
      p.ao_distance = o.distance; p.distance_power = o.distance_power; p.bias = o.bias; p.thickness = o.thickness; p.spp = o.spp;
      p.blue_noise_index = next_blue(o.blue_noise_start, ch->bn_ao);
      st = hbao(ctx, stream, &p, f->depth, normal, &ch->target.buf[wr], (uint32_t)kr.r0, (uint32_t)kr.r1, carry);
    } else {
      rfx_hbao_horizon_params p{};
      memcpy(p.projection, f->projection, 64);
      memcpy(p.projection_inverse, f->projection_inverse, 64);
      memcpy(p.camera_matrix_world, f->camera_matrix_world, 64);
      memcpy(p.view_matrix, f->view_matrix, 64);
      p.resolution[0] = rx; p.resolution[1] = ry;
      p.distance = o.distance; p.angle_bias = o.angle_bias; p.intensity = o.intensity; p.max_radius_pixels = o.max_radius_pixels;
      p.directions = o.directions; p.steps = o.steps;
      p.blue_noise_index = next_blue(o.blue_noise_start, ch->bn_ao);
      st = hbao_horizon(ctx, stream, &p, f->depth, &ch->target.buf[wr], normal, (uint32_t)kr.r0, (uint32_t)kr.r1, carry);
    }
    if (st != RFX_OK) return st;
  }
  k++;
  // ---- K3  PoissonDenoisePass.render with AOEffect's options: one plane, velocity-layout normals, LINEAR input (the RGBA16F AO target)
  rfx_poisson_params pp{};
  pp.radius = o.radius; pp.phi = o.phi; pp.luma_phi = ch->luma_phi; pp.depth_phi = ch->depth_phi; pp.normal_phi = ch->normal_phi;
  pp.texture_count = 1; pp.gbuffer_texture = 0; pp.input_linear = 1;
  bool decoded = false;
  for (int i = 0; i < 2 * o.iterations; i++, k++) {
    const bool horizontal = (i % 2) == 0;
    HistPlane& inp = i == 0 ? ch->target : (horizontal ? ch->dnB : ch->dnA);
    HistPlane& outp = horizontal ? ch->dnA : ch->dnB;
    pp.blue_noise_index = next_blue(o.denoise_blue_noise_start, ch->bn_dn);
    const Rows kr = launch_rows(ranges, k, (int)o.height);
    PeerCarry pc{};
    pc.p[0] = outp.view[rd];  // the target's plane of last frame
    st = poisson_denoise(ctx, stream, &pp, f->depth, f->velocity, &inp.buf[wr], nullptr, &outp.buf[wr], nullptr, kr.r0, kr.r1, decoded, peer ? &pc : nullptr);
    if (st != RFX_OK) return st;
    decoded = true;  // the velocity plane does not change within a frame; the first pass's rows are the widest
  }
  // ---- K7  ao_compose.frag over AOEffect's `texture` (with the TRAA tail: into the composer buffer the TRAA EffectPass reads)
  if (f->output) {
    rfx_ao_compose_params cp{};
    cp.power = o.power;
    memcpy(cp.color, o.color, 12);
    const Rows kr = launch_rows(ranges, k, (int)o.height);
    const HistPlane& tex = o.iterations > 0 ? ch->dnB : ch->target;
    st = ao_compose(ctx, stream, &cp, f->depth, &tex.buf[wr], f->input, t ? &ch->tail.mid_w() : f->output, (uint32_t)kr.r0, (uint32_t)kr.r1);
    if (st != RFX_OK) return st;
  }
  k++;
  // ---- the TRAA tail: TRAAEffect's temporal pass over the K7 plane, then K9 into frame->output (with the cosmetic stage on: K9 into the
  // stage's plane, then the stage into frame->output on launch k + 1's rows, the band)
  if (t) {
    const rfx_plane* tail_out = f->output;
    if (ch->tail.fx) {
      const Rows fr = launch_rows(ranges, k + 1, (int)o.height);
      ch->tail.fx_job = {ch->tail.fx_plane, *f->depth, *f->velocity, *f->output, fr.r0, fr.r1};
      tail_out = &ch->tail.fx_plane;
    }
    rfx_temporal_params cam{};
    const rfx_ao_traa_frame& prev = ch->traa_have_prev ? ch->traa_prev : *t;  // TemporalReprojectPass.js:94-97 on the first frame
    cam.cam = t->cam;
    memcpy(cam.prev_view_matrix, prev.cam.view_matrix, 64); memcpy(cam.prev_camera_matrix_world, prev.cam.camera_matrix_world, 64);
    memcpy(cam.prev_projection, prev.cam.projection, 64); memcpy(cam.prev_projection_inverse, prev.cam.projection_inverse, 64);
    memcpy(cam.camera_pos, t->camera_pos, 12); memcpy(cam.prev_camera_pos, prev.camera_pos, 12);
    st = traa_launches(ctx, stream, traa_params(ch->tail, cam, t->camera_moved), ch->tail, f->velocity, ch->group_peer, tail_out,
                       launch_rows(ranges, k, (int)o.height));
    if (st != RFX_OK) return st;
    ch->traa_prev = *t;
    ch->traa_have_prev = true;
  }
  return RFX_OK;
}

// The entry points: the tail's camera is given exactly when the tail is on.
static rfx_status ao_check_traa(rfx_ao_chain* ch, const rfx_ao_traa_frame* t, const char* who) {
  if (ch->tail.on && !t) return fail(ch->ctx, RFX_ERR_INVALID_ARG, "%s: the TRAA tail is on and needs the camera (render with the _traa entry point)", who);
  if (!ch->tail.on && t) return fail(ch->ctx, RFX_ERR_NOT_READY, "%s: the TRAA tail is off (rfx_ao_chain_enable_traa)", who);
  return RFX_OK;
}

extern "C" {

rfx_status rfx_ao_chain_render(rfx_ao_chain* ch, void* stream, const rfx_ao_frame* f) {
  if (!ch || !f) return RFX_ERR_INVALID_ARG;
  rfx_status st = ao_check_traa(ch, nullptr, "ao_chain_render");
  return st != RFX_OK ? st : ao_render_impl(ch, stream, f, nullptr, nullptr);
}

rfx_status rfx_ao_chain_render_traa(rfx_ao_chain* ch, void* stream, const rfx_ao_frame* f, const rfx_ao_traa_frame* t) {
  if (!ch || !f || !t) return RFX_ERR_INVALID_ARG;
  rfx_status st = ao_check_traa(ch, t, "ao_chain_render_traa");
  return st != RFX_OK ? st : ao_render_impl(ch, stream, f, nullptr, t);
}

}  // extern "C"

// Host-buffer path: the pipeline of rfx_ssgi_chain_submit_host around ao_render_impl's launches.  Frame i uploads into staging set
// i & 1 on the copy stream, renders on the context stream once ev_up fires, and downloads on the third stream once its kernels are done.
// Hazards, all resolved on the device:
//   staging set reuse - the upload of frame i+2 waits for frame i's kernels (ev_rendered);
//   the downloaded planes - the chain renders its kept planes (AO target, Poisson targets, the tail's K7 and accumulated planes) in place,
//     so frame i+1's kernels overwrite what frame i's D2H would read.  The tail's output and K7's output are frame->output, which here
//     is the set's out_color plane.  Output 1 (Poisson target B, or the AO target) is copied on the context stream into the set's out_ao
//     plane after the frame's kernels: a device copy of W*H*8 bytes, where ordering frame i+1's first writer of that plane after frame
//     i's D2H would serialise the PCIe download with the next frame's kernels.  Both per-set planes are next written by frame i+2,
//     whose kernels wait for frame i's D2H (ev_dn).
static rfx_status ao_host_planes(rfx_ao_chain* ch, const rfx_ao_host_frame* hf) {
  const uint32_t W = ch->opt.width, H = ch->opt.height;
  rfx_status st = RFX_OK;
  auto need = [&](bool used, int fmt, rfx_plane* p) {
    for (int i = 0; i < 2; i++)
      if (used && st == RFX_OK && !p[i].ptr) st = rfx_plane_alloc(ch->ctx, fmt, W, H, &p[i]);
  };
  need(true, RFX_FMT_R32F, ch->in_depth);
  need(true, RFX_FMT_RGBA32F, ch->in_vel);
  need(ch->opt.use_normal_plane != 0, RFX_FMT_RGBA8, ch->in_normal);
  need(hf->input != nullptr, RFX_FMT_RGBA16F, ch->in_input);
  need(hf->input != nullptr, RFX_FMT_RGBA16F, ch->out_color);
  need(hf->out_ao != nullptr, RFX_FMT_RGBA16F, ch->out_ao);  // output 1 is at most W x H (the AO target is smaller with resolution_scale < 1)
  return st != RFX_OK ? st : host_pipe_init(ch->ctx, ch->host);
}

extern "C" {

rfx_status rfx_ao_chain_submit_host(rfx_ao_chain* ch, const rfx_ao_host_frame* hf) {
  if (!ch || !hf) return RFX_ERR_INVALID_ARG;
  rfx_ctx* ctx = ch->ctx;
  if (ch->tail.pending) return fail(ctx, RFX_ERR_NOT_READY, "ao_chain_submit_host: the last row-sharded frame waits for its second phase (render_sharded_finish)");
  if (ch->group && rfx_group_world(ch->group) > 1)
    return fail(ctx, RFX_ERR_UNSUPPORTED, "ao_chain_submit_host: the chain is in a row-sharded group of n > 1, whose ranks upload their own rows (parallel.ShardedAoChain.submit_host)");
  if (!hf->depth || !hf->velocity) return fail(ctx, RFX_ERR_INVALID_ARG, "ao_chain_submit_host: depth and velocity are required");
  if (ch->opt.use_normal_plane && !hf->normal) return fail(ctx, RFX_ERR_INVALID_ARG, "ao_chain_submit_host: use_normal_plane needs the normal plane");
  if ((hf->input != nullptr) != (hf->out_color != nullptr)) return fail(ctx, RFX_ERR_INVALID_ARG, "ao_chain_submit_host: input and out_color go together (K7 composes input into out_color)");
  if (!hf->input && !hf->out_ao) return fail(ctx, RFX_ERR_INVALID_ARG, "ao_chain_submit_host: without input the frame downloads out_ao, which may not be NULL then");
  if (ch->tail.on && !hf->input) return fail(ctx, RFX_ERR_INVALID_ARG, "ao_chain_submit_host: the TRAA tail renders into out_color over input: both are required");
  rfx_status st = ao_check_traa(ch, hf->traa, "ao_chain_submit_host");
  if (st != RFX_OK || (st = ao_host_planes(ch, hf)) != RFX_OK) return st;
  HostPipe& hp = ch->host;
  const int set = hp.set();
  if (hp.submitted >= 2) CU(cudaStreamWaitEvent(hp.s_up, hp.ev_rendered[set], 0));
  if ((st = rfx_plane_upload(ctx, hp.s_up, &ch->in_depth[set], hf->depth, 0)) != RFX_OK) return st;
  if ((st = rfx_plane_upload(ctx, hp.s_up, &ch->in_vel[set], hf->velocity, 0)) != RFX_OK) return st;
  if (ch->opt.use_normal_plane && (st = rfx_plane_upload(ctx, hp.s_up, &ch->in_normal[set], hf->normal, 0)) != RFX_OK) return st;
  if (hf->input && (st = rfx_plane_upload(ctx, hp.s_up, &ch->in_input[set], hf->input, 0)) != RFX_OK) return st;
  CU(cudaEventRecord(hp.ev_up[set], hp.s_up));
  CU(cudaStreamWaitEvent(ctx->stream, hp.ev_up[set], 0));
  if (hp.submitted >= 2) CU(cudaStreamWaitEvent(ctx->stream, hp.ev_dn[set], 0));  // out_color / out_ao of this set: frame i-2's D2H
  rfx_ao_frame f{};
  memcpy(f.projection, hf->projection, 64); memcpy(f.projection_inverse, hf->projection_inverse, 64);
  memcpy(f.camera_matrix_world, hf->camera_matrix_world, 64); memcpy(f.view_matrix, hf->view_matrix, 64);
  f.depth = &ch->in_depth[set]; f.velocity = &ch->in_vel[set];
  f.normal = ch->opt.use_normal_plane ? &ch->in_normal[set] : nullptr;
  f.input = hf->input ? &ch->in_input[set] : nullptr;
  f.output = hf->input ? &ch->out_color[set] : nullptr;
  if ((st = ao_render_impl(ch, nullptr, &f, nullptr, hf->traa)) != RFX_OK) return st;
  rfx_plane ao{};
  if (hf->out_ao) {
    rfx_plane o1{};
    if ((st = rfx_ao_chain_output(ch, 1, &o1)) != RFX_OK) return st;
    ao = ch->out_ao[set];
    ao.width = o1.width; ao.height = o1.height;
    CU(cudaMemcpy2DAsync(ao.ptr, ao.pitch, o1.ptr, o1.pitch, (size_t)o1.width * 8, o1.height, cudaMemcpyDeviceToDevice, ctx->stream));
  }
  CU(cudaEventRecord(hp.ev_rendered[set], ctx->stream));
  CU(cudaStreamWaitEvent(hp.s_dn, hp.ev_rendered[set], 0));
  if (hf->input && (st = rfx_plane_download(ctx, hp.s_dn, &ch->out_color[set], hf->out_color, 0)) != RFX_OK) return st;
  if (hf->out_ao && (st = rfx_plane_download(ctx, hp.s_dn, &ao, hf->out_ao, 0)) != RFX_OK) return st;
  CU(cudaEventRecord(hp.ev_dn[set], hp.s_dn));
  hp.submitted++;
  return RFX_OK;
}

rfx_status rfx_ao_chain_wait_host(rfx_ao_chain* ch, int32_t max_in_flight) {
  if (!ch) return RFX_ERR_INVALID_ARG;
  if (max_in_flight < 0 || max_in_flight > 1) return fail(ch->ctx, RFX_ERR_INVALID_ARG, "ao_chain_wait_host: max_in_flight must be 0 or 1 (two staging sets)");
  return host_pipe_wait(ch->ctx, ch->host, max_in_flight);
}

rfx_status rfx_ao_chain_render_host(rfx_ao_chain* ch, const rfx_ao_host_frame* hf) {
  rfx_status st = rfx_ao_chain_submit_host(ch, hf);
  return st != RFX_OK ? st : rfx_ao_chain_wait_host(ch, 0);
}

}  // extern "C"

#include "rfx_group.inl"
