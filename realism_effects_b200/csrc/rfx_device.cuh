// rfx_device.cuh — device-side vocabulary shared by the sm_90a kernels.
//
// fp32 lowering contract (the kernels are compiled with -fmad=false, so nothing is contracted
// implicitly; the only fused operations are the explicit fma_() below):
//   dot          fma chain, last component outermost
//   mixf(x,y,a)  fma(y, a, x*(1-a))
//   M*v / v*M    fma chain per component, .w term innermost
//   cross        fma(a.y, b.z, -(b.y*a.z)) ...
//   normalize    a * (1/sqrt(dot(a,a)))      (IEEE sqrt + IEEE reciprocal)
//   division / sqrt: IEEE (-prec-div=true -prec-sqrt=true are nvcc defaults)
//   transcendentals of the exact K1 and K2: evaluated in double and rounded once to fp32 (the *cr
//   functions below), as the oracle does.  The fp32 device libm (sinf/cosf/expf/logf/powf/atan2f/
//   acosf/log2f) is 1-2 ulp off the correctly rounded value, and one such ulp that crosses an fp16
//   rounding boundary of K1's packed output changes the output's bits.
// These are the rules the parity oracle states in oracle/glsl.h; keeping them identical makes the
// exact K1 and K2 bit-identical to the oracle; elsewhere parity differences come only from the device libm.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#define RFX_D __device__ __forceinline__

namespace rfx {

struct v2 { float x, y; };
struct v3 { float x, y, z; };
struct v4 { float x, y, z, w; };

RFX_D v2 mk2(float x, float y) { v2 r; r.x = x; r.y = y; return r; }
RFX_D v3 mk3(float x, float y, float z) { v3 r; r.x = x; r.y = y; r.z = z; return r; }
RFX_D v3 mk3(float s) { return mk3(s, s, s); }
RFX_D v4 mk4(float x, float y, float z, float w) { v4 r; r.x = x; r.y = y; r.z = z; r.w = w; return r; }
RFX_D v4 mk4(v3 a, float w) { return mk4(a.x, a.y, a.z, w); }
RFX_D v3 xyz(v4 a) { return mk3(a.x, a.y, a.z); }

#define RFX_OP3(op)                                                               \
  RFX_D v3 operator op(v3 a, v3 b) { return mk3(a.x op b.x, a.y op b.y, a.z op b.z); } \
  RFX_D v3 operator op(v3 a, float s) { return mk3(a.x op s, a.y op s, a.z op s); }     \
  RFX_D v3 operator op(float s, v3 a) { return mk3(s op a.x, s op a.y, s op a.z); }
#define RFX_OP2(op)                                                        \
  RFX_D v2 operator op(v2 a, v2 b) { return mk2(a.x op b.x, a.y op b.y); } \
  RFX_D v2 operator op(v2 a, float s) { return mk2(a.x op s, a.y op s); }  \
  RFX_D v2 operator op(float s, v2 a) { return mk2(s op a.x, s op a.y); }
#define RFX_OP4(op)                                                                              \
  RFX_D v4 operator op(v4 a, v4 b) { return mk4(a.x op b.x, a.y op b.y, a.z op b.z, a.w op b.w); } \
  RFX_D v4 operator op(v4 a, float s) { return mk4(a.x op s, a.y op s, a.z op s, a.w op s); }
RFX_OP2(+) RFX_OP2(-) RFX_OP2(*)
RFX_OP3(+) RFX_OP3(-) RFX_OP3(*)
RFX_OP4(+) RFX_OP4(-) RFX_OP4(*)
// division: vector / vector is component-wise IEEE; vector / SCALAR = one IEEE reciprocal + multiplies (oracle/glsl.h rule)
RFX_D v2 operator/(v2 a, v2 b) { return mk2(a.x / b.x, a.y / b.y); }
RFX_D v3 operator/(v3 a, v3 b) { return mk3(a.x / b.x, a.y / b.y, a.z / b.z); }
RFX_D v2 operator/(v2 a, float s) { const float r = 1.0f / s; return mk2(a.x * r, a.y * r); }
RFX_D v3 operator/(v3 a, float s) { const float r = 1.0f / s; return mk3(a.x * r, a.y * r, a.z * r); }
RFX_D v4 operator/(v4 a, float s) { const float r = 1.0f / s; return mk4(a.x * r, a.y * r, a.z * r, a.w * r); }
RFX_D v3 operator-(v3 a) { return mk3(-a.x, -a.y, -a.z); }

RFX_D float fma_(float a, float b, float c) { return __fmaf_rn(a, b, c); }
RFX_D float dot(v2 a, v2 b) { return fma_(a.y, b.y, a.x * b.x); }
RFX_D float dot(v3 a, v3 b) { return fma_(a.z, b.z, fma_(a.y, b.y, a.x * b.x)); }
RFX_D float length(v2 a) { return sqrtf(dot(a, a)); }
RFX_D float length(v3 a) { return sqrtf(dot(a, a)); }
RFX_D v3 normalize(v3 a) { return a * (1.0f / sqrtf(dot(a, a))); }
RFX_D v3 cross(v3 a, v3 b) {
  return mk3(fma_(a.y, b.z, -(b.y * a.z)), fma_(a.z, b.x, -(b.z * a.x)), fma_(a.x, b.y, -(b.x * a.y)));
}
RFX_D v3 reflect(v3 I, v3 N) {
  float k = 2.0f * dot(N, I);
  return mk3(fma_(-k, N.x, I.x), fma_(-k, N.y, I.y), fma_(-k, N.z, I.z));
}
RFX_D float clampf(float x, float lo, float hi) { return fminf(fmaxf(x, lo), hi); }
RFX_D float mixf(float x, float y, float a) { return fma_(y, a, x * (1.0f - a)); }
RFX_D v3 mix(v3 x, v3 y, float a) { return mk3(mixf(x.x, y.x, a), mixf(x.y, y.y, a), mixf(x.z, y.z, a)); }
RFX_D v2 mix(v2 x, v2 y, float a) { return mk2(mixf(x.x, y.x, a), mixf(x.y, y.y, a)); }
RFX_D float smoothstepf(float e0, float e1, float x) {
  float t = clampf((x - e0) / (e1 - e0), 0.0f, 1.0f);
  return t * t * (3.0f - 2.0f * t);
}
RFX_D v3 vmin(v3 a, v3 b) { return mk3(fminf(a.x, b.x), fminf(a.y, b.y), fminf(a.z, b.z)); }
RFX_D v3 vmax(v3 a, v3 b) { return mk3(fmaxf(a.x, b.x), fmaxf(a.y, b.y), fmaxf(a.z, b.z)); }
RFX_D v3 vabs(v3 a) { return mk3(fabsf(a.x), fabsf(a.y), fabsf(a.z)); }
// correctly rounded fp32 transcendentals (oracle/glsl.h): the double result is within 1-2 double ulps, so rounding it to fp32
// gives the correctly rounded value except where that value sits within ~1e-16 relative of an fp32 rounding midpoint
RFX_D float sincr(float x) { return (float)sin((double)x); }
RFX_D float coscr(float x) { return (float)cos((double)x); }
RFX_D float expcr(float x) { return (float)exp((double)x); }
RFX_D float logcr(float x) { return (float)log((double)x); }
RFX_D float log2cr(float x) { return (float)log2((double)x); }
RFX_D float powcr(float x, float y) { return (float)pow((double)x, (double)y); }
RFX_D float atan2cr(float y, float x) { return (float)atan2((double)y, (double)x); }
RFX_D float acoscr(float x) { return (float)acos((double)x); }

// ---- mat4 (column-major float[16]; M[col*4+row]) ----------------------------------------
struct M4 { float m[16]; };
RFX_D v4 mul(const M4& M, v4 v) {  // M * v
  v4 r;
  r.x = fma_(M.m[0], v.x, fma_(M.m[4], v.y, fma_(M.m[8], v.z, M.m[12] * v.w)));
  r.y = fma_(M.m[1], v.x, fma_(M.m[5], v.y, fma_(M.m[9], v.z, M.m[13] * v.w)));
  r.z = fma_(M.m[2], v.x, fma_(M.m[6], v.y, fma_(M.m[10], v.z, M.m[14] * v.w)));
  r.w = fma_(M.m[3], v.x, fma_(M.m[7], v.y, fma_(M.m[11], v.z, M.m[15] * v.w)));
  return r;
}
RFX_D v4 mul(v4 v, const M4& M) {  // v * M == transpose(M) * v
  v4 r;
  r.x = fma_(v.x, M.m[0], fma_(v.y, M.m[1], fma_(v.z, M.m[2], v.w * M.m[3])));
  r.y = fma_(v.x, M.m[4], fma_(v.y, M.m[5], fma_(v.z, M.m[6], v.w * M.m[7])));
  r.z = fma_(v.x, M.m[8], fma_(v.y, M.m[9], fma_(v.z, M.m[10], v.w * M.m[11])));
  r.w = fma_(v.x, M.m[12], fma_(v.y, M.m[13], fma_(v.z, M.m[14], v.w * M.m[15])));
  return r;
}
// (vec4(d, 0.) * M).xyz — bit-identical to mul(mk4(d,0),M) (the w term is an exact zero)
RFX_D v3 mul_dir_left(v3 d, const M4& M) {
  return mk3(fma_(d.x, M.m[0], fma_(d.y, M.m[1], fma_(d.z, M.m[2], 0.0f * M.m[3]))),
             fma_(d.x, M.m[4], fma_(d.y, M.m[5], fma_(d.z, M.m[6], 0.0f * M.m[7]))),
             fma_(d.x, M.m[8], fma_(d.y, M.m[9], fma_(d.z, M.m[10], 0.0f * M.m[11]))));
}

// ---- half / packing ----------------------------------------------------------------------
RFX_D uint32_t packHalf2x16(float a, float b) {
  return (uint32_t)__half_as_ushort(__float2half_rn(a)) | ((uint32_t)__half_as_ushort(__float2half_rn(b)) << 16);
}
RFX_D v2 unpackHalf2x16(uint32_t u) {
  return mk2(__half2float(__ushort_as_half((unsigned short)(u & 0xffffu))), __half2float(__ushort_as_half((unsigned short)(u >> 16))));
}

// gbuffer_packing.glsl (reference src/gbuffer/shader/gbuffer_packing.glsl)
#define RFX_NON_ZERO_OFFSET 0.0001f
RFX_D v3 decodeOctWrap(v2 f) {  // :52-59
  f = f * 2.0f - 1.0f;
  v3 n = mk3(f.x, f.y, 1.0f - fabsf(f.x) - fabsf(f.y));
  float t = fmaxf(-n.z, 0.0f);
  n.x += n.x >= 0.0f ? -t : t;
  n.y += n.y >= 0.0f ? -t : t;
  return normalize(n);
}
RFX_D v3 unpackNormal(float packed) { return decodeOctWrap(unpackHalf2x16(__float_as_uint(packed))); }  // :63
RFX_D v4 floatToVec4(float f) {  // :151-164
  uint32_t v = __float_as_uint(f);
  v4 r = mk4((float)(v & 0xFFu) / 255.0f, (float)((v >> 8) & 0xFFu) / 255.0f, (float)((v >> 16) & 0xFFu) / 255.0f,
             (float)((v >> 24) & 0xFFu) / 255.0f);
  r.x = fmaxf(r.x - RFX_NON_ZERO_OFFSET, 0.0f); r.y = fmaxf(r.y - RFX_NON_ZERO_OFFSET, 0.0f);
  r.z = fmaxf(r.z - RFX_NON_ZERO_OFFSET, 0.0f); r.w = fmaxf(r.w - RFX_NON_ZERO_OFFSET, 0.0f);
  return r;
}
// The byte-field decodes feed floor(): they keep IEEE division (__fdiv_rn) even in a TU built with -prec-div=false, where an
// approximate quotient one ulp below an integer would land in the wrong field.
RFX_D float mod_gl(float x, float y) { return x - y * floorf(__fdiv_rn(x, y)); }
// float2color(...).r / .g  = roughness / metalness  (:24-34,189-191)
RFX_D float gb_roughness(float b) { return fmaxf(mod_gl(b, 257.0f) / 256.0f - RFX_NON_ZERO_OFFSET, 0.0f); }
RFX_D float gb_metalness(float b) { return fmaxf(floorf(__fdiv_rn(b, 257.0f * 257.0f)) / 256.0f - RFX_NON_ZERO_OFFSET, 0.0f); }
// EXACT_EXP2: exp2 rounded from double, as the oracle's exp2cr (oracle/glsl.h).  fExp is never an integer (floatToVec4 subtracts 1e-4),
// where exp2f may be 2 ulp off; the G-buffer debug view shows the decoded value itself and takes the exact form.
template <bool EXACT_EXP2 = false>
RFX_D v3 decodeRGBE8(v4 rgbe) {  // :136-141
  float fExp = rgbe.w * 255.0f - 128.0f;
  if constexpr (EXACT_EXP2) return xyz(rgbe) * (float)exp2((double)fExp);
  else return xyz(rgbe) * exp2f(fExp);
}
RFX_D void unpackTwoVec4(float4 e, v4& a, v4& b) {  // :85-98
  v2 p = unpackHalf2x16(__float_as_uint(e.x)), q = unpackHalf2x16(__float_as_uint(e.y));
  v2 r = unpackHalf2x16(__float_as_uint(e.z)), s = unpackHalf2x16(__float_as_uint(e.w));
  a = mk4(p.x - RFX_NON_ZERO_OFFSET, p.y - RFX_NON_ZERO_OFFSET, q.x - RFX_NON_ZERO_OFFSET, q.y - RFX_NON_ZERO_OFFSET);
  b = mk4(r.x - RFX_NON_ZERO_OFFSET, r.y - RFX_NON_ZERO_OFFSET, s.x - RFX_NON_ZERO_OFFSET, s.y - RFX_NON_ZERO_OFFSET);
}
RFX_D float4 packTwoVec4(v4 a, v4 b) {  // :65-83
  float4 e;
  e.x = __uint_as_float(packHalf2x16(a.x + RFX_NON_ZERO_OFFSET, a.y + RFX_NON_ZERO_OFFSET));
  e.y = __uint_as_float(packHalf2x16(a.z + RFX_NON_ZERO_OFFSET, a.w + RFX_NON_ZERO_OFFSET));
  e.z = __uint_as_float(packHalf2x16(b.x + RFX_NON_ZERO_OFFSET, b.y + RFX_NON_ZERO_OFFSET));
  e.w = __uint_as_float(packHalf2x16(b.z + RFX_NON_ZERO_OFFSET, b.w + RFX_NON_ZERO_OFFSET));
  return e;
}

// three.js <packing>
RFX_D float perspectiveDepthToViewZ(float d, float n, float f) { return (n * f) / ((f - n) * d - f); }
RFX_D float orthographicDepthToViewZ(float d, float n, float f) { return d * (n - f) - n; }

// ---- planes / samplers ----------------------------------------------------------------------
struct PV {  // device view of an rfx_plane
  const unsigned char* p;
  int w, h;
  long long pitch;
};
RFX_D int clampi(int i, int n) { return min(max(i, 0), n - 1); }
// byte offsets are computed in 32 bits (planes are < 4 GiB; the C ABI rejects larger ones): one IMAD instead of a 64-bit chain
RFX_D unsigned pv_off(const PV& t, int x, int y, int bytes) { return (unsigned)y * (unsigned)t.pitch + (unsigned)x * (unsigned)bytes; }
RFX_D float ld_r32f(const PV& t, int x, int y) { return __ldg((const float*)(t.p + pv_off(t, x, y, 4))); }
RFX_D float4 ld_f4(const PV& t, int x, int y) { return __ldg((const float4*)(t.p + pv_off(t, x, y, 16))); }
RFX_D v4 half4_to_v4(uint2 u) {
  v2 a = unpackHalf2x16(u.x), b = unpackHalf2x16(u.y);
  return mk4(a.x, a.y, b.x, b.y);
}
RFX_D v4 ld_h4(const PV& t, int x, int y) { return half4_to_v4(__ldg((const uint2*)(t.p + pv_off(t, x, y, 8)))); }
RFX_D void st_h4(unsigned char* base, long long pitch, int x, int y, v4 v) {
  uint2 u;
  u.x = packHalf2x16(v.x, v.y);
  u.y = packHalf2x16(v.z, v.w);
  *((uint2*)(base + ((unsigned)y * (unsigned)pitch + (unsigned)x * 8u))) = u;
}
RFX_D void st_f4(unsigned char* base, long long pitch, int x, int y, float4 v) { *((float4*)(base + ((unsigned)y * (unsigned)pitch + (unsigned)x * 16u))) = v; }

// NEAREST texel index for coordinate u in a texture of n texels (clamp-to-edge): floor + convert in one F2I.FLOOR
RFX_D int nearest_i(float u, int n) { return clampi(__float2int_rd(u * (float)n), n); }
RFX_D float tex_r32f_nearest(const PV& t, v2 uv) { return ld_r32f(t, nearest_i(uv.x, t.w), nearest_i(uv.y, t.h)); }
RFX_D float4 tex_f4_nearest(const PV& t, v2 uv) { return ld_f4(t, nearest_i(uv.x, t.w), nearest_i(uv.y, t.h)); }
RFX_D v4 f4v(float4 a) { return mk4(a.x, a.y, a.z, a.w); }

struct Bilin { int x0, x1, y0, y1; float w00, w10, w01, w11; };
RFX_D Bilin bilin_setup(v2 uv, int w, int h) {
  Bilin b;
  float fx = uv.x * (float)w - 0.5f, fy = uv.y * (float)h - 0.5f;
  float x0 = floorf(fx), y0 = floorf(fy);
  float ax = fx - x0, ay = fy - y0;
  int ix = (int)x0, iy = (int)y0;
  b.x0 = clampi(ix, w); b.x1 = clampi(ix + 1, w); b.y0 = clampi(iy, h); b.y1 = clampi(iy + 1, h);
  b.w00 = (1.0f - ax) * (1.0f - ay); b.w10 = ax * (1.0f - ay); b.w01 = (1.0f - ax) * ay; b.w11 = ax * ay;
  return b;
}
RFX_D float bilin_blend(const Bilin& b, float t00, float t10, float t01, float t11) {
  return fma_(t11, b.w11, fma_(t01, b.w01, fma_(t10, b.w10, t00 * b.w00)));
}
RFX_D v4 bilin_blend4(const Bilin& b, v4 t00, v4 t10, v4 t01, v4 t11) {
  return mk4(bilin_blend(b, t00.x, t10.x, t01.x, t11.x), bilin_blend(b, t00.y, t10.y, t01.y, t11.y),
             bilin_blend(b, t00.z, t10.z, t01.z, t11.z), bilin_blend(b, t00.w, t10.w, t01.w, t11.w));
}
RFX_D v4 tex_h4_linear(const PV& t, v2 uv) {
  Bilin b = bilin_setup(uv, t.w, t.h);
  return bilin_blend4(b, ld_h4(t, b.x0, b.y0), ld_h4(t, b.x1, b.y0), ld_h4(t, b.x0, b.y1), ld_h4(t, b.x1, b.y1));
}
RFX_D v4 tex_f4_linear(const PV& t, v2 uv) {  // LINEAR fetch of an RGBA32F plane (the FramebufferTexture history of denoiseMode "full_temporal")
  Bilin b = bilin_setup(uv, t.w, t.h);
  return bilin_blend4(b, f4v(ld_f4(t, b.x0, b.y0)), f4v(ld_f4(t, b.x1, b.y0)), f4v(ld_f4(t, b.x0, b.y1)), f4v(ld_f4(t, b.x1, b.y1)));
}
RFX_D v4 tex_h4_nearest(const PV& t, v2 uv) { return ld_h4(t, nearest_i(uv.x, t.w), nearest_i(uv.y, t.h)); }

// ---- blue noise (reference src/utils/shader/blue_noise.glsl:9-48) ---------------------------
struct BlueShift { int sx, sy; };  // per-pass shift, computed once on the host (depends only on the index)
RFX_D v4 blue_noise_fetch(const uchar4* __restrict__ tex, int size, int px, int py, BlueShift s) {
  uchar4 t = __ldg(tex + ((py + s.sy) % size) * size + ((px + s.sx) % size));
  return mk4((float)t.x / 255.0f, (float)t.y / 255.0f, (float)t.z / 255.0f, (float)t.w / 255.0f);
}

// ---- thread -> pixel mapping: a warp covers an 8x4 pixel tile made of 2x2 quads whose four
// pixels sit in lanes 4q..4q+3, so GLSL fwidth() is two __shfl_xor (lane^1 = horizontal
// neighbour, lane^2 = vertical neighbour).
RFX_D void lane_to_pixel(int lane, int& lx, int& ly) {
  int q = lane >> 2;
  lx = ((q & 3) << 1) | (lane & 1);
  ly = ((q >> 2) << 1) | ((lane >> 1) & 1);
}
RFX_D float fwidth_f(float v) {
  const unsigned full = 0xffffffffu;
  float h = __shfl_xor_sync(full, v, 1), w = __shfl_xor_sync(full, v, 2);
  return fabsf(h - v) + fabsf(w - v);
}
RFX_D v3 fwidth_3(v3 v) { return mk3(fwidth_f(v.x), fwidth_f(v.y), fwidth_f(v.z)); }

RFX_D v2 pixel_uv(int x, int y, int W, int H) { return mk2(((float)x + 0.5f) / (float)W, ((float)y + 0.5f) / (float)H); }

// ------------------------------------------------------------------------------------------
// BRDF helpers shared by K1 and K4 (reference denoiser_compose_functions.glsl:22-51 == ssgi_utils.frag:153-180)
// ------------------------------------------------------------------------------------------
RFX_D void Onb(v3 N, v3& T, v3& B) {
  v3 up = fabsf(N.z) < 0.9999999f ? mk3(0, 0, 1) : mk3(1, 0, 0);
  T = normalize(cross(up, N));
  B = cross(N, T);
}
RFX_D v3 ToLocal(v3 X, v3 Y, v3 Z, v3 V) { return mk3(dot(V, X), dot(V, Y), dot(V, Z)); }
RFX_D v3 ToWorld(v3 X, v3 Y, v3 Z, v3 V) { return V.x * X + V.y * Y + V.z * Z; }
// SampleGGXVNDF with (cos(2 pi r2), sin(2 pi r2)) supplied by the caller
RFX_D v3 SampleGGXVNDF_cs(v3 V, float ax, float ay, float r1, float cphi, float sphi) {
  v3 Vh = normalize(mk3(ax * V.x, ay * V.y, V.z));
  float lensq = Vh.x * Vh.x + Vh.y * Vh.y;
  v3 T1 = lensq > 0.0f ? mk3(-Vh.y, Vh.x, 0.0f) * (1.0f / sqrtf(lensq)) : mk3(1.0f, 0.0f, 0.0f);
  v3 T2 = cross(Vh, T1);
  float r = sqrtf(r1);
  float t1 = r * cphi;
  float t2 = r * sphi;
  float s = 0.5f * (1.0f + Vh.z);
  t2 = (1.0f - s) * sqrtf(1.0f - t1 * t1) + s * t2;
  v3 Nh = t1 * T1 + t2 * T2 + sqrtf(fmaxf(0.0f, 1.0f - t1 * t1 - t2 * t2)) * Vh;
  return normalize(mk3(ax * Nh.x, ay * Nh.y, fmaxf(0.0f, Nh.z)));
}

// ---- SFU arithmetic for the fast kernel variants (values downstream of every per-pixel DECISION; 1-2 ulp) -----------
RFX_D float fx_rcp(float x) { float r; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
RFX_D float fx_sqrt(float x) { float r; asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
RFX_D float fx_rsqrt(float x) { float r; asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
RFX_D float fx_lg2(float x) { float r; asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
RFX_D float fx_ex2(float x) { float r; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
RFX_D v3 fx_normalize(v3 a) { return a * fx_rsqrt(dot(a, a)); }
RFX_D float fx_length(v3 a) { return fx_sqrt(dot(a, a)); }
// clamp an integer texel index to [0, n-1] in two VIMNMX (max(min(i, n-1), 0))
RFX_D int clamp_idx(int i, int nm1) { return max(min(i, nm1), 0); }
RFX_D uint32_t pack_h2(float a, float b) {  // packHalf2x16 in one F2FP
  const __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<const uint32_t*>(&h);
}
RFX_D float h_lo(uint32_t u) { return __half2float(__ushort_as_half((unsigned short)(u & 0xffffu))); }
RFX_D float h_hi(uint32_t u) { return __half2float(__ushort_as_half((unsigned short)(u >> 16))); }

// ---- paired fp32 arithmetic.  The fast chain's value arithmetic is the same expression for the diffuse and the specular
// plane, so the two planes travel together as one (lo, hi) pair.  sm_90 has no packed fp32x2 instructions: each operation is two
// scalar IEEE fp32 operations with explicit rounding (never contracted), so the results are those of the packed form bit for bit.
struct f2 { float lo, hi; };
RFX_D f2 mkf2(float lo, float hi) { return f2{lo, hi}; }
RFX_D f2 mkf2(float s) { return mkf2(s, s); }
RFX_D float f2lo(f2 a) { return a.lo; }
RFX_D float f2hi(f2 a) { return a.hi; }
RFX_D f2 f2fma(f2 a, f2 b, f2 c) { return f2{__fmaf_rn(a.lo, b.lo, c.lo), __fmaf_rn(a.hi, b.hi, c.hi)}; }
RFX_D f2 f2mul(f2 a, f2 b) { return f2{__fmul_rn(a.lo, b.lo), __fmul_rn(a.hi, b.hi)}; }
RFX_D f2 f2add(f2 a, f2 b) { return f2{__fadd_rn(a.lo, b.lo), __fadd_rn(a.hi, b.hi)}; }
RFX_D f2 f2sub(f2 a, f2 b) { return f2{__fsub_rn(a.lo, b.lo), __fsub_rn(a.hi, b.hi)}; }
RFX_D f2 f2lg2(f2 a) { return mkf2(fx_lg2(f2lo(a)), fx_lg2(f2hi(a))); }
RFX_D f2 f2ex2(f2 a) { return mkf2(fx_ex2(f2lo(a)), fx_ex2(f2hi(a))); }

// ---- chain-internal plane formats (fast chain, k_chain.cu) -----------------------------------------------------------
// nrdz: float4 (n.x, n.y, n.z, depth); the 9-bit roughness code k = mod(gBuffer.b, 257) rides in the low mantissa bits of
//       n.x (5 bits) and n.y (4 bits): |dn| <= 2^-19 relative.  roughness = max(k/256 - 1e-4, 0)  (gbuffer_packing.glsl:24-34,189)
RFX_D float nrdz_roughness(float4 t) {
  // (float)k through the 2^23 trick (k < 2^9): integer -> float conversions run on the quarter-rate XU pipe, which the Poisson
  // passes already load to ~60 % with their lg2 / ex2
  const uint32_t kb = (__float_as_uint(t.x) & 31u) | ((__float_as_uint(t.y) & 15u) << 5) | 0x4B000000u;
  return fmaxf((__uint_as_float(kb) - 8388608.0f) * 0.00390625f - RFX_NON_ZERO_OFFSET, 0.0f);
}
// floor(v) for |v| < 2^22 without the conversion (XU) pipe: FADD.RM against 1.5 * 2^23 leaves floor(v) in the low mantissa bits
RFX_D int floor_i(float v, float& fl) {
  const float t = __fadd_rd(v, 12582912.0f);
  fl = t - 12582912.0f;
  return __float_as_int(t) - 0x4B400000;
}
RFX_D int floor_i(float v) { return __float_as_int(__fadd_rd(v, 12582912.0f)) - 0x4B400000; }
RFX_D float4 nrdz_pack(v3 n, float rough_code, float depth) {
  const uint32_t k = (uint32_t)rough_code;
  return make_float4(__uint_as_float((__float_as_uint(n.x) & ~31u) | (k & 31u)), __uint_as_float((__float_as_uint(n.y) & ~15u) | ((k >> 5) & 15u)), n.z, depth);
}

}  // namespace rfx
