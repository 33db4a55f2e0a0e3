// k_ssgi.cu — K1 SSGI / SSR depth-buffer ray march (sm_90a).
//
// Replaces the fullscreen draw of reference src/ssgi/pass/SSGIPass.js:93-94
// (shader src/ssgi/shader/ssgi.frag:105-503 + ssgi_utils.frag).
//
// Mapping: one thread per pixel, a warp owns an 8x4 pixel tile laid out in 2x2 quads so
// the implicit-LOD env fetch (ssgi_utils.frag:218) gets its quad derivatives from two shuffles.
// The march is a data-dependent gather over an L2-resident plane.  Three things keep the per-tap
// instruction count low without changing a single bit of the tap positions:
//   * a per-frame prepass turns the depth plane into a view-space-z plane with the shader's own
//     getViewZ() arithmetic, so a tap is one 4-byte load + two compares (no divide per tap);
//   * when the projection matrix has the perspective sparsity pattern (detected on the host) the
//     fma chain of `projectionMatrix * vec4(p, 1)` drops its exact-zero terms: x' = fma(P00,x,P20*z),
//     y' = fma(P11,y,P21*z), w' = -z — bit-identical to the full chain;
//   * the fast variant (ssgi_fast_kernel) projects and fetches RFX_K1_BATCH march steps together and tests them in order.
// All blue-noise driven transcendentals (sin/cos of 2*pi*k/255, the march step profile
// 1-exp(-0.25 (i+b-0.5)^2)) come from small host-built tables indexed by the 8-bit noise value.
// FAST = true additionally moves the remaining continuous transcendentals to the SFU pipe.
#include "rfx_kernels.h"

namespace rfx {

#define SSGI_EPSILON 0.00001f
#define SSGI_ONE_MINUS_EPSILON (1.0f - 0.00001f)
#define PI_F 3.1415926535897932384626433832795f

RFX_D float lum_s(v3 a) { return dot(mk3(0.2125f, 0.7154f, 0.0721f), a); }  // ssgi_utils.frag:3
RFX_D float lg2a_(float x) { float r; asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }

// FAST-variant arithmetic (AP = true) for everything downstream of the per-pixel DECISIONS (diffuse/specular lottery, env-sample
// choice): SFU reciprocal / sqrt / rsqrt, 1-2 ulp.  The decision chain itself (view position, normals, VNDF sample, Fresnel
// weights, env-sample probability) stays IEEE in both variants: its thresholds are compared with 8-bit blue-noise values, and a
// one-ulp change there flips the lottery for ~1e-4 of the pixels - a different ray, not a rounding difference.
template <bool AP> RFX_D float rcp_(float x) { if (AP) { float r; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; } return 1.0f / x; }
template <bool AP> RFX_D float div_(float a, float b) { return AP ? a * rcp_<true>(b) : a / b; }
template <bool AP> RFX_D float sqrt_(float x) { if (AP) { float r; asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; } return sqrtf(x); }
template <bool AP> RFX_D v3 normalize_(v3 a) {
  if (AP) { float r; asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(dot(a, a))); return a * r; }
  return normalize(a);
}
template <bool AP> RFX_D v3 vdiv_(v3 a, float s) { return a * rcp_<AP>(s); }  // vector / scalar = one reciprocal + multiplies
template <bool AP> RFX_D float smoothstep_(float e0, float e1, float x) {
  const float t = clampf(div_<AP>(x - e0, e1 - e0), 0.0f, 1.0f);
  return t * t * (3.0f - 2.0f * t);
}

// getViewZ  ssgi_utils.frag:7-13
RFX_D float ssgi_view_z(const SsgiArgs& a, float depth) {
  if (a.cam.perspective) return a.near_mul_far / (a.far_minus_near * depth - a.cam.far_plane);
  return depth * a.near_minus_far - a.cam.near_plane;
}

// prepass: viewZ plane = getViewZ(depth), same arithmetic as the shader => bit-identical taps
__global__ void __launch_bounds__(256) viewz_kernel(PV depth, OutV vz, int W, int H, float near_mul_far, float far_minus_near, float near_minus_far,
                                                    float near_plane, float far_plane, int perspective) {
  const int x = (blockIdx.x * 256 + threadIdx.x) * 4, y = blockIdx.y;
  if (x >= W) return;
  const float* src = (const float*)(depth.p + (long long)y * depth.pitch) + x;
  float* dst = (float*)(vz.p + (long long)y * vz.pitch) + x;
  float d[4];
  if (x + 3 < W) { const float4 t = __ldg((const float4*)src); d[0] = t.x; d[1] = t.y; d[2] = t.z; d[3] = t.w; }
  else { for (int i = 0; i < 4; i++) d[i] = x + i < W ? __ldg(src + i) : 0.0f; }
  float o[4];
#pragma unroll
  for (int i = 0; i < 4; i++) o[i] = perspective ? near_mul_far / (far_minus_near * d[i] - far_plane) : d[i] * near_minus_far - near_plane;
  if (x + 3 < W) *(float4*)dst = make_float4(o[0], o[1], o[2], o[3]);
  else { for (int i = 0; i < 4 && x + i < W; i++) dst[i] = o[i]; }
}
cudaError_t launch_viewz(const SsgiArgs& a, OutV vz, cudaStream_t s) {
  const int W = a.depth.w, H = a.depth.h;  // the depth plane's own size (larger than the render target when resolutionScale < 1)
  dim3 grid((W / 4 + 255) / 256 + 1, H);
  viewz_kernel<<<grid, 256, 0, s>>>(a.depth, vz, W, H, a.near_mul_far, a.far_minus_near, a.near_minus_far, a.cam.near_plane, a.cam.far_plane,
                                    a.cam.perspective);
  return cudaGetLastError();
}

// viewSpaceToScreenSpace  ssgi_utils.frag:26-33  (vector / scalar = reciprocal + multiplies, see rfx_device.cuh)
template <bool SPARSE, bool AP>
RFX_D v2 view_to_screen(const SsgiArgs& a, v3 p) {
  float cx, cy, cw;
  const float* M = a.cam.projection.m;
  if (SPARSE) {
    cx = fma_(M[0], p.x, M[8] * p.z);
    cy = fma_(M[5], p.y, M[9] * p.z);
    cw = -p.z;
  } else {
    cx = fma_(M[0], p.x, fma_(M[4], p.y, fma_(M[8], p.z, M[12])));
    cy = fma_(M[1], p.x, fma_(M[5], p.y, fma_(M[9], p.z, M[13])));
    cw = fma_(M[3], p.x, fma_(M[7], p.y, fma_(M[11], p.z, M[15])));
  }
  const float r = rcp_<AP>(cw);
  return mk2((cx * r) * 0.5f + 0.5f, (cy * r) * 0.5f + 0.5f);
}

// Polynomial atan2 / acos (Abramowitz-Stegun 4.4.49 / 4.4.46 evaluated in fp32: 3e-7 / 1.3e-5 rad, i.e. < 0.003 texel of a
// 512-row env map) for the fast kernel's env lookup, ~45 instructions per fetch fewer than libm.
RFX_D float acos_poly(float x) {
  const float ax = fabsf(x);
  float p = -0.0012624911f;
  p = fma_(p, ax, 0.0066700901f); p = fma_(p, ax, -0.0170881256f); p = fma_(p, ax, 0.0308918810f); p = fma_(p, ax, -0.0501743046f);
  p = fma_(p, ax, 0.0889789874f); p = fma_(p, ax, -0.2145988016f); p = fma_(p, ax, 1.5707963050f);
  float s;
  asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(s) : "f"(fmaxf(1.0f - ax, 0.0f)));
  const float r = s * p;
  return x < 0.0f ? PI_F - r : r;
}
RFX_D float atan2_poly(float y, float x) {
  const float ay = fabsf(y), ax = fabsf(x), mx = fmaxf(ay, ax), mn = fminf(ay, ax);
  if (mx == 0.0f) return 0.0f;
  float inv;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(inv) : "f"(mx));
  const float t = mn * inv, s = t * t;
  float q = 0.0028662257f;
  q = fma_(q, s, -0.0161657367f); q = fma_(q, s, 0.0429096138f); q = fma_(q, s, -0.0752896400f); q = fma_(q, s, 0.1065626393f);
  q = fma_(q, s, -0.1420889944f); q = fma_(q, s, 0.1999355085f); q = fma_(q, s, -0.3333314528f); q = fma_(q, s, 1.0f);
  float r = t * q;
  if (ay > ax) r = 0.5f * PI_F - r;
  if (x < 0.0f) r = PI_F - r;
  return y < 0.0f ? -r : r;
}

template <bool AP, bool POLY = false>
RFX_D v2 equirectDirectionToUv(v3 d) {  // ssgi_utils.frag:64-74
  v2 uv = POLY ? mk2(atan2_poly(d.z, d.x), acos_poly(d.y)) : mk2(atan2cr(d.z, d.x), acoscr(d.y));
  uv = mk2(div_<AP>(uv.x, 2.0f * PI_F), div_<AP>(uv.y, PI_F));
  uv.x += 0.5f;
  uv.y = 1.0f - uv.y;
  return uv;
}
template <bool FAST>
RFX_D v3 equirectUvToDirection(v2 uv) {  // :77-86
  uv.x -= 0.5f;
  uv.y = 1.0f - uv.y;
  const float theta = uv.x * 2.0f * PI_F;
  const float phi = uv.y * PI_F;
  if (FAST) {
    float st, ct, sp, cp;
    __sincosf(theta, &st, &ct);
    __sincosf(phi, &sp, &cp);
    return mk3(sp * ct, cp, sp * st);
  }
  const float sinPhi = sincr(phi);
  return mk3(sinPhi * coscr(theta), coscr(phi), sinPhi * sincr(theta));
}
template <bool FAST>
RFX_D float pow5(float x) {
  if (FAST) { const float x2 = x * x; return x2 * x2 * x; }
  return powcr(x, 5.0f);
}
template <bool FAST>
RFX_D float F_Schlick1(float f0, float f90, float theta) { return f0 + (f90 - f0) * pow5<FAST>(1.0f - theta); }
template <bool AP>
RFX_D float D_GTR2(float roughness, float NoH) {  // D_GTR(roughness, NoH, 2.)
  const float a2 = roughness * roughness;
  const float t = (NoH * NoH) * (a2 * a2 - 1.0f) + 1.0f;
  return div_<AP>(a2, PI_F * (t * t));
}
template <bool AP>
RFX_D float SmithG(float NDotV, float alphaG) {
  const float a = alphaG * alphaG;
  const float b = NDotV * NDotV;
  return div_<AP>(2.0f * NDotV, NDotV + sqrt_<AP>(a + b - a * b));
}
template <bool AP>
RFX_D float GGXVNDFPdf(float NoH, float NoV, float roughness) {
  const float D = D_GTR2<AP>(roughness, NoH);
  const float G1 = SmithG<AP>(NoV, roughness * roughness);
  return div_<AP>(D * G1, fmaxf(0.00001f, 4.0f * NoV));
}
template <bool FAST>
RFX_D float evalDisneyDiffuse(float NoL, float NoV, float LoH, float roughness, float metalness) {
  const float FD90 = 0.5f + 2.0f * roughness * (LoH * LoH);
  const float a = F_Schlick1<FAST>(1.0f, FD90, NoL);
  const float b = F_Schlick1<FAST>(1.0f, FD90, NoV);
  return div_<FAST>(a * b, PI_F) * (1.0f - metalness);
}
template <bool AP>
RFX_D float evalDisneySpecular(float roughness, float NoH, float NoV, float NoL) {
  const float D = D_GTR2<AP>(roughness, NoH);
  float ag = 0.5f + roughness * 0.5f;
  ag = ag * ag;
  const float a2 = ag * ag;  // GeometryTerm: a2 = roughness * roughness with roughness := pow(.5 + r*.5, 2.)
  const float G = SmithG<AP>(NoV, a2) * SmithG<AP>(NoL, a2);
  return div_<AP>(D * G, 4.0f * NoL * NoV);
}
template <bool AP>
RFX_D v3 cosineSampleHemisphere_cs(v3 n, float ux, float sth, float cth) {  // ssgi_utils.frag:183-191
  const float r = sqrt_<AP>(ux);
  const v3 b = normalize_<AP>(cross(n, mk3(0.0f, 1.0f, 1.0f)));
  const v3 t = cross(b, n);
  return normalize_<AP>(r * sth * b + sqrt_<AP>(1.0f - ux) * n + r * cth * t);
}
template <bool AP>
RFX_D void calculateAngles(v3 l, v3 v, v3 n, float& NoL, float& NoH, float& LoH, float& VoH) {  // ssgi.frag:93-100
  const v3 h = normalize_<AP>(v + l);
  NoL = clampf(dot(n, l), SSGI_EPSILON, SSGI_ONE_MINUS_EPSILON);
  NoH = clampf(dot(n, h), SSGI_EPSILON, SSGI_ONE_MINUS_EPSILON);
  LoH = clampf(dot(l, h), SSGI_EPSILON, SSGI_ONE_MINUS_EPSILON);
  VoH = clampf(dot(v, h), SSGI_EPSILON, SSGI_ONE_MINUS_EPSILON);
}

// textureLod(map, uv, lod) with linear-mipmap-linear / clamp
RFX_D v3 env_trilinear(const EnvD& e, v2 uv, float lod) {
  const float l = clampf(lod, 0.0f, (float)(e.levels - 1));
  const int l0 = (int)floorf(l);
  const int l1 = min(l0 + 1, e.levels - 1);
  const float f = l - (float)l0;
  const v4 A = tex_h4_linear(e.mip[l0], uv);
  if (f == 0.0f || l1 == l0) return xyz(A);
  const v4 B = tex_h4_linear(e.mip[l1], uv);
  return mk3(mixf(A.x, B.x, f), mixf(A.y, B.y, f), mixf(A.z, B.z, f));
}

// getEnvColor  ssgi.frag:311-346
template <bool AP, bool POLY = false>
RFX_D v3 getEnvColor(const SsgiArgs& a, v3 l, float roughness, bool isDiffuseSample, bool isEnvSample) {
  if (!(a.flags & RFX_SSGI_USE_ENVMAP)) return mk3(0.0f);
  const v3 reflectedWS = normalize_<AP>(mul_dir_left(l, a.cam.view_matrix));
  float mip = a.env_blur * a.max_env_mip;
  if (!isDiffuseSample && roughness < 0.15f) mip *= div_<AP>(roughness, 0.15f);
  v3 s = env_trilinear(a.env, equirectDirectionToUv<AP, POLY>(reflectedWS), mip);
  const float maxEnvLum = isEnvSample ? 100.0f : 25.0f;
  const float envLum = lum_s(s);
  if (envLum > maxEnvLum) s = s * div_<AP>(maxEnvLum, envLum);
  return s;
}

template <bool AP>
RFX_D float getSaturation(v3 c) {  // :348-360
  const float mx = fmaxf(fmaxf(c.x, c.y), c.z), mn = fminf(fminf(c.x, c.y), c.z);
  if (mx == mn) return 0.0f;
  return div_<AP>(mx - mn, mx);
}

// RayMarch + BinarySearch  ssgi.frag:441-503.  `dir` is l scaled in place like the shader's inout.
// Returns the hit uv; sets hit=false and hitPos=(10e9) on a miss.
template <bool SPARSE, bool AP>
RFX_D v2 rayMarch(const SsgiArgs& a, v3& dir, v3& hitPos, int noiseB, bool& hit) {
  dir = dir * (a.ray_distance / (float)a.steps);
  v2 uv = mk2(0.0f, 0.0f);
  hit = false;
  const float* cs_row = a.step_table + noiseB;  // cs(i, b) at [(i-1)*256 + b]
  for (int i = 1; i < a.steps && !hit; i++, cs_row += 256) {
    hitPos = hitPos + dir * __ldg(cs_row);
    uv = view_to_screen<SPARSE, AP>(a, hitPos);
    const float diff = tex_r32f_nearest(a.viewz, uv) - hitPos.z;
    hit = diff >= 0.0f && diff < a.thickness;
  }
  if (!hit) {
    hitPos = mk3(10.0e9f);
    return uv;
  }
  if (a.refine_steps == 0) return uv;
  // BinarySearch
  dir = dir * 0.5f;
  hitPos = hitPos - dir;
  for (int r = 0; r < a.refine_steps; r++) {
    const v2 u = view_to_screen<SPARSE, AP>(a, hitPos);
    const float diff = tex_r32f_nearest(a.viewz, u) - hitPos.z;
    dir = dir * 0.5f;
    if (diff >= 0.0f) hitPos = hitPos - dir; else hitPos = hitPos + dir;
  }
  return view_to_screen<SPARSE, AP>(a, hitPos);
}

struct PixelMat {
  v3 diffuse;
  float roughness, metalness;
};

// doSample  ssgi.frag:362-439
template <bool SPARSE, bool FAST>
RFX_D v3 doSample(const SsgiArgs& a, const PixelMat& m, v3 viewPos, v3 viewNormal, float roughnessSq, bool isDiffuseSample, bool isEnvSample,
                  float NoV, float NoL, float NoH, float LoH, int noiseB, v3& l, v3& hitPos, float& brdf, float& pdf) {
  const float cosTheta = fmaxf(0.0f, dot(viewNormal, l));
  if (isDiffuseSample) {
    brdf = evalDisneyDiffuse<FAST>(NoL, NoV, LoH, roughnessSq, m.metalness);
    pdf = div_<FAST>(NoL, PI_F);
  } else {
    brdf = evalDisneySpecular<FAST>(roughnessSq, NoH, NoV, NoL);
    pdf = GGXVNDFPdf<FAST>(NoH, NoV, roughnessSq);
  }
  brdf *= cosTheta;
  pdf = fmaxf(SSGI_EPSILON, pdf);
  hitPos = viewPos;
  bool hit;
  const v2 coords = rayMarch<SPARSE, FAST>(a, l, hitPos, noiseB, hit);
  const bool allowMissedRays = (a.flags & RFX_SSGI_MISSED_RAYS) != 0;
  if (!hit && !allowMissedRays) return getEnvColor<FAST>(a, l, roughnessSq, isDiffuseSample, isEnvSample);
  v2 vel = mk2(0.0f, 0.0f);
  if (a.velocity.p) { const float4 t = tex_f4_nearest(a.velocity, coords); vel = mk2(t.x, t.y); }  // :400 (null sampler => 0)
  const v2 ruv = coords - vel;
  const bool reproj_ok = ruv.x >= 0.0f && ruv.x <= 1.0f && ruv.y >= 0.0f && ruv.y <= 1.0f;
  // FAST: a hit whose borderFactor is exactly 1 (the inner 70 % x 70 % of the screen) resolves to mix(env, rgi, 1) = env*0 + rgi = rgi
  // for any finite env texel, so the env fetch (equirect mapping + mip select + bilinear taps) is only done when it can matter.
  const bool inner = FAST && reproj_ok && coords.x >= 0.15f && coords.x <= 1.0f - 0.15f && coords.y >= 0.15f && coords.y <= 1.0f - 0.15f;
  v3 envColor = mk3(0.0f);
  if (!inner) envColor = getEnvColor<FAST>(a, l, roughnessSq, isDiffuseSample, isEnvSample);
  v3 SSGI;
  if (reproj_ok) {
    v3 rgi = mk3(0.0f);
    if (a.accumulated.p) rgi = xyz(f4v(tex_f4_nearest(a.accumulated, ruv)));
    const float saturation = getSaturation<FAST>(m.diffuse);
    rgi = mix(rgi, mk3(lum_s(rgi)), (1.0f - roughnessSq) * saturation * 0.4f);
    const float border = 0.15f;
    float bf = smoothstep_<FAST>(0.0f, border, coords.x) * smoothstep_<FAST>(1.0f, 1.0f - border, coords.x) *
               smoothstep_<FAST>(0.0f, border, coords.y) * smoothstep_<FAST>(1.0f, 1.0f - border, coords.y);
    bf = sqrt_<FAST>(bf);
    SSGI = mix(envColor, rgi, bf);
  } else {
    return envColor;
  }
  if (allowMissedRays) {  // envMapSample is vec3(0.) here (:393,430-436)
    if (0.0f > lum_s(SSGI)) SSGI = mk3(0.0f);
  }
  return SSGI;
}

template <int MODE, bool IS, bool SPARSE, bool FAST>
#ifndef RFX_K1_MIN_BLOCKS
#define RFX_K1_MIN_BLOCKS 4  // 64 registers/thread, 4 blocks (32 warps) per SM.  tools/sweep_k1.sh on H100 at 4K: 3 and 4 give the same K1 time, 5 is ~10 % slower
#endif
__global__ void __launch_bounds__(kThreads, RFX_K1_MIN_BLOCKS) ssgi_kernel(const __grid_constant__ SsgiArgs a) {
  int x, y;
  const bool in_rows = range_pixel(a.row0, a.row1, x, y);
  const bool active = x < a.W && y < a.H && in_rows;
  const uchar4 bn = __ldg(a.blue.tex + ((y + a.blue.shift.sy) % a.blue.size) * a.blue.size + ((x + a.blue.shift.sx) % a.blue.size));
  const v4 random = mk4((float)bn.x / 255.0f, (float)bn.y / 255.0f, (float)bn.z / 255.0f, (float)bn.w / 255.0f);

  // env importance sample: CDF lookup + implicit-LOD colour fetch need all four quad lanes (SURVEY.md A3)
  v2 cdfUv = mk2(0.0f, 0.0f);
  float lambda = 0.0f;
  if (IS) {
    const float v = ld_r32f(a.env.marginal, nearest_i(random.x, a.env.marginal.w), 0);                                        // ssgi_utils.frag:212
    const float u = ld_r32f(a.env.conditional, nearest_i(random.y, a.env.conditional.w), nearest_i(v, a.env.conditional.h));  // :213
    cdfUv = mk2(u, v);
    const unsigned full = 0xffffffffu;
    const v2 ux = mk2(__shfl_xor_sync(full, u, 1), __shfl_xor_sync(full, v, 1));
    const v2 uy = mk2(__shfl_xor_sync(full, u, 2), __shfl_xor_sync(full, v, 2));
    const v2 sz = mk2(a.env.size_x, a.env.size_y);
    const v2 ddx = (ux - cdfUv) * sz, ddy = (uy - cdfUv) * sz;
    const float rho = fmaxf(length(ddx), length(ddy));
    lambda = rho > 0.0f ? (FAST ? lg2a_(rho) : log2cr(rho)) : -1000.0f;
  }
  if (!active) return;

  const v2 vUv = pixel_uv(x, y, a.W, a.H);
  const float unpackedDepth = a.scaled ? tex_r32f_nearest(a.depth, vUv) : ld_r32f(a.depth, x, y);  // scaled: NEAREST by uv in the full-size plane
  if (unpackedDepth == 1.0f) {  // background :109-113
    v4 dl = mk4(0.0f, 0.0f, 0.0f, 1.0f);
    if (a.direct.p) dl = tex_h4_linear(a.direct, vUv);
    st_f4(a.out.p, a.out.pitch, x, y, packTwoVec4(dl, dl));
    return;
  }
  const float4 g = a.scaled ? tex_f4_nearest(a.gb, vUv) : ld_f4(a.gb, x, y);
  PixelMat m;
  m.diffuse = xyz(floatToVec4(g.x));
  const v3 worldNormal = unpackNormal(g.y);
  m.roughness = gb_roughness(g.z);
  m.metalness = gb_metalness(g.z);
  const float roughnessSq = clampf(m.roughness * m.roughness, 0.000001f, 1.0f);

  const float viewZ = ssgi_view_z(a, unpackedDepth);
  // getViewPosition  ssgi_utils.frag:17-24
  v3 viewPos;
  {
    const float clipW = a.cam.projection.m[2 * 4 + 3] * viewZ + a.cam.projection.m[3 * 4 + 3];
    v4 clip = mk4((vUv.x - 0.5f) * 2.0f, (vUv.y - 0.5f) * 2.0f, (viewZ - 0.5f) * 2.0f, 1.0f);
    clip = mk4(clip.x * clipW, clip.y * clipW, clip.z * clipW, clip.w * clipW);
    viewPos = xyz(mul(a.cam.projection_inverse, clip));
    viewPos.z = viewZ;
  }
  const v3 viewDir = normalize(viewPos);
  const v3 viewNormal = normalize(mul_dir_left(worldNormal, a.cam.camera_matrix_world));
  const v3 n = viewNormal;
  const v3 v = -viewDir;
  const float NoV = fmaxf(SSGI_EPSILON, dot(n, v));
  v3 V = mul_dir_left(v, a.cam.view_matrix);
  const v3 N = worldNormal;
  v3 T, B;
  Onb(N, T, B);
  V = ToLocal(T, B, N, V);
  const v3 f0 = mix(mk3(0.04f), m.diffuse, m.metalness);

  const float2 sc = __ldg(a.rot_table + bn.y);  // (sin, cos) of 2*pi*random.g
  v3 Hh = SampleGGXVNDF_cs(V, roughnessSq, roughnessSq, random.x, sc.y, sc.x);
  if (Hh.z < 0.0f) Hh = -Hh;
  v3 l = normalize(reflect(-V, Hh));
  l = ToWorld(T, B, N, l);
  l = mul_dir_left(l, a.cam.camera_matrix_world);
  l = normalize(l);
  float NoL, NoH, LoH, VoH;
  calculateAngles<false>(l, v, n, NoL, NoH, LoH, VoH);  // VoH feeds the lottery threshold: IEEE in both variants

  bool isDiffuseSample = false;
  if (MODE == RFX_MODE_SSGI) {
    const v3 F = f0 + (mk3(1.0f) - f0) * pow5<FAST>(1.0f - VoH);
    float diffW = (1.0f - m.metalness) * lum_s(m.diffuse);
    float specW = lum_s(F);
    diffW = fmaxf(diffW, SSGI_EPSILON);
    specW = fmaxf(specW, SSGI_EPSILON);
    const float invW = 1.0f / (diffW + specW);
    diffW *= invW;
    isDiffuseSample = random.z < diffW;
  }

  float emsPdf = 1.0f, emsProbability = 0.0f;
  bool emsIsEnvSample = false;
  v3 envMisDir = mk3(0.0f);
  if (IS) {  // ssgi.frag:197-215, ssgi_utils.frag:210-225
    envMisDir = equirectUvToDirection<FAST>(cdfUv);
    const v3 color = env_trilinear(a.env, cdfUv, lambda);
    const float totalSum = a.env.total_sum_whole + a.env.total_sum_decimal;
    const float pdf0 = lum_s(color) / totalSum;
    emsPdf = a.env.size_x * a.env.size_y * pdf0;
    envMisDir = normalize(mul_dir_left(envMisDir, a.cam.camera_matrix_world));
    emsProbability = dot(envMisDir, viewNormal);
    emsProbability *= m.roughness;
    emsProbability = fminf(SSGI_ONE_MINUS_EPSILON, emsProbability);
    emsIsEnvSample = random.w < emsProbability;
    if (emsIsEnvSample) {
      emsPdf /= 1.0f - emsProbability;
      l = envMisDir;
      calculateAngles<FAST>(l, v, n, NoL, NoH, LoH, VoH);
    } else {
      emsPdf = 1.0f - emsProbability;
    }
  }
  const v3 diffuseRay = emsIsEnvSample ? envMisDir : cosineSampleHemisphere_cs<FAST>(viewNormal, random.x, sc.x, sc.y);
  const v3 specularRay = emsIsEnvSample ? envMisDir : l;

  v3 diffuseGI = mk3(0.0f), specularGI = mk3(0.0f), hitPos = mk3(0.0f);
  float brdf, pdf;
  bool haveDiffuse = false;
  if (MODE == RFX_MODE_SSGI && isDiffuseSample) {  // :222-242
    l = diffuseRay;
    calculateAngles<FAST>(l, v, n, NoL, NoH, LoH, VoH);
    v3 gi = doSample<SPARSE, FAST>(a, m, viewPos, viewNormal, roughnessSq, true, emsIsEnvSample, NoV, NoL, NoH, LoH, bn.z, l, hitPos, brdf, pdf);
    gi = gi * brdf;
    if (emsIsEnvSample) { const float aa = emsPdf * emsPdf, bb = pdf * pdf; gi = gi * div_<FAST>(aa, aa + bb); } else gi = vdiv_<FAST>(gi, pdf);
    gi = vdiv_<FAST>(gi, emsPdf);
    diffuseGI = mix(diffuseGI, gi, 1.0f / 1.0f);  // diffuseSamples == 1
    haveDiffuse = true;
  }
  l = specularRay;  // :246-265
  calculateAngles<FAST>(l, v, n, NoL, NoH, LoH, VoH);
  {
    v3 gi = doSample<SPARSE, FAST>(a, m, viewPos, viewNormal, roughnessSq, isDiffuseSample, emsIsEnvSample, NoV, NoL, NoH, LoH, bn.z, l, hitPos, brdf, pdf);
    gi = gi * brdf;
    if (emsIsEnvSample) { const float aa = emsPdf * emsPdf, bb = pdf * pdf; gi = gi * div_<FAST>(aa, aa + bb); } else gi = vdiv_<FAST>(gi, pdf);
    gi = vdiv_<FAST>(gi, emsPdf);
    specularGI = mix(specularGI, gi, 1.0f / 1.0f);
  }
  const v3 specularHitPos = hitPos;
  if (a.flags & RFX_SSGI_USE_DIRECT_LIGHT) {  // :267-272
    v3 dl = mk3(0.0f);
    if (a.direct.p) dl = xyz(tex_h4_linear(a.direct, vUv));
    diffuseGI = diffuseGI + dl;
    specularGI = specularGI + dl;
  }
  float rayLength = 0.0f;
  if (!(hitPos.x > 10.0e8f)) {  // :288-296
    const v3 cameraPosWS = mk3(a.cam.camera_matrix_world.m[12], a.cam.camera_matrix_world.m[13], a.cam.camera_matrix_world.m[14]);
    const v3 hitPosWS = xyz(mul(a.cam.camera_matrix_world, mk4(specularHitPos, 1.0f)));
    const v3 dWS = cameraPosWS - hitPosWS;
    rayLength = sqrt_<FAST>(dot(dWS, dWS));
  }
  if (MODE == RFX_MODE_SSGI) {
    if (!haveDiffuse) diffuseGI = mk3(-1.0f);
    st_f4(a.out.p, a.out.pitch, x, y, packTwoVec4(mk4(diffuseGI, m.roughness), mk4(specularGI, rayLength)));
  } else {
    const float al = __uint_as_float(packHalf2x16(rayLength, m.roughness));
    st_f4(a.out.p, a.out.pitch, x, y, make_float4(specularGI.x, specularGI.y, specularGI.z, al));
  }
}

// ==========================================================================================================================
// K1, fast variant (fast_math on, full-size target): same shader, restructured for what bounds it (issue
// 68 %, 22.5 of 32 lanes active, 58 instructions per march tap).  Tried and dropped: compacting the
// diffuse rays of a block through shared memory so that full warps trace them — lane use stayed at 22 / 32 (the waste is rays
// leaving the loop at different steps, not the lottery) while the two block barriers cost 0.1 ms.
//   * the march tap is ~25 instructions: projection rows pre-scaled to texel units on the host, packed fp32x2 arithmetic
//     (paired fp32, rfx_device.cuh), one-instruction index clamps, 32-bit word indexing of the viewZ plane;
//   * in a row-sharded group (PEER) last frame's `composed` is sampled in place on the rank that owns the row (NVLink loads).
// The per-pixel DECISIONS (lottery, env-sample choice) keep the IEEE arithmetic of the exact variant; the march positions may
// differ from the oracle's by an ulp (measured at 4K: ~1e-5 of the rays resolve differently, tools/parity_at_size.py).
// ==========================================================================================================================
template <bool SPARSE>
RFX_D float tap_viewz(const SsgiArgs& a, v3 p) {
  f2 t;
  if (SPARSE) {
    const f2 c = f2fma(mkf2(p.x, p.y), mkf2(a.ps_x0, a.ps_y1), f2mul(mkf2(p.z), mkf2(a.ps_x2, a.ps_y2)));
    t = f2fma(c, mkf2(fx_rcp(-p.z)), mkf2(a.ps_hw, a.ps_hh));
  } else {
    const v2 uv = view_to_screen<false, true>(a, p);
    t = mkf2(uv.x * (float)a.W, uv.y * (float)a.H);
  }
  const int ix = clamp_idx(__float2int_rd(f2lo(t)), a.W - 1), iy = clamp_idx(__float2int_rd(f2hi(t)), a.H - 1);
  return __ldg((const float*)a.viewz.p + (iy * a.vz_pitchw + ix));
}
RFX_D v3 fma3(v3 d, float s, v3 p) {
  const f2 xy = f2fma(mkf2(d.x, d.y), mkf2(s), mkf2(p.x, p.y));
  return mk3(f2lo(xy), f2hi(xy), fma_(d.z, s, p.z));
}
// RayMarch + BinarySearch  ssgi.frag:441-503.  The ray positions do not depend on the fetched depths, so BATCH steps are projected
// and fetched together and tested in order: the march is a chain of dependent L2-latency gathers (L1 hit ~50 %), and at ~25
// instructions per tap the other resident warps no longer hide that latency on their own (at most BATCH - 1 wasted taps per hit).
#ifndef RFX_K1_BATCH
#define RFX_K1_BATCH 4  // tools/sweep_k1.sh on H100 at 4K: 2 and 4 are within the run-to-run spread, 1 is slower
#endif
static_assert(RFX_K1_BATCH >= 1 && RFX_K1_BATCH <= 4, "the host step table (ensure_step_table) carries 3 spare rows for the speculative reads");
template <bool SPARSE>
RFX_D v2 march_fast(const SsgiArgs& a, v3& dir, v3& hitPos, int noiseB, bool& hit) {
  constexpr int BATCH = RFX_K1_BATCH;
  dir = dir * (a.ray_distance / (float)a.steps);
  hit = false;
  const float* cs_row = a.step_table + noiseB;  // row i-1 holds cs(i, b); the table carries BATCH spare rows for the speculative reads
  v3 p = hitPos;
  for (int i = 1; i < a.steps && !hit; i += BATCH, cs_row += 256 * BATCH) {
    v3 q[BATCH];
    float z[BATCH];
    v3 t = p;
#pragma unroll
    for (int k = 0; k < BATCH; k++) {  // BATCH steps are projected and fetched together ...
      t = fma3(dir, __ldg(cs_row + 256 * k), t);
      q[k] = t;
      z[k] = tap_viewz<SPARSE>(a, t);
    }
#pragma unroll
    for (int k = 0; k < BATCH; k++) {  // ... and tested in order
      if (!hit && i + k < a.steps) {
        p = q[k];
        const float d = z[k] - q[k].z;
        hit = d >= 0.0f && d < a.thickness;
      }
    }
  }
  if (!hit) {  // the shader returns the uv of the last step tested; with steps = 1 none is, and its uv keeps (0, 0)
    hitPos = mk3(10.0e9f);
    return a.steps > 1 ? view_to_screen<SPARSE, true>(a, p) : mk2(0.0f, 0.0f);
  }
  if (a.refine_steps > 0) {
    dir = dir * 0.5f;
    p = p - dir;
    for (int r = 0; r < a.refine_steps; r++) {
      const float diff = tap_viewz<SPARSE>(a, p) - p.z;
      dir = dir * 0.5f;
      p = diff >= 0.0f ? p - dir : p + dir;
    }
  }
  hitPos = p;
  return view_to_screen<SPARSE, true>(a, p);
}

// doSample  ssgi.frag:362-439 (SFU arithmetic; `desat` = (1 - roughnessSq) * saturation(diffuse) * 0.4)
template <bool SPARSE, bool PEER>
RFX_D v3 sample_fast(const SsgiArgs& a, v3 viewPos, v3 viewNormal, float roughnessSq, float metalness, float desat, bool isDiffuseSample, bool isEnvSample, float NoV,
                     float NoL, float NoH, float LoH, int noiseB, v3 l, v3& hitPos, float& brdf, float& pdf) {
  const float cosTheta = fmaxf(0.0f, dot(viewNormal, l));
  if (isDiffuseSample) {
    brdf = evalDisneyDiffuse<true>(NoL, NoV, LoH, roughnessSq, metalness);
    pdf = NoL * (1.0f / PI_F);
  } else {
    brdf = evalDisneySpecular<true>(roughnessSq, NoH, NoV, NoL);
    pdf = GGXVNDFPdf<true>(NoH, NoV, roughnessSq);
  }
  brdf *= cosTheta;
  pdf = fmaxf(SSGI_EPSILON, pdf);
  hitPos = viewPos;
  bool hit;
  const v2 coords = march_fast<SPARSE>(a, l, hitPos, noiseB, hit);
  const bool allowMissedRays = (a.flags & RFX_SSGI_MISSED_RAYS) != 0;
  if (!hit && !allowMissedRays) return getEnvColor<true, true>(a, l, roughnessSq, isDiffuseSample, isEnvSample);
  v2 vel = mk2(0.0f, 0.0f);
  if (a.velocity.p) { const float4 t = tex_f4_nearest(a.velocity, coords); vel = mk2(t.x, t.y); }
  const v2 ruv = coords - vel;
  const bool reproj_ok = ruv.x >= 0.0f && ruv.x <= 1.0f && ruv.y >= 0.0f && ruv.y <= 1.0f;
  // a hit whose borderFactor is exactly 1 (the inner 70 % x 70 % of the screen) resolves to mix(env, rgi, 1) = rgi: no env fetch
  const bool inner = reproj_ok && coords.x >= 0.15f && coords.x <= 1.0f - 0.15f && coords.y >= 0.15f && coords.y <= 1.0f - 0.15f;
  v3 envColor = mk3(0.0f);
  if (!inner) envColor = getEnvColor<true, true>(a, l, roughnessSq, isDiffuseSample, isEnvSample);
  if (!reproj_ok) return envColor;
  v3 rgi = mk3(0.0f);
  if (a.accumulated.p) {
    const int ix = nearest_i(ruv.x, a.W), iy = nearest_i(ruv.y, a.H);
    const unsigned char* base = PEER ? peer_row_base(a.acc_peer, iy) : a.accumulated.p;
    const float4 t = __ldg((const float4*)(base + ((unsigned)iy * (unsigned)a.accumulated.pitch + (unsigned)ix * 16u)));
    rgi = mk3(t.x, t.y, t.z);
  }
  rgi = mix(rgi, mk3(lum_s(rgi)), desat);
  v3 SSGI = rgi;
  if (!inner) {
    const float border = 0.15f;
    float bf = smoothstep_<true>(0.0f, border, coords.x) * smoothstep_<true>(1.0f, 1.0f - border, coords.x) * smoothstep_<true>(0.0f, border, coords.y) *
               smoothstep_<true>(1.0f, 1.0f - border, coords.y);
    bf = sqrt_<true>(bf);
    SSGI = mix(envColor, rgi, bf);
  }
  if (allowMissedRays && 0.0f > lum_s(SSGI)) SSGI = mk3(0.0f);
  return SSGI;
}

template <int MODE, bool IS, bool SPARSE, bool PEER>
__global__ void __launch_bounds__(kThreads, RFX_K1_MIN_BLOCKS) ssgi_fast_kernel(const __grid_constant__ SsgiArgs a) {
  int x, y;
  const bool in_rows = range_pixel(a.row0, a.row1, x, y);
  const bool active = x < a.W && y < a.H && in_rows;
  const uchar4 bn = __ldg(a.blue.tex + blue_index(a.blue, x, y));
  const v4 random = mk4((float)bn.x / 255.0f, (float)bn.y / 255.0f, (float)bn.z / 255.0f, (float)bn.w / 255.0f);
  const unsigned full = 0xffffffffu;
  v2 cdfUv = mk2(0.0f, 0.0f);
  float lambda = 0.0f;
  if (IS) {  // env importance sample: the implicit-LOD colour fetch needs all four quad lanes (SURVEY.md A3)
    const float v = ld_r32f(a.env.marginal, nearest_i(random.x, a.env.marginal.w), 0);
    const float u = ld_r32f(a.env.conditional, nearest_i(random.y, a.env.conditional.w), nearest_i(v, a.env.conditional.h));
    cdfUv = mk2(u, v);
    const v2 ux = mk2(__shfl_xor_sync(full, u, 1), __shfl_xor_sync(full, v, 1));
    const v2 uy = mk2(__shfl_xor_sync(full, u, 2), __shfl_xor_sync(full, v, 2));
    const v2 sz = mk2(a.env.size_x, a.env.size_y);
    const v2 ddx = (ux - cdfUv) * sz, ddy = (uy - cdfUv) * sz;
    const float rho = fmaxf(length(ddx), length(ddy));
    lambda = rho > 0.0f ? lg2a_(rho) : -1000.0f;
  }
  if (!active) return;
  const v2 vUv = pixel_uv(x, y, a.W, a.H);
  const float unpackedDepth = ld_r32f(a.depth, x, y);
  if (unpackedDepth == 1.0f) {  // background :109-113
    v4 dl = mk4(0.0f, 0.0f, 0.0f, 1.0f);
    if (a.direct.p) dl = tex_h4_linear(a.direct, vUv);
    st_f4(a.out.p, a.out.pitch, x, y, packTwoVec4(dl, dl));
    return;
  }
  const float4 g = ld_f4(a.gb, x, y);
  PixelMat m;
  m.diffuse = xyz(floatToVec4(g.x));
  const v3 worldNormal = unpackNormal(g.y);
  m.roughness = gb_roughness(g.z);
  m.metalness = gb_metalness(g.z);
  const float roughnessSq = clampf(m.roughness * m.roughness, 0.000001f, 1.0f);
  const float viewZ = ssgi_view_z(a, unpackedDepth);
  v3 viewPos;
  {
    const float clipW = a.cam.projection.m[2 * 4 + 3] * viewZ + a.cam.projection.m[3 * 4 + 3];
    v4 clip = mk4((vUv.x - 0.5f) * 2.0f, (vUv.y - 0.5f) * 2.0f, (viewZ - 0.5f) * 2.0f, 1.0f);
    clip = mk4(clip.x * clipW, clip.y * clipW, clip.z * clipW, clip.w * clipW);
    viewPos = xyz(mul(a.cam.projection_inverse, clip));
    viewPos.z = viewZ;
  }
  const v3 viewDir = normalize(viewPos);
  const v3 viewNormal = normalize(mul_dir_left(worldNormal, a.cam.camera_matrix_world));
  const v3 n = viewNormal;
  const v3 v = -viewDir;
  const float NoV = fmaxf(SSGI_EPSILON, dot(n, v));
  v3 V = mul_dir_left(v, a.cam.view_matrix);
  const v3 N = worldNormal;
  v3 T, B;
  Onb(N, T, B);
  V = ToLocal(T, B, N, V);
  const v3 f0 = mix(mk3(0.04f), m.diffuse, m.metalness);
  const float2 sc = __ldg(a.rot_table + bn.y);
  v3 Hh = SampleGGXVNDF_cs(V, roughnessSq, roughnessSq, random.x, sc.y, sc.x);
  if (Hh.z < 0.0f) Hh = -Hh;
  v3 l = normalize(reflect(-V, Hh));
  l = ToWorld(T, B, N, l);
  l = mul_dir_left(l, a.cam.camera_matrix_world);
  l = normalize(l);
  float NoL, NoH, LoH, VoH;
  calculateAngles<false>(l, v, n, NoL, NoH, LoH, VoH);  // VoH feeds the lottery threshold: IEEE
  bool isDiffuseSample = false;
  if (MODE == RFX_MODE_SSGI) {
    const v3 F = f0 + (mk3(1.0f) - f0) * pow5<true>(1.0f - VoH);
    float diffW = (1.0f - m.metalness) * lum_s(m.diffuse);
    float specW = lum_s(F);
    diffW = fmaxf(diffW, SSGI_EPSILON);
    specW = fmaxf(specW, SSGI_EPSILON);
    const float invW = 1.0f / (diffW + specW);
    diffW *= invW;
    isDiffuseSample = random.z < diffW;
  }
  float emsPdf = 1.0f, emsProbability = 0.0f;
  bool emsIsEnvSample = false;
  v3 envMisDir = mk3(0.0f);
  if (IS) {  // ssgi.frag:197-215, ssgi_utils.frag:210-225
    envMisDir = equirectUvToDirection<true>(cdfUv);
    const v3 color = env_trilinear(a.env, cdfUv, lambda);
    const float totalSum = a.env.total_sum_whole + a.env.total_sum_decimal;
    const float pdf0 = lum_s(color) / totalSum;
    emsPdf = a.env.size_x * a.env.size_y * pdf0;
    envMisDir = normalize(mul_dir_left(envMisDir, a.cam.camera_matrix_world));
    emsProbability = dot(envMisDir, viewNormal);
    emsProbability *= m.roughness;
    emsProbability = fminf(SSGI_ONE_MINUS_EPSILON, emsProbability);
    emsIsEnvSample = random.w < emsProbability;
    if (emsIsEnvSample) {
      emsPdf /= 1.0f - emsProbability;
      l = envMisDir;
    } else {
      emsPdf = 1.0f - emsProbability;
    }
  }
  const float desat = (1.0f - roughnessSq) * getSaturation<true>(m.diffuse) * 0.4f;
  const float inv_ems = rcp_<true>(emsPdf);
  v3 diffuseGI = mk3(0.0f), specularGI, hitPos;
  float brdf, pdf;
  if (MODE == RFX_MODE_SSGI && isDiffuseSample) {  // :222-242
    const v3 dray = emsIsEnvSample ? envMisDir : cosineSampleHemisphere_cs<true>(viewNormal, random.x, sc.x, sc.y);
    calculateAngles<true>(dray, v, n, NoL, NoH, LoH, VoH);
    v3 gi = sample_fast<SPARSE, PEER>(a, viewPos, viewNormal, roughnessSq, m.metalness, desat, true, emsIsEnvSample, NoV, NoL, NoH, LoH, bn.z, dray, hitPos, brdf, pdf);
    gi = gi * brdf;
    if (emsIsEnvSample) { const float aa = emsPdf * emsPdf, bb = pdf * pdf; gi = gi * div_<true>(aa, aa + bb); } else gi = vdiv_<true>(gi, pdf);
    diffuseGI = gi * inv_ems;
  }
  calculateAngles<true>(l, v, n, NoL, NoH, LoH, VoH);  // the specular ray :246-265
  {
    v3 gi = sample_fast<SPARSE, PEER>(a, viewPos, viewNormal, roughnessSq, m.metalness, desat, isDiffuseSample, emsIsEnvSample, NoV, NoL, NoH, LoH, bn.z, l, hitPos, brdf, pdf);
    gi = gi * brdf;
    if (emsIsEnvSample) { const float aa = emsPdf * emsPdf, bb = pdf * pdf; gi = gi * div_<true>(aa, aa + bb); } else gi = vdiv_<true>(gi, pdf);
    specularGI = gi * inv_ems;
  }
  float rayLength = 0.0f;
  if (!(hitPos.x > 10.0e8f)) {  // :288-296
    const v3 cameraPosWS = mk3(a.cam.camera_matrix_world.m[12], a.cam.camera_matrix_world.m[13], a.cam.camera_matrix_world.m[14]);
    const v3 hitPosWS = xyz(mul(a.cam.camera_matrix_world, mk4(hitPos, 1.0f)));
    const v3 dWS = cameraPosWS - hitPosWS;
    rayLength = sqrt_<true>(dot(dWS, dWS));
  }
  if (a.flags & RFX_SSGI_USE_DIRECT_LIGHT) {  // :267-272
    v3 dl = mk3(0.0f);
    if (a.direct.p) dl = xyz(tex_h4_linear(a.direct, vUv));
    diffuseGI = diffuseGI + dl;
    specularGI = specularGI + dl;
  }
  if (MODE == RFX_MODE_SSGI) {
    if (!isDiffuseSample) diffuseGI = mk3(-1.0f);
    st_f4(a.out.p, a.out.pitch, x, y, packTwoVec4(mk4(diffuseGI, m.roughness), mk4(specularGI, rayLength)));
  } else {
    const float al = __uint_as_float(packHalf2x16(rayLength, m.roughness));
    st_f4(a.out.p, a.out.pitch, x, y, make_float4(specularGI.x, specularGI.y, specularGI.z, al));
  }
}

template <int MODE, bool IS>
static void launch_ssgi_t(const SsgiArgs& a, dim3 grid, cudaStream_t s) {
  if (a.fast && !a.scaled) {  // the fused fast kernel addresses texels by pixel index: a scaled target takes the general kernel
#define RFX_K1F(SP, PE) ssgi_fast_kernel<MODE, IS, SP, PE><<<grid, kThreads, 0, s>>>(a)
    const bool peer = a.acc_peer.n > 1;
    if (a.proj_sparse) { if (peer) RFX_K1F(true, true); else RFX_K1F(true, false); }
    else { if (peer) RFX_K1F(false, true); else RFX_K1F(false, false); }
#undef RFX_K1F
  } else {
#define RFX_K1(SP, F) ssgi_kernel<MODE, IS, SP, F><<<grid, kThreads, 0, s>>>(a)
    if (a.proj_sparse) { if (a.fast) RFX_K1(true, true); else RFX_K1(true, false); }
    else { if (a.fast) RFX_K1(false, true); else RFX_K1(false, false); }
#undef RFX_K1
  }
}

cudaError_t launch_ssgi(const SsgiArgs& a, cudaStream_t s) {
  dim3 grid((a.W + kTileW - 1) / kTileW, row_tiles(a.row0, a.row1));
  const bool is = (a.flags & RFX_SSGI_IMPORTANCE_SAMPLING) != 0;
  if (a.mode == RFX_MODE_SSGI) {
    if (is) launch_ssgi_t<RFX_MODE_SSGI, true>(a, grid, s); else launch_ssgi_t<RFX_MODE_SSGI, false>(a, grid, s);
  } else {
    if (is) launch_ssgi_t<RFX_MODE_SSR, true>(a, grid, s); else launch_ssgi_t<RFX_MODE_SSR, false>(a, grid, s);
  }
  return cudaGetLastError();
}

}  // namespace rfx
