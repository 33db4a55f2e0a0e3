// k_denoise.cu — K3 Poisson bilateral denoise, K4 GI compose, K5 ssgi compose (sm_90a).
//
// K3 replaces reference src/denoise/shader/poisson_denoise.frag:126-208 (one ping-pong pass of
// src/denoise/pass/PoissonDenoisePass.js:135-149); K4 replaces the fullscreen draw of
// src/denoise/pass/DenoiserComposePass.js:58-85 (+ denoiser_compose_functions.glsl:53-107);
// K5 replaces src/ssgi/shader/ssgi_compose.frag:20-44.
#include "rfx_kernels.h"

namespace rfx {

// luminance() of poisson_denoise.frag:28
RFX_D float lum_p(v3 a) { return powf(dot(mk3(0.2125f, 0.7154f, 0.0721f), a), 0.125f); }

template <bool LINEAR, bool HALF>
RFX_D v4 fetch_in(const PV& t, v2 uv) {
  if (LINEAR) return tex_h4_linear(t, uv);  // Poisson targets are RGBA16F + LinearFilter (PoissonDenoisePass.js:75-81)
  if (HALF) return tex_h4_nearest(t, uv);
  return f4v(tex_f4_nearest(t, uv));        // pass 0 reads the NEAREST fp32 temporal targets
}

// CARRY (row-sharded group): out0 / out1 are double-buffered and a discarded pixel copies last frame's texels from their owner (`c`)
template <int TC, bool GB, bool LINEAR, bool HALF, bool CARRY>
__global__ void __launch_bounds__(kThreads) poisson_kernel(const __grid_constant__ PoissonArgs a, const __grid_constant__ PeerCarry c) {
  int x, y;
  const bool in_rows = range_pixel(a.row0, a.row1, x, y);
  const bool active = x < a.W && y < a.H && in_rows;
  // helper pixels beyond the edge evaluate at the clamped texel (clamp-to-edge sampling)
  const int xc = min(x, a.W - 1), yc = min(y, a.H - 1);
  const v2 vUv = pixel_uv(x, y, a.W, a.H);

  const float depth = ld_r32f(a.depth, xc, yc);
  const float fwd = fwidth_f(depth);
  const float4 gbc = ld_f4(a.gb, xc, yc);                  // packed gBuffer texel or velocity-layout texel
  const v3 normal = unpackNormal(GB ? gbc.y : gbc.z);      // getNormal()  :80-87
  const float fwn = length(fwidth_3(normal));              // :172
  if (!active) return;
  if (depth == 1.0f && fwd == 0.0f) {                      // discard :129-132 (target keeps its texel)
    if (CARRY) { carry_texel<8>(c.p[0], a.out0, x, y); if (TC == 2) carry_texel<8>(c.p[1], a.out1, x, y); }
    return;
  }

  // mat = getMaterial(gBufferTexture, vUv) — without GBUFFER_TEXTURE the sampler is null => texel (0,0,0,1)
  const float roughness = GB ? gb_roughness(gbc.z) : gb_roughness(0.0f);

  const PV* ins[2] = {&a.in0, TC == 1 ? &a.in0 : &a.in1};
  const int spec[2] = {a.spec0, a.spec1};
  v3 rgb[2];
  float alpha[2], lumc[2], age[2], tw[2];
#pragma unroll
  for (int i = 0; i < TC; i++) {  // :138-164
    const PV& tex = spec[i] ? *ins[1] : a.in0;
    v4 t = fetch_in<LINEAR, HALF>(tex, vUv);
    age[i] = 1.0f / powf(t.w + 1.0f, 1.2f * a.phi);
    v3 c = xyz(t) * 1.0003f;
    c = vlog1p_(c);
    rgb[i] = c; alpha[i] = t.w; lumc[i] = lum_p(c); tw[i] = 1.0f;
  }
  const float glossiness = fmaxf(0.0f, 4.0f * (1.0f - roughness / 0.25f));
  const float specularFactor = expf(-glossiness * a.specular_phi);
  float flatness = 1.0f - fminf(fwn, 1.0f);
  flatness = flatness * flatness * 0.75f + 0.25f;  // pow(flatness, 2.) * 0.75 + 0.25

  // rotate the poisson disk by blueNoise().r : (sin, cos) of (k/255)*2*pi from the host table
  const uchar4 bn = __ldg(a.blue.tex + ((y + a.blue.shift.sy) % a.blue.size) * a.blue.size + ((x + a.blue.shift.sx) % a.blue.size));
  const float2 sc = __ldg(a.rot_table + bn.x);
  const float k = a.radius * flatness;
  const float m00 = k * sc.y, m01 = k * -sc.x, m10 = k * sc.x, m11 = k * sc.y;  // mat2 columns (c,-s),(s,c)
  const float resx = (float)a.W, resy = (float)a.H;
  const float SQ = 1.41421356237f;
  const float px[8] = {-1.0f, 0.0f, 1.0f, 0.0f, -0.25f * SQ, 0.25f * SQ, 0.25f * SQ, -0.25f * SQ};
  const float py[8] = {0.0f, -1.0f, 0.0f, 1.0f, -0.25f * SQ, -0.25f * SQ, 0.25f * SQ, 0.25f * SQ};

#pragma unroll
  for (int i = 0; i < 8; i++) {
    const float ox = px[i] / resx, oy = py[i] / resy;
    const v2 nuv = mk2(vUv.x + (m00 * ox + m10 * oy), vUv.y + (m01 * ox + m11 * oy));
    // getBasicNeighborWeight :52-78
    const int nx = nearest_i(nuv.x, a.W), ny = nearest_i(nuv.y, a.H);
    const float4 g = ld_f4(a.gb, nx, ny);
    const float ndepth = GB ? ld_r32f(a.depth, nx, ny) : g.w;
    float wBasic = 0.0f;
    if (ndepth != 1.0f) {
      const v3 nn = unpackNormal(GB ? g.y : g.z);
      const float normalDiff = 1.0f - fmaxf(dot(normal, nn), 0.0f);
      const float depthDiff = 10000.0f * fabsf(depth - ndepth);
      if (GB) {
        const float roughnessDiff = fabsf(roughness - gb_roughness(g.z));
        wBasic = expf(-normalDiff * a.normal_phi - depthDiff * a.depth_phi - roughnessDiff * a.roughness_phi);
      } else {
        wBasic = expf(-normalDiff * a.normal_phi - depthDiff * a.depth_phi);
      }
    }
#pragma unroll
    for (int j = 0; j < TC; j++) {  // applyWeight :102-124
      float w = wBasic;
      const PV& tex = spec[j] ? *ins[1] : a.in0;
      if (spec[j]) w *= specularFactor;
      v4 t = fetch_in<LINEAR, HALF>(tex, nuv);
      v3 c = vlog1p_(xyz(t));
      const float disocclW = powf(w, 0.1f);
      float lumaDiff = fabsf(lumc[j] - lum_p(c));
      lumaDiff = fminf(lumaDiff, 0.5f);
      const float lumaFactor = expf(-lumaDiff * a.luma_phi);
      w = mixf(w * lumaFactor, disocclW, age[j]) * age[j];
      w *= (w < 0.0001f) ? 0.0f : 1.0f;  // step(0.0001, w)
      rgb[j] = rgb[j] + w * c;
      tw[j] += w;
    }
  }
#pragma unroll
  for (int j = 0; j < TC; j++) {  // outputTexel :94-100
    v3 c = vexpm1_(rgb[j] / tw[j]);
    const OutV& o = j == 0 ? a.out0 : a.out1;
    st_h4(o.p, o.pitch, x, y, mk4(c, alpha[j]));
  }
}

// ------------------------------------------------------------------------------------------
// K0  per-frame G-buffer decode prepass: (world normal xyz, roughness) as one float4 per pixel.
// K3 decodes the packed G-buffer 9x per pixel per pass (centre + 8 taps) and runs 2*iterations passes;
// decoding once per frame with the *same* arithmetic (bit-identical values) removes ~1.6k instructions
// per pixel per frame.  For the velocity-layout variant (no GBUFFER_TEXTURE) roughness decodes the
// null-sampler texel (0,0,0,1) => 0 and the normal comes from .b.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) gbuffer_decode_kernel(PV gb, OutV nrd, int W, int row0, int row1, int gbuffer_texture) {
  const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = row0 + blockIdx.y * 8 + (threadIdx.x >> 5);
  if (x >= W || y >= row1) return;
  const float4 g = ld_f4(gb, x, y);
  const v3 n = unpackNormal(gbuffer_texture ? g.y : g.z);
  // .w: roughness (packed gBuffer) or, for the velocity layout, the texel's own depth (its taps read depth from there: poisson_denoise.frag:58-60)
  const float r = gbuffer_texture ? gb_roughness(g.z) : g.w;
  st_f4(nrd.p, nrd.pitch, x, y, make_float4(n.x, n.y, n.z, r));
}
// Decodes the rows the Poisson taps of output rows [row0, row1) can reach: the range widened by `halo` rows (ceil(radius) + 1: tap
// offsets are at most `radius` pixels, + 1 for the quad-derivative helper row).  A rank that owns a band of a tall frame decodes
// that band only, not the whole plane.
cudaError_t launch_gbuffer_decode(PV gb, OutV nrd, int W, int H, int gbuffer_texture, int row0, int row1, int halo, cudaStream_t s) {
  const int r0 = max(0, row0 - halo), r1 = min(H, row1 + halo);
  if (r0 < r1) gbuffer_decode_kernel<<<dim3((W + 31) / 32, (r1 - r0 + 7) / 8), 256, 0, s>>>(gb, nrd, W, r0, r1, gbuffer_texture);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------
// K3 fast variant.  Same algorithm and the same tap geometry (the tap coordinates, nearest texel
// choices and bilinear weights are computed with exactly the arithmetic of poisson_kernel above),
// but the transcendental work is restructured for the SFU pipe (MUFU.LG2 / MUFU.EX2):
//   log(c+1)                   -> lg2(c+1) * ln2
//   luminance = pow(d, 0.125)  -> ex2(0.125 * lg2(d))
//   wBasic = exp(A), w*specularFactor = exp(A + S), pow(w, 0.1) = exp(0.1*(A [+ S])),
//   w * lumaFactor = exp(A [+ S] - lumaDiff*lumaPhi)     (one ex2 each, no pow)
//   age = ex2(-1.2*phi*lg2(a + 1)),  exp(x) - 1 -> ex2(x*log2e) - 1
// The approximate lg2/ex2 have ~2^-22 relative error, far inside the 1e-3 parity budget (the outputs are
// rounded to fp16 anyway); the exact variant above stays available (rfx_ctx_set_fast_math(ctx, 0)).
// ------------------------------------------------------------------------------------------
RFX_D float lg2a(float x) { float r; asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
RFX_D float ex2a(float x) { float r; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
#define RFX_LN2 0.69314718055994530942f
#define RFX_LOG2E 1.44269504088896340736f
// The colours are carried in LOG2 units: lc2 = lg2(c + 1) = log(c + 1) / ln2.  The weighted average is linear, so the final
// exp(avg_ln) - 1 is ex2(avg_lg2) - 1 and the ln2 factor never has to be applied; the luminance pow(dot(w, ln-values), 0.125)
// becomes ex2(0.125 * lg2(dot(w, lc2)) + 0.125 * lg2(ln2)).
RFX_D v3 flog1p3(v3 c) { return mk3(lg2a(c.x + 1.0f), lg2a(c.y + 1.0f), lg2a(c.z + 1.0f)); }
#define RFX_LUM_C (-0.06609580f)  /* 0.125 * log2(ln 2) */
RFX_D float flum(v3 c2) { return ex2a(fma_(0.125f, lg2a(dot(mk3(0.2125f, 0.7154f, 0.0721f), c2)), RFX_LUM_C)); }

template <bool LINEAR>
RFX_D void fetch2(const PoissonArgs& a, v2 uv, bool two, v3& c0, v3& c1, float* alpha0 = nullptr, float* alpha1 = nullptr) {
  if (LINEAR) {  // RGBA16F + LinearFilter: one bilinear setup shared by both planes, in texels of the input (it may be smaller than the output)
    const Bilin b = bilin_setup(uv, a.in0.w, a.in0.h);
    {
      const v4 t00 = ld_h4(a.in0, b.x0, b.y0), t10 = ld_h4(a.in0, b.x1, b.y0), t01 = ld_h4(a.in0, b.x0, b.y1), t11 = ld_h4(a.in0, b.x1, b.y1);
      c0 = mk3(bilin_blend(b, t00.x, t10.x, t01.x, t11.x), bilin_blend(b, t00.y, t10.y, t01.y, t11.y), bilin_blend(b, t00.z, t10.z, t01.z, t11.z));
      if (alpha0) *alpha0 = bilin_blend(b, t00.w, t10.w, t01.w, t11.w);
    }
    if (two) {
      const v4 t00 = ld_h4(a.in1, b.x0, b.y0), t10 = ld_h4(a.in1, b.x1, b.y0), t01 = ld_h4(a.in1, b.x0, b.y1), t11 = ld_h4(a.in1, b.x1, b.y1);
      c1 = mk3(bilin_blend(b, t00.x, t10.x, t01.x, t11.x), bilin_blend(b, t00.y, t10.y, t01.y, t11.y), bilin_blend(b, t00.z, t10.z, t01.z, t11.z));
      if (alpha1) *alpha1 = bilin_blend(b, t00.w, t10.w, t01.w, t11.w);
    }
  } else {  // pass 0: NEAREST fp32 temporal targets
    const int nx = nearest_i(uv.x, a.W), ny = nearest_i(uv.y, a.H);
    const float4 t = ld_f4(a.in0, nx, ny);
    c0 = mk3(t.x, t.y, t.z);
    if (alpha0) *alpha0 = t.w;
    if (two) {
      const float4 u = ld_f4(a.in1, nx, ny);
      c1 = mk3(u.x, u.y, u.z);
      if (alpha1) *alpha1 = u.w;
    }
  }
}

// TC planes; plane j is "specular" per a.spec0/spec1; with TC == 2 plane 1 reads in1, with TC == 1 the single plane reads in0.
// CARRY: as poisson_kernel's
template <int TC, bool LINEAR, bool GB, bool CARRY>
#ifndef RFX_K3_MIN_BLOCKS
#define RFX_K3_MIN_BLOCKS 4
#endif
__global__ void __launch_bounds__(kThreads, RFX_K3_MIN_BLOCKS) poisson_fast_kernel(const __grid_constant__ PoissonArgs a, const __grid_constant__ PeerCarry c) {
  int x, y;
  const bool in_rows = range_pixel(a.row0, a.row1, x, y);
  const bool active = x < a.W && y < a.H && in_rows;
  const int xc = min(x, a.W - 1), yc = min(y, a.H - 1);
  const v2 vUv = pixel_uv(x, y, a.W, a.H);
  const float depth = ld_r32f(a.depth, xc, yc);
  const float fwd = fwidth_f(depth);
  const float4 nc = ld_f4(a.nrd, xc, yc);
  const v3 normal = mk3(nc.x, nc.y, nc.z);
  const float fwn = length(fwidth_3(normal));
  if (!active) return;
  if (depth == 1.0f && fwd == 0.0f) {
    if (CARRY) { carry_texel<8>(c.p[0], a.out0, x, y); if (TC == 2) carry_texel<8>(c.p[1], a.out1, x, y); }
    return;
  }
  const float roughness = GB ? nc.w : 0.0f;  // without GBUFFER_TEXTURE getMaterial() decodes the null sampler's (0,0,0,1): roughness 0 (A8)

  v3 rgb[2];
  float alpha[2], lumc[2], age[2], tw[2];
  {
    v3 c[2];
    fetch2<LINEAR>(a, vUv, TC == 2, c[0], c[1], &alpha[0], &alpha[1]);
#pragma unroll
    for (int i = 0; i < TC; i++) {
      age[i] = ex2a(-1.2f * a.phi * lg2a(alpha[i] + 1.0f));
      rgb[i] = flog1p3(c[i] * 1.0003f);
      lumc[i] = flum(rgb[i]);
      tw[i] = 1.0f;
    }
  }
  const float glossiness = fmaxf(0.0f, 4.0f * (1.0f - roughness / 0.25f));
  // exponent (natural-log units) added for specular planes: w *= exp(-glossiness * specularPhi)
  const float specArg = -glossiness * a.specular_phi;
  const float sarg[2] = {a.spec0 ? specArg : 0.0f, a.spec1 ? specArg : 0.0f};
  // per-pixel constants of the two per-tap exponentials, in log2 units: w*lumaFactor = ex2(A2 + sarg2 - lumaDiff*lphi2) and
  // pow(w, 0.1) = ex2(0.1*A2) * ex2(0.1*sarg2) - the second factor does not depend on the tap, so the planes share one ex2
  const float sarg2[2] = {sarg[0] * RFX_LOG2E, sarg[1] * RFX_LOG2E};
  const float swd[2] = {a.spec0 ? ex2a(sarg2[0] * 0.1f) : 1.0f, a.spec1 ? ex2a(sarg2[1] * 0.1f) : 1.0f};
  const float lphi2 = a.luma_phi * RFX_LOG2E;
  float flatness = 1.0f - fminf(fwn, 1.0f);
  flatness = flatness * flatness * 0.75f + 0.25f;
  const uchar4 bn = __ldg(a.blue.tex + ((y + a.blue.shift.sy) % a.blue.size) * a.blue.size + ((x + a.blue.shift.sx) % a.blue.size));
  const float2 sc = __ldg(a.rot_table + bn.x);
  const float k = a.radius * flatness;
  const float m00 = k * sc.y, m01 = k * -sc.x, m10 = k * sc.x, m11 = k * sc.y;

#pragma unroll
  for (int i = 0; i < 8; i++) {
    const float ox = a.tap_ox[i], oy = a.tap_oy[i];  // POISSON[i] / resolution, divided on the host (IEEE, same value)
    const v2 nuv = mk2(vUv.x + (m00 * ox + m10 * oy), vUv.y + (m01 * ox + m11 * oy));
    const int nx = nearest_i(nuv.x, a.W), ny = nearest_i(nuv.y, a.H);
    float4 nn;
    float ndepth;
    if (GB) {
      ndepth = ld_r32f(a.depth, nx, ny);
      if (ndepth == 1.0f) continue;  // wBasic = 0 => w = 0 for every plane: the tap contributes nothing
      nn = ld_f4(a.nrd, nx, ny);
    } else {  // velocity layout: the tap's depth is the normal texel's alpha
      nn = ld_f4(a.nrd, nx, ny);
      ndepth = nn.w;
      if (ndepth == 1.0f) continue;
    }
    const float normalDiff = 1.0f - fmaxf(dot(normal, mk3(nn.x, nn.y, nn.z)), 0.0f);
    const float depthDiff = 10000.0f * fabsf(depth - ndepth);
    const float A = GB ? -normalDiff * a.normal_phi - depthDiff * a.depth_phi - fabsf(roughness - nn.w) * a.roughness_phi : -normalDiff * a.normal_phi - depthDiff * a.depth_phi;
    const float A2 = A * RFX_LOG2E;
    const float wdA = ex2a(A2 * 0.1f);
    v3 c[2];
    fetch2<LINEAR>(a, nuv, TC == 2, c[0], c[1]);
#pragma unroll
    for (int j = 0; j < TC; j++) {
      const v3 lc = flog1p3(c[j]);
      const float lumaDiff = fminf(fabsf(lumc[j] - flum(lc)), 0.5f);
      const float wl = ex2a(fma_(-lumaDiff, lphi2, A2 + sarg2[j]));  // w * lumaFactor
      const float wd = wdA * swd[j];                                  // pow(w, 0.1)
      float w = mixf(wl, wd, age[j]) * age[j];
      w = (w < 0.0001f) ? 0.0f : w;
      rgb[j] = mk3(fma_(w, lc.x, rgb[j].x), fma_(w, lc.y, rgb[j].y), fma_(w, lc.z, rgb[j].z));
      tw[j] += w;
    }
  }
#pragma unroll
  for (int j = 0; j < TC; j++) {
    const float inv = __frcp_rn(tw[j]);
    const v3 m = rgb[j] * inv;
    const v3 c = mk3(ex2a(m.x) - 1.0f, ex2a(m.y) - 1.0f, ex2a(m.z) - 1.0f);  // m is in log2 units
    const OutV& o = j == 0 ? a.out0 : a.out1;
    st_h4(o.p, o.pitch, x, y, mk4(c, alpha[j]));
  }
}

cudaError_t launch_poisson_fast(const PoissonArgs& a, cudaStream_t s, const PeerCarry* carry) {
  dim3 grid((a.W + kTileW - 1) / kTileW, row_tiles(a.row0, a.row1));
  if (a.input_linear && !a.in_half) return cudaErrorInvalidValue;
  if (!a.input_linear && a.in_half) return cudaErrorNotSupported;
  const PeerCarry c = carry ? *carry : PeerCarry{};
#define RFX_PF2(TC, LIN, GB) do { if (carry) poisson_fast_kernel<TC, LIN, GB, true><<<grid, kThreads, 0, s>>>(a, c); else poisson_fast_kernel<TC, LIN, GB, false><<<grid, kThreads, 0, s>>>(a, c); } while (0)
#define RFX_PF(TC, LIN) do { if (a.gbuffer_texture) RFX_PF2(TC, LIN, true); else RFX_PF2(TC, LIN, false); } while (0)
  if (a.texture_count == 2) { if (a.input_linear) RFX_PF(2, true); else RFX_PF(2, false); }
  else { if (a.input_linear) RFX_PF(1, true); else RFX_PF(1, false); }
#undef RFX_PF
#undef RFX_PF2
  return cudaGetLastError();
}

cudaError_t launch_poisson(const PoissonArgs& a, cudaStream_t s, const PeerCarry* carry) {
  dim3 grid((a.W + kTileW - 1) / kTileW, row_tiles(a.row0, a.row1));
  const PeerCarry c = carry ? *carry : PeerCarry{};
#define RFX_LP(TC, GB, LIN, HALF) do { if (carry) poisson_kernel<TC, GB, LIN, HALF, true><<<grid, kThreads, 0, s>>>(a, c); else poisson_kernel<TC, GB, LIN, HALF, false><<<grid, kThreads, 0, s>>>(a, c); } while (0)
  const bool lin = a.input_linear, half = a.in_half, gb = a.gbuffer_texture;
  if (lin && !half) return cudaErrorInvalidValue;
  if (a.texture_count == 2) {
    if (gb) { if (lin) RFX_LP(2, true, true, true); else if (half) RFX_LP(2, true, false, true); else RFX_LP(2, true, false, false); }
    else    { if (lin) RFX_LP(2, false, true, true); else if (half) RFX_LP(2, false, false, true); else RFX_LP(2, false, false, false); }
  } else {
    if (gb) { if (lin) RFX_LP(1, true, true, true); else if (half) RFX_LP(1, true, false, true); else RFX_LP(1, true, false, false); }
    else    { if (lin) RFX_LP(1, false, true, true); else if (half) RFX_LP(1, false, false, true); else RFX_LP(1, false, false, false); }
  }
#undef RFX_LP
  return cudaGetLastError();
}

// CARRY: `out` is double-buffered and a discarded pixel copies last frame's texel from its owner (`c`), as in poisson_kernel
template <bool CARRY>
__global__ void __launch_bounds__(kThreads) gi_compose_kernel(const __grid_constant__ ComposeArgs a, const __grid_constant__ PeerPV c) {
  int x, y;
  const bool in_rows = range_pixel(a.row0, a.row1, x, y);
  const bool active = x < a.W && y < a.H && in_rows;
  const int xc = min(x, a.W - 1), yc = min(y, a.H - 1);
  const float depth = ld_r32f(a.depth, xc, yc);
  const float fwd = fwidth_f(depth);
  if (!active) return;
  if (depth == 1.0f && fwd == 0.0f) {  // DenoiserComposePass.js:61-64
    if (CARRY) carry_texel<16>(c, a.out, x, y);
    return;
  }
  const v2 vUv = pixel_uv(x, y, a.W, a.H);
  const float4 g = ld_f4(a.gb, x, y);
  const v3 diffuse = xyz(floatToVec4(g.x));
  const v3 wn = unpackNormal(g.y);
  const float rough0 = gb_roughness(g.z), metalness = gb_metalness(g.z);
  const v4 rgbe = floatToVec4(g.w);
  const v3 emissive = a.fast ? decodeRGBE8(rgbe) : decodeRGBE8<true>(rgbe);

  const v3 viewNormal = mul_dir_left(wn, a.cam.camera_matrix_world);
  const float gz = a.cam.perspective ? perspectiveDepthToViewZ(depth, a.cam.near_plane, a.cam.far_plane)
                                     : orthographicDepthToViewZ(depth, a.cam.near_plane, a.cam.far_plane);
  const float viewZ = -gz;
  // getViewPosition  denoiser_compose_functions.glsl:13-20
  const float clipW = a.cam.projection.m[2 * 4 + 3] * viewZ + a.cam.projection.m[3 * 4 + 3];
  v4 clip = mk4((vUv.x - 0.5f) * 2.0f, (vUv.y - 0.5f) * 2.0f, (viewZ - 0.5f) * 2.0f, 1.0f);
  clip = mk4(clip.x * clipW, clip.y * clipW, clip.z * clipW, clip.w * clipW);
  v3 viewPos = xyz(mul(a.cam.projection_inverse, clip));
  viewPos.z = -viewZ;
  const v3 viewDir = normalize(viewPos);
  // pixel-centre fetch of the LINEAR Poisson targets: the literal bilinear fetch a GL sampler performs, in both variants.  Its weights
  // are (1,0,0,0) only up to a few ulps of u*W - 0.5, so the centre texel alone is off by up to ~1e-3 x the neighbour contrast on
  // wide frames (3840 columns), which GI planes with 64x contrast between neighbours push past the 1e-3 bar.
  // a texture the inputType does not bind is a null sampler: (0,0,0,1)  (DenoiserComposePass.js:23-33)
  const v4 nul = mk4(0.0f, 0.0f, 0.0f, 1.0f);
  const v4 dgi = !a.diffuse.p ? nul : (a.gi_f32 ? f4v(ld_f4(a.diffuse, x, y)) : tex_h4_linear(a.diffuse, vUv));
  const v4 sgi = !a.specular.p ? nul : (a.gi_f32 ? f4v(ld_f4(a.specular, x, y)) : tex_h4_linear(a.specular, vUv));

  // constructGlobalIllumination :53-107
  const float roughness = rough0 * rough0;
  const v3 normal = mul_dir_left(viewNormal, a.cam.view_matrix);
  v3 T, B;
  const v3 v = -viewDir;
  v3 V = mul_dir_left(v, a.cam.view_matrix);
  const v3 N = normal;
  Onb(N, T, B);
  V = ToLocal(T, B, N, V);
  // r2 = 0.25 => phi = pi/2: (cos, sin) correctly rounded in fp32
  const float phi = 2.0f * 3.1415926535897932384626433832795f * 0.25f;
  const float cphi = -4.37113883e-08f;  // (float)cos((double)phi), phi = fp32(pi/2)
  const float sphi = 1.0f;
  (void)phi;
  v3 Hh = SampleGGXVNDF_cs(V, roughness, roughness, 0.25f, cphi, sphi);
  if (Hh.z < 0.0f) Hh = -Hh;
  v3 l = normalize(reflect(-V, Hh));
  l = ToWorld(T, B, N, l);
  l = xyz(mul(mk4(l, 1.0f), a.cam.camera_matrix_world));  // vec4(l, 1.) * cameraMatrixWorld  (:81)
  l = normalize(l);
  if (dot(viewNormal, l) < 0.0f) l = -l;
  const v3 h = normalize(v + l);
  const float VoH = fmaxf(1e-6f, dot(v, h));
  const v3 f0 = mix(mk3(0.04f), diffuse, metalness);
  const float omv = 1.0f - VoH, omv2 = omv * omv;
  const v3 F = f0 + (mk3(1.0f) - f0) * (a.fast ? omv2 * omv2 * omv : powcr(omv, 5.0f));
  // TYPE_SPECULAR (SSR): the diffuse component is the scene colour (composer input buffer, LINEAR)  denoiser_compose_functions.glsl:97-101
  const v3 diffuseComponent = a.input_type != RFX_INPUT_SPECULAR ? diffuse * (1.0f - metalness) * (mk3(1.0f) - F) * xyz(dgi)
                                                                 : (a.scene.p ? xyz(tex_h4_linear(a.scene, vUv)) : mk3(0.0f));
  const v3 specularComponent = xyz(sgi) * F;
  const v3 gi = diffuseComponent + specularComponent + emissive;
  st_f4(a.out.p, a.out.pitch, x, y, make_float4(gi.x, gi.y, gi.z, 1.0f));
}

cudaError_t launch_gi_compose(const ComposeArgs& a, cudaStream_t s, const PeerPV* carry) {
  dim3 grid((a.W + kTileW - 1) / kTileW, row_tiles(a.row0, a.row1));
  if (carry) gi_compose_kernel<true><<<grid, kThreads, 0, s>>>(a, *carry);
  else gi_compose_kernel<false><<<grid, kThreads, 0, s>>>(a, PeerPV{});
  return cudaGetLastError();
}

__global__ void __launch_bounds__(256) ssgi_compose_kernel(const __grid_constant__ SsgiComposeArgs a) {
  const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = a.row0 + blockIdx.y * 8 + (threadIdx.x >> 5);
  if (x >= a.W || y >= a.row1) return;
  st_h4(a.out.p, a.out.pitch, x, y, ssgi_compose_px(a, x, y));
}
cudaError_t launch_ssgi_compose(const SsgiComposeArgs& a, cudaStream_t s) {
  dim3 grid((a.W + 31) / 32, (a.row1 - a.row0 + 7) / 8);
  ssgi_compose_kernel<<<grid, 256, 0, s>>>(a);
  return cudaGetLastError();
}

}  // namespace rfx
