// k_chain.cu — the fast SSGI chain's kernels K2 / K3 / K4 on chain-internal plane formats (sm_90a).
//
// Same passes as k_temporal.cu / k_denoise.cu (reference: temporal_reproject.frag + reproject.frag, poisson_denoise.frag:126-208,
// DenoiserComposePass.js:58-85 + denoiser_compose_functions.glsl:53-107) with the same tap geometry, texel choices and per-pixel
// decisions (those stay in the IEEE arithmetic the oracle uses), restructured around what bounds them — instruction issue
// and L1 wavefronts, not HBM:
//   * the two denoise planes travel as ONE 16-byte texel {diffuse rgba, specular rgba} in fp16 (one LDG.128 per bilinear corner
//     instead of two LDG.64, one address computation instead of two), the temporal targets as one 32-byte fp32 texel;
//   * the tap texel of the decoded G-buffer carries depth and roughness too (nrdz, one LDG.128 per tap instead of LDG.128 + LDG.32);
//   * the GI compose runs inside the last Poisson pass (its only neighbourhood is the pixel itself in the fast variant), which
//     removes a launch and a round trip of depth + G-buffer + both denoise planes;
//   * value arithmetic downstream of the decisions uses the SFU (rcp / rsqrt / lg2 / ex2 .approx).
// Row-sharded frames (PEER = true) read rows of last frame's history owned by another rank in place, through peer-mapped
// pointers (NVLink loads), instead of receiving replicated planes.
#include "rfx_kernels.h"

namespace rfx {

#define C_LN2 0.69314718055994530942f
#define C_LOG2E 1.44269504088896340736f

// ------------------------------------------------------------------------------------------------------------------
// decode prepass: gBuffer + depth -> nrdz
// ------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) cdecode_kernel(const CDecodeArgs a, int row0, int row1) {
  const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = row0 + blockIdx.y * 8 + (threadIdx.x >> 5);
  if (x >= a.W || y >= row1) return;
  const float4 g = ld_f4(a.gb, x, y);
  const v3 n = unpackNormal(g.y);
  const float k = mod_gl(g.z, 257.0f);  // float2color(...).r * 256 : the 9-bit roughness code (gbuffer_packing.glsl:24-34)
  st_f4(a.nrdz.p, a.nrdz.pitch, x, y, nrdz_pack(n, fminf(fmaxf(k, 0.0f), 256.0f), ld_r32f(a.depth, x, y)));
}
cudaError_t launch_cdecode(const CDecodeArgs& a, int row0, int row1, int halo, cudaStream_t s) {
  const int r0 = max(0, row0 - halo), r1 = min(a.H, row1 + halo);
  if (r0 < r1) cdecode_kernel<<<dim3((a.W + 31) / 32, (r1 - r0 + 7) / 8), 256, 0, s>>>(a, r0, r1);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------------------------
// K2 (SSGI form: 2 planes, packed K1 input, logTransform, LINEAR history)
// ------------------------------------------------------------------------------------------------------------------
struct CTState {
  v2 vUv, velocity;
  v3 worldNormal, worldPos;
  float depth, curvature, rayLength, roughness, moveFactor;
};

// reproject.frag:21-28; EXACT = the IEEE perspective divide (the result feeds texel choices), else SFU reciprocal (distances only)
template <bool EXACT>
RFX_D v3 c_screen_to_world(v2 uv, float depth, const M4& world, const M4& projInv) {
  const v4 ndc = mk4((uv.x - 0.5f) * 2.0f, (uv.y - 0.5f) * 2.0f, (depth - 0.5f) * 2.0f, 1.0f);
  const v4 clip = mul(projInv, ndc);
  const float r = EXACT ? 1.0f / clip.w : fx_rcp(clip.w);
  return xyz(mul(world, mk4(clip.x * r, clip.y * r, clip.z * r, clip.w * r)));
}
RFX_D v3 c_log1p(v3 c) { return mk3(fx_lg2(c.x + 1.0f) * C_LN2, fx_lg2(c.y + 1.0f) * C_LN2, fx_lg2(c.z + 1.0f) * C_LN2); }
RFX_D v3 c_expm1(v3 c) { return mk3(fx_ex2(c.x * C_LOG2E) - 1.0f, fx_ex2(c.y * C_LOG2E) - 1.0f, fx_ex2(c.z * C_LOG2E) - 1.0f); }
RFX_D float c_pow(float x, float p) { return fx_ex2(p * fx_lg2(x)); }
RFX_D v3 c_unpack_normal(float packed) {  // unpackNormal with an SFU normalise
  v2 f = unpackHalf2x16(__float_as_uint(packed));
  f = f * 2.0f - 1.0f;
  v3 n = mk3(f.x, f.y, 1.0f - fabsf(f.x) - fabsf(f.y));
  const float t = fmaxf(-n.z, 0.0f);
  n.x += n.x >= 0.0f ? -t : t;
  n.y += n.y >= 0.0f ? -t : t;
  return fx_normalize(n);
}

// validateReprojectedUV  reproject.frag:130-167
RFX_D float c_validate(const CTemporalArgs& a, const CTState& s, v2 ruv, float distFactor) {
  if (ruv.x > 1.0f || ruv.x < 0.0f || ruv.y > 1.0f || ruv.y < 0.0f) return 0.0f;
  const float4 t = tex_f4_nearest(a.velocity, ruv);
  const v3 lastWorldNormal = c_unpack_normal(t.z);
  const v3 lastWorldPos = c_screen_to_world<false>(ruv, t.w, a.prev_world, a.prev_proj_inv);
  const v3 dpos = s.worldPos - lastWorldPos;
  float disoccl = fx_length(dpos) * 0.1f * distFactor;
  disoccl += fabsf(dot(dpos, s.worldNormal)) * 0.05f * distFactor;
  disoccl += fminf(1.0f - dot(s.worldNormal, lastWorldNormal), 1.0f) * distFactor;
  const float confidence = fmaxf(1.0f - fminf(disoccl, 1.0f), 0.0f);
  return c_pow(confidence, a.confidence_power);
}

// reprojectHitPoint  reproject.frag:169-193 — IEEE throughout: the result selects history / velocity texels
RFX_D v2 c_reproject_hit(const CTemporalArgs& a, const CTState& s) {
  if (s.curvature > 0.05f || s.rayLength < 0.01f) return mk2(-1.0f, -1.0f);
  const v3 cameraPos = mk3(a.camera_pos[0], a.camera_pos[1], a.camera_pos[2]);
  const v3 cameraRay = normalize(s.worldPos - cameraPos);
  const v3 hit = cameraPos + cameraRay * s.rayLength;
  const v4 rh = mul(a.prev_proj_view, mk4(hit, 1.0f));
  const v2 q = mk2(rh.x, rh.y) / rh.w;
  return mk2(q.x * 0.5f + 0.5f, q.y * 0.5f + 0.5f);
}

// one LINEAR fetch of plane `PL` (0 diffuse, 1 specular) of the interleaved dn history; channels packed as (r,g) and (b,a)
struct H4 { f2 rg, ba; };
template <int PL, bool PEER>
RFX_D H4 c_hist_bilinear(const PeerPV& h, v2 uv) {
  const Bilin b = bilin_setup(uv, h.local.w, h.local.h);
  const unsigned char* r0 = PEER ? peer_row_base(h, b.y0) : h.local.p;
  const unsigned char* r1 = PEER ? peer_row_base(h, b.y1) : h.local.p;
  const unsigned o0 = (unsigned)b.y0 * (unsigned)h.local.pitch + 8u * PL, o1 = (unsigned)b.y1 * (unsigned)h.local.pitch + 8u * PL;
  const uint2 t00 = __ldg((const uint2*)(r0 + (o0 + (unsigned)b.x0 * 16u))), t10 = __ldg((const uint2*)(r0 + (o0 + (unsigned)b.x1 * 16u)));
  const uint2 t01 = __ldg((const uint2*)(r1 + (o1 + (unsigned)b.x0 * 16u))), t11 = __ldg((const uint2*)(r1 + (o1 + (unsigned)b.x1 * 16u)));
#define C_BL(M) f2fma(mkf2(h_lo(t11.M), h_hi(t11.M)), mkf2(b.w11), f2fma(mkf2(h_lo(t01.M), h_hi(t01.M)), mkf2(b.w01), \
                f2fma(mkf2(h_lo(t10.M), h_hi(t10.M)), mkf2(b.w10), f2mul(mkf2(h_lo(t00.M), h_hi(t00.M)), mkf2(b.w00)))))
  H4 r;
  r.rg = C_BL(x); r.ba = C_BL(y);
#undef C_BL
  return r;
}

// BiCubicCatmullRom5Tap  reproject.frag:212-255 (texel choice: IEEE; weights: SFU reciprocals)
template <int PL, bool PEER>
RFX_D H4 c_catmull5(const CTemporalArgs& a, v2 P) {
  const v2 inv = mk2(a.inv_w, a.inv_h);
  const v2 UV = mk2(P.x / inv.x, P.y / inv.y);
  const v2 tc = mk2(floorf(UV.x - 0.5f) + 0.5f, floorf(UV.y - 0.5f) + 0.5f);
  const v2 f = UV - tc;
  const v2 f2_ = f * f;
  const v2 f3 = f2_ * f;
  const v2 w0 = f2_ - 0.5f * (f3 + f);
  const v2 w1 = 1.5f * f3 - 2.5f * f2_ + mk2(1.0f, 1.0f);
  const v2 w3 = 0.5f * (f3 - f2_);
  const v2 w2 = mk2(1.0f, 1.0f) - w0 - w1 - w3;
  const v2 W0 = w0, W1 = w1 + w2, W2 = w3;
  const v2 S0 = (tc - mk2(1.0f, 1.0f)) * inv, S1 = mk2((tc.x + w2.x * fx_rcp(W1.x)) * inv.x, (tc.y + w2.y * fx_rcp(W1.y)) * inv.y), S2 = (tc + mk2(2.0f, 2.0f)) * inv;
  const float sw0 = W1.x * W0.y, sw1 = W0.x * W1.y, sw2 = W1.x * W1.y, sw3 = W2.x * W1.y, sw4 = W1.x * W2.y;
  const H4 Ct = c_hist_bilinear<PL, PEER>(a.hist, mk2(S1.x, S0.y)), Cl = c_hist_bilinear<PL, PEER>(a.hist, mk2(S0.x, S1.y)),
           Cc = c_hist_bilinear<PL, PEER>(a.hist, mk2(S1.x, S1.y)), Cr = c_hist_bilinear<PL, PEER>(a.hist, mk2(S2.x, S1.y)),
           Cb = c_hist_bilinear<PL, PEER>(a.hist, mk2(S1.x, S2.y));
  const f2 wm = mkf2(fx_rcp(sw0 + sw1 + sw2 + sw3 + sw4));
  const f2 rg = f2mul(f2fma(Cb.rg, mkf2(sw4), f2fma(Cr.rg, mkf2(sw3), f2fma(Cc.rg, mkf2(sw2), f2fma(Cl.rg, mkf2(sw1), f2mul(Ct.rg, mkf2(sw0)))))), wm);
  const f2 ba = f2mul(f2fma(Cb.ba, mkf2(sw4), f2fma(Cr.ba, mkf2(sw3), f2fma(Cc.ba, mkf2(sw2), f2fma(Cl.ba, mkf2(sw1), f2mul(Ct.ba, mkf2(sw0)))))), wm);
  H4 r;
  r.rg = mkf2(fmaxf(f2lo(rg), 0.0f), fmaxf(f2hi(rg), 0.0f));
  r.ba = mkf2(fmaxf(f2lo(ba), 0.0f), fmaxf(f2hi(ba), 0.0f));
  return r;
}

// reproject() + accumulate() (temporal_reproject.frag:83-122, 42-79) for BOTH planes at once: every quantity is a packed pair
// (.lo = diffuse plane, .hi = specular plane), so the arithmetic the two planes share is written once (rfx_device.cuh: f2).
RFX_D f2 p_log1p(f2 c) { return f2mul(f2lg2(f2add(c, mkf2(1.0f))), mkf2(C_LN2)); }
RFX_D f2 p_expm1(f2 c) { return f2sub(f2ex2(f2mul(c, mkf2(C_LOG2E))), mkf2(1.0f)); }
RFX_D f2 p_min(f2 a, f2 b) { return mkf2(fminf(f2lo(a), f2lo(b)), fminf(f2hi(a), f2hi(b))); }
RFX_D f2 p_max(f2 a, f2 b) { return mkf2(fmaxf(f2lo(a), f2lo(b)), fmaxf(f2hi(a), f2hi(b))); }
RFX_D f2 p_sel(bool s0, bool s1, f2 a, f2 b) { return mkf2(s0 ? f2lo(a) : f2lo(b), s1 ? f2hi(a) : f2hi(b)); }
RFX_D f2 p_rcp(f2 a) { return mkf2(fx_rcp(f2lo(a)), fx_rcp(f2hi(a))); }
RFX_D f2 p_mix(f2 x, f2 y, f2 t, f2 omt) { return f2fma(y, t, f2mul(x, omt)); }  // mix(x, y, t) with omt = 1 - t

template <bool PEER>
RFX_D void c_temporal_planes(const CTemporalArgs& a, const CTState& s, v3 ruvD, v3 ruvS, const v4* inp, const bool* sampled, const v3* mn, const v3* mx, float4& out0, float4& out1) {
  const H4 h0 = c_catmull5<0, PEER>(a, mk2(ruvD.x, ruvD.y)), h1 = c_catmull5<1, PEER>(a, mk2(ruvS.x, ruvS.y));
  const f2 one = mkf2(1.0f);
  f2 accR = p_log1p(mkf2(f2lo(h0.rg), f2lo(h1.rg))), accG = p_log1p(mkf2(f2hi(h0.rg), f2hi(h1.rg))), accB = p_log1p(mkf2(f2lo(h0.ba), f2lo(h1.ba)));
  f2 accA = mkf2(f2hi(h0.ba), f2hi(h1.ba));
  const f2 conf = mkf2(ruvD.z, ruvS.z);
  const bool s0 = sampled[0], s1 = sampled[1];
  f2 inR = mkf2(inp[0].x, inp[1].x), inG = mkf2(inp[0].y, inp[1].y), inB = mkf2(inp[0].z, inp[1].z);
  {  // sampled this frame: clamp the history towards the neighbourhood AABB (always evaluated; selected per plane below)
    const f2 loR = p_log1p(mkf2(mn[0].x, mn[1].x)), loG = p_log1p(mkf2(mn[0].y, mn[1].y)), loB = p_log1p(mkf2(mn[0].z, mn[1].z));
    const f2 hiR = p_log1p(mkf2(mx[0].x, mx[1].x)), hiG = p_log1p(mkf2(mx[0].y, mx[1].y)), hiB = p_log1p(mkf2(mx[0].z, mx[1].z));
    const f2 clR = p_min(p_max(accR, loR), hiR), clG = p_min(p_max(accG, loG), hiG), clB = p_min(p_max(accB, loB), hiB);
    const f2 aggr = p_min(one, f2mul(conf, mkf2(1.0f, s.roughness)));
    const f2 ci = f2mul(mkf2(fminf(1.0f, fma_(s.moveFactor, 50.0f, a.clamp_intensity))), aggr);
    const f2 omci = f2sub(one, ci);
    const f2 nR = p_mix(accR, clR, ci, omci), nG = p_mix(accG, clG, ci, omci), nB = p_mix(accB, clB, ci, omci);
    const f2 dR = f2sub(nR, accR), dG = f2sub(nG, accG), dB = f2sub(nB, accB);
    const f2 l2 = f2fma(dB, dB, f2fma(dG, dG, f2mul(dR, dR)));
    const f2 cd = p_min(mkf2(fx_sqrt(f2lo(l2)), fx_sqrt(f2hi(l2))), one);
    const f2 accAs = f2mul(f2add(accA, one), f2sub(one, cd));
    // not sampled: inputTexel.rgb = accumulatedTexel.rgb, history untouched
    inR = p_sel(s0, s1, inR, accR); inG = p_sel(s0, s1, inG, accG); inB = p_sel(s0, s1, inB, accB);
    accR = p_sel(s0, s1, nR, accR); accG = p_sel(s0, s1, nG, accG); accB = p_sel(s0, s1, nB, accB);
    accA = p_sel(s0, s1, accAs, accA);
  }
  const f2 confidence = f2ex2(f2mul(f2lg2(conf), mkf2(a.confidence_power)));
  const f2 accumBlend = f2mul(f2sub(one, p_rcp(f2add(accA, one))), confidence);
  const float mv = (a.full_accumulate ? 1.0f : a.max_blend) * a.keep_data;
  float mvS = mv;
  if (s.roughness >= 0.0f && s.roughness < 0.1f) mvS = mixf(mv, mv * (s.roughness * 10.0f), fminf(100.0f * s.moveFactor, 1.0f));
  const f2 tmix = p_min(accumBlend, mkf2(mv, mvS));
  const f2 omt = f2sub(one, tmix);
  const f2 oa = p_min(mkf2(65536.0f), f2sub(p_rcp(omt), one));
  const f2 oR = p_expm1(p_mix(inR, accR, tmix, omt)), oG = p_expm1(p_mix(inG, accG, tmix, omt)), oB = p_expm1(p_mix(inB, accB, tmix, omt));
  out0 = make_float4(f2lo(oR), f2lo(oG), f2lo(oB), f2lo(oa));
  out1 = make_float4(f2hi(oR), f2hi(oG), f2hi(oB), f2hi(oa));
}

template <bool PEER>
__global__ void __launch_bounds__(kThreads, 4) ctemporal_kernel(const __grid_constant__ CTemporalArgs a) {
  int x, y;
  const bool in_rows = range_pixel(a.row0, a.row1, x, y);
  const bool active = x < a.W && y < a.H && in_rows;
  const int xc = min(x, a.W - 1), yc = min(y, a.H - 1);
  CTState s;
  s.vUv = pixel_uv(x, y, a.W, a.H);
  // getVelocityNormalDepth  reproject.frag:97-105
  const float4 vt = ld_f4(a.velocity, xc, yc);
  s.velocity = mk2(vt.x, vt.y);
  s.worldNormal = c_unpack_normal(vt.z);
  s.depth = vt.w;
  const float fwd = fwidth_f(s.depth);
  s.curvature = fx_length(fwidth_3(s.worldNormal));
  if (!active) return;
  if (s.depth == 1.0f && fwd == 0.0f) return;  // discard  temporal_reproject.frag:188-193 (the target keeps its texel)

  v4 inp[2];
  unpackTwoVec4(ld_f4(a.input, x, y), inp[0], inp[1]);
  bool sampled[2];
#pragma unroll
  for (int i = 0; i < 2; i++) {
    sampled[i] = inp[i].x >= 0.0f;
    const v3 c = c_log1p(vmax(xyz(inp[i]), mk3(0.0f)));
    inp[i] = mk4(c, inp[i].w);
  }
  s.worldPos = c_screen_to_world<true>(s.vUv, s.depth, a.cam.camera_matrix_world, a.cam.projection_inverse);
  s.rayLength = inp[1].w;
  s.roughness = clampf(inp[0].w, 0.0f, 1.0f);
  v3 ruvD, ruvS;
  {
    const float gz = a.cam.perspective ? (a.cam.near_plane * a.cam.far_plane) * fx_rcp((a.cam.far_plane - a.cam.near_plane) * s.depth - a.cam.far_plane)
                                       : orthographicDepthToViewZ(s.depth, a.cam.near_plane, a.cam.far_plane);
    const float distFactor = 1.0f + fx_rcp(fabsf(gz) + 1.0f);
    const v2 r = s.vUv - s.velocity;
    ruvD = mk3(r.x, r.y, c_validate(a, s, r, distFactor));
    const v2 h = c_reproject_hit(a, s);
    ruvS = mk3(h.x, h.y, c_validate(a, s, h, distFactor));
    if (ruvS.x == -1.0f) ruvS = ruvD;
  }
  s.moveFactor = fminf(dot(s.velocity, s.velocity) * 10000.0f, 1.0f);

  // neighbourhood AABBs: one merged 5x5 sweep on the packed fp16 pairs (see k_temporal.cu)
  v3 mn[2], mx[2];
  int radius[2] = {2, s.roughness < 0.25f ? 1 : 2};
#pragma unroll
  for (int i = 0; i < 2; i++) {
    const v3 inLin = c_expm1(xyz(inp[i]));
    mn[i] = inLin; mx[i] = inLin;
  }
  if (sampled[0] || sampled[1]) {
    const __half2 pinf = __floats2half2_rn(INFINITY, INFINITY), ninf = __floats2half2_rn(-INFINITY, -INFINITY);
    __half2 mn_rg[2] = {pinf, pinf}, mn_ba[2] = {pinf, pinf}, mx_rg[2] = {ninf, ninf}, mx_ba[2] = {ninf, ninf};
    for (int dy = -2; dy <= 2; dy++) {
      const int ty = clampi(y + dy, a.H);
#pragma unroll
      for (int dx = -2; dx <= 2; dx++) {
        const int tx = clampi(x + dx, a.W);
        const float4 e = ld_f4(a.input, tx, ty);
#pragma unroll
        for (int i = 0; i < 2; i++) {
          const unsigned urg = __float_as_uint(i ? e.z : e.x), uba = __float_as_uint(i ? e.w : e.y);
          const __half2 rg = *reinterpret_cast<const __half2*>(&urg), ba = *reinterpret_cast<const __half2*>(&uba);
          const bool inside = abs(dx) <= radius[i] && abs(dy) <= radius[i];
          if (inside && (__low2float(rg) - RFX_NON_ZERO_OFFSET) >= 0.0f) {
            mn_rg[i] = __hmin2(mn_rg[i], rg); mx_rg[i] = __hmax2(mx_rg[i], rg);
            mn_ba[i] = __hmin2(mn_ba[i], ba); mx_ba[i] = __hmax2(mx_ba[i], ba);
          }
        }
      }
    }
#pragma unroll
    for (int i = 0; i < 2; i++) {
      const v3 lo = mk3(__low2float(mn_rg[i]) - RFX_NON_ZERO_OFFSET, __high2float(mn_rg[i]) - RFX_NON_ZERO_OFFSET, __low2float(mn_ba[i]) - RFX_NON_ZERO_OFFSET);
      const v3 hi = mk3(__low2float(mx_rg[i]) - RFX_NON_ZERO_OFFSET, __high2float(mx_rg[i]) - RFX_NON_ZERO_OFFSET, __low2float(mx_ba[i]) - RFX_NON_ZERO_OFFSET);
      mn[i] = vmin(lo, mn[i]);
      mx[i] = vmax(hi, mx[i]);
    }
  }
  float4* o = (float4*)(a.out.p + ((unsigned)y * (unsigned)a.out.pitch + (unsigned)x * 32u));
  float4 o0, o1;
  c_temporal_planes<PEER>(a, s, ruvD, ruvS, inp, sampled, mn, mx, o0, o1);
  o[0] = o0;
  o[1] = o1;
}

cudaError_t launch_ctemporal(const CTemporalArgs& a, cudaStream_t s) {
  dim3 grid((a.W + kTileW - 1) / kTileW, row_tiles(a.row0, a.row1));
  if (a.hist.n > 1) ctemporal_kernel<true><<<grid, kThreads, 0, s>>>(a);
  else ctemporal_kernel<false><<<grid, kThreads, 0, s>>>(a);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------------------------
// K4 as a device function: constructGlobalIllumination (denoiser_compose_functions.glsl:53-107)
// ------------------------------------------------------------------------------------------------------------------
// The arithmetic is the exact K4's IEEE division / sqrt (k_denoise.cu: gi_compose_kernel): the two fp16 inputs already sit up to
// one fp16 ulp (9.8e-4) from the oracle's, so composed pixels crowd the 1e-3 line, and SFU reciprocals were measured to more than
// double the pixels outside it (DESIGN.md §2).  The perspective viewZ divides once, as perspectiveDepthToViewZ: near depth 1 the
// denominator cancels, and the reciprocal's second rounding moved composed pixels by up to 70 %.  The pixel-centre fetch is the centre
// texel (the literal LINEAR fetch would need the neighbours' dn texels, which other blocks of the fused last Poisson pass write; on
// 3840-wide frames it puts up to 8.8e-4 of the pixels outside 1e-3, tests/test_gpu_compose_options.py) and pow(x, 5) is multiplies.
RFX_D float4 c_compose(const CamD& cam, int x, int y, int W, int H, float4 g, float rough0, float depth, v3 dgi, v3 sgi) {
  const v2 vUv = pixel_uv(x, y, W, H);
  const v3 diffuse = xyz(floatToVec4(g.x));
  const v3 wn = unpackNormal(g.y);  // the exact packed normal (the nrdz copy carries the roughness code in its low mantissa bits)
  const float metalness = gb_metalness(g.z);
  const v4 e = floatToVec4(g.w);
  const float fexp = e.w * 255.0f - 128.0f;
  const v3 emissive = xyz(e) * exp2f(fexp);  // decodeRGBE8
  const v3 viewNormal = mul_dir_left(wn, cam.camera_matrix_world);
  const float gz = cam.perspective ? perspectiveDepthToViewZ(depth, cam.near_plane, cam.far_plane) : orthographicDepthToViewZ(depth, cam.near_plane, cam.far_plane);
  const float viewZ = -gz;
  const float clipW = cam.projection.m[2 * 4 + 3] * viewZ + cam.projection.m[3 * 4 + 3];
  v4 clip = mk4((vUv.x - 0.5f) * 2.0f, (vUv.y - 0.5f) * 2.0f, (viewZ - 0.5f) * 2.0f, 1.0f);
  clip = mk4(clip.x * clipW, clip.y * clipW, clip.z * clipW, clip.w * clipW);
  v3 viewPos = xyz(mul(cam.projection_inverse, clip));
  viewPos.z = -viewZ;
  const v3 viewDir = normalize(viewPos);
  const float roughness = rough0 * rough0;
  const v3 N = mul_dir_left(viewNormal, cam.view_matrix);
  v3 T, B;
  const v3 v = -viewDir;
  v3 V = mul_dir_left(v, cam.view_matrix);
  Onb(N, T, B);
  V = ToLocal(T, B, N, V);
  v3 Hh = SampleGGXVNDF_cs(V, roughness, roughness, 0.25f, -4.37113883e-08f, 1.0f);  // r2 = 0.25: (cos, sin) of fp32(pi/2)
  if (Hh.z < 0.0f) Hh = -Hh;
  v3 l = normalize(reflect(-V, Hh));
  l = ToWorld(T, B, N, l);
  l = xyz(mul(mk4(l, 1.0f), cam.camera_matrix_world));
  l = normalize(l);
  if (dot(viewNormal, l) < 0.0f) l = -l;
  const v3 h = normalize(v + l);
  const float VoH = fmaxf(1e-6f, dot(v, h));
  const v3 f0 = mix(mk3(0.04f), diffuse, metalness);
  const float omv = 1.0f - VoH, omv2 = omv * omv;
  const v3 F = f0 + (mk3(1.0f) - f0) * (omv2 * omv2 * omv);
  const v3 gi = diffuse * (1.0f - metalness) * (mk3(1.0f) - F) * dgi + sgi * F + emissive;
  return make_float4(gi.x, gi.y, gi.z, 1.0f);
}

// ------------------------------------------------------------------------------------------------------------------
// K3  Poisson pass on the interleaved planes.  FIRST: `in` = tr (fp32, NEAREST); else `in` = dn (fp16, LINEAR).
// Arithmetic = poisson_fast_kernel (k_denoise.cu): colours in log2 units, merged exponents.
// ------------------------------------------------------------------------------------------------------------------
RFX_D v3 cp_log1p(v3 c) { return mk3(fx_lg2(c.x + 1.0f), fx_lg2(c.y + 1.0f), fx_lg2(c.z + 1.0f)); }
#define CP_LUM_C (-0.06609580f) /* 0.125 * log2(ln 2) */
RFX_D float cp_lum(v3 c2) { return fx_ex2(fma_(0.125f, fx_lg2(dot(mk3(0.2125f, 0.7154f, 0.0721f), c2)), CP_LUM_C)); }

// The two planes ride in the two halves of packed fp32x2 registers (f2: .lo = diffuse plane, .hi = specular plane).
struct CTexel2 { f2 r, g, b, a; };
// TMA-staged tile of this block (cpoisson_tma_kernel): texel (x, y) of `in` / `nrdz` lives at ((y - y0) * bw + (x - x0)) * 16
struct SmemTile { const unsigned char* in; const unsigned char* nrdz; int x0, y0, bw; };
// INTERIOR: every tap of this block stays inside the image, so no index is clamped and the four bilinear corners are
// p, p + 16, p + pitch, p + pitch + 16 (immediate offsets off two address computations).
template <bool FIRST, bool ALPHA, bool INTERIOR, bool SMEM = false>
RFX_D CTexel2 cp_fetch(const CPoissonArgs& a, float fxn, float fyn, int nx, int ny, const SmemTile& st) {
  CTexel2 t;
  t.a = mkf2(0.0f);
  if (FIRST) {  // NEAREST fp32 pair
    const float4* p = (const float4*)(a.in.p + ((unsigned)ny * (unsigned)a.in.pitch + (unsigned)nx * 32u));
    const float4 u0 = __ldg(p), u1 = __ldg(p + 1);
    t.r = mkf2(u0.x, u1.x); t.g = mkf2(u0.y, u1.y); t.b = mkf2(u0.z, u1.z);
    if (ALPHA) t.a = mkf2(u0.w, u1.w);
  } else {      // LINEAR fp16 pair: one bilinear setup, one LDG.128 per corner (fxn = uv.x * W, the product bilin_setup forms)
    const float fx = fxn - 0.5f, fy = fyn - 0.5f;
    float x0f, y0f;
    const int ix = floor_i(fx, x0f), iy = floor_i(fy, y0f);
    const float ax = fx - x0f, ay = fy - y0f;
    const float w00 = (1.0f - ax) * (1.0f - ay), w10 = ax * (1.0f - ay), w01 = (1.0f - ax) * ay, w11 = ax * ay;
    uint4 t00, t10, t01, t11;
    if (SMEM) {  // the four corners from the staged tile (LDS.128)
      const unsigned char* p0 = st.in + (((iy - st.y0) * st.bw + (ix - st.x0)) << 4);
      const unsigned char* p1 = p0 + (st.bw << 4);
      t00 = *(const uint4*)p0; t10 = *(const uint4*)(p0 + 16); t01 = *(const uint4*)p1; t11 = *(const uint4*)(p1 + 16);
    } else if (INTERIOR) {
      const unsigned char* p0 = a.in.p + ((unsigned)iy * (unsigned)a.in.pitch + (unsigned)ix * 16u);
      const unsigned char* p1 = p0 + a.in.pitch;
      t00 = __ldg((const uint4*)p0); t10 = __ldg((const uint4*)(p0 + 16)); t01 = __ldg((const uint4*)p1); t11 = __ldg((const uint4*)(p1 + 16));
    } else {
      const int x0 = clamp_idx(ix, a.W - 1), x1 = clamp_idx(ix + 1, a.W - 1), y0 = clamp_idx(iy, a.H - 1), y1 = clamp_idx(iy + 1, a.H - 1);
      const unsigned r0 = (unsigned)y0 * (unsigned)a.in.pitch, r1 = (unsigned)y1 * (unsigned)a.in.pitch;
      t00 = __ldg((const uint4*)(a.in.p + (r0 + (unsigned)x0 * 16u))); t10 = __ldg((const uint4*)(a.in.p + (r0 + (unsigned)x1 * 16u)));
      t01 = __ldg((const uint4*)(a.in.p + (r1 + (unsigned)x0 * 16u))); t11 = __ldg((const uint4*)(a.in.p + (r1 + (unsigned)x1 * 16u)));
    }
    // weighted sum in the sampler's order: fma(t11, w11, fma(t01, w01, fma(t10, w10, t00 * w00)))
#define CP_BL(F, M0, M1) f2fma(mkf2(F(t11.M0), F(t11.M1)), mkf2(w11), f2fma(mkf2(F(t01.M0), F(t01.M1)), mkf2(w01), \
                         f2fma(mkf2(F(t10.M0), F(t10.M1)), mkf2(w10), f2mul(mkf2(F(t00.M0), F(t00.M1)), mkf2(w00)))))
    t.r = CP_BL(h_lo, x, z); t.g = CP_BL(h_hi, x, z); t.b = CP_BL(h_lo, y, w);
    if (ALPHA) t.a = CP_BL(h_hi, y, w);
#undef CP_BL
  }
  return t;
}
RFX_D f2 cp_lum2(f2 r, f2 g, f2 b) {  // luminance(): pow(dot(w, c), 0.125) on log2-unit colours, both planes
  const f2 d = f2fma(b, mkf2(0.0721f), f2fma(g, mkf2(0.7154f), f2mul(r, mkf2(0.2125f))));
  return f2ex2(f2fma(f2lg2(d), mkf2(0.125f), mkf2(CP_LUM_C)));
}

template <bool FIRST, bool COMPOSE, bool IMAGE, bool INTERIOR, bool SMEM = false>
RFX_D void cpoisson_body(const CPoissonArgs& a, int x, int y, float4 nc, float fwn, const SmemTile& st = SmemTile{}) {
  const v2 vUv = pixel_uv(x, y, a.W, a.H);
  const float depth = nc.w;
  const v3 normal = mk3(nc.x, nc.y, nc.z);
  const float roughness = nrdz_roughness(nc);
  const float resx = (float)a.W, resy = (float)a.H;
  f2 accr, accg, accb, tw = mkf2(1.0f), lumc, age, alpha;
  {
    const CTexel2 c = cp_fetch<FIRST, true, INTERIOR, SMEM>(a, vUv.x * resx, vUv.y * resy, x, y, st);
    alpha = c.a;
    age = f2ex2(f2mul(f2lg2(f2add(alpha, mkf2(1.0f))), mkf2(-1.2f * a.phi)));
    accr = f2lg2(f2fma(c.r, mkf2(1.0003f), mkf2(1.0f))); accg = f2lg2(f2fma(c.g, mkf2(1.0003f), mkf2(1.0f))); accb = f2lg2(f2fma(c.b, mkf2(1.0003f), mkf2(1.0f)));
    lumc = cp_lum2(accr, accg, accb);
  }
  const float glossiness = fmaxf(0.0f, 4.0f * (1.0f - roughness * 4.0f));
  const float sarg2 = (-glossiness * a.specular_phi) * C_LOG2E;   // specular plane only: w *= exp(-glossiness * specularPhi)
  const f2 sargp = mkf2(0.0f, sarg2), swdp = mkf2(1.0f, fx_ex2(sarg2 * 0.1f));
  const f2 nlphi2 = mkf2(-a.luma_phi * C_LOG2E);
  float flatness = 1.0f - fminf(fwn, 1.0f);
  flatness = flatness * flatness * 0.75f + 0.25f;
  const uchar4 bn = __ldg(a.blue.tex + blue_index(a.blue, x, y));
  const float2 sc = __ldg(a.rot_table + bn.x);
  const float k = a.radius * flatness;
  const float m00 = k * sc.y, m01 = k * -sc.x, m10 = k * sc.x, m11 = k * sc.y;
  const f2 oma = f2sub(mkf2(1.0f), age);
  const f2 agewd = f2mul(age, swdp);  // age * (1, specular share of pow(w, 0.1))

#pragma unroll
  for (int i = 0; i < 8; i++) {
    const float ox = a.tap_ox[i], oy = a.tap_oy[i];
    const v2 nuv = mk2(vUv.x + (m00 * ox + m10 * oy), vUv.y + (m01 * ox + m11 * oy));  // tap position: the oracle's arithmetic, op for op
    const float fxn = nuv.x * resx, fyn = nuv.y * resy;
    int nx = floor_i(fxn), ny = floor_i(fyn);
    if (!INTERIOR) { nx = clamp_idx(nx, a.W - 1); ny = clamp_idx(ny, a.H - 1); }
    const float4 nn = SMEM ? *(const float4*)(st.nrdz + (((ny - st.y0) * st.bw + (nx - st.x0)) << 4)) : ld_f4(a.nrdz, nx, ny);
    if (nn.w == 1.0f) continue;  // background tap: wBasic = 0
    const float normalDiff = 1.0f - fmaxf(dot(normal, mk3(nn.x, nn.y, nn.z)), 0.0f);
    const float depthDiff = 10000.0f * fabsf(depth - nn.w);
    const float roughnessDiff = fabsf(roughness - nrdz_roughness(nn));
    const float A2 = (-normalDiff * a.normal_phi - depthDiff * a.depth_phi - roughnessDiff * a.roughness_phi) * C_LOG2E;
    const float wdA = fx_ex2(A2 * 0.1f);
    const CTexel2 c = cp_fetch<FIRST, false, INTERIOR, SMEM>(a, fxn, fyn, nx, ny, st);
    const f2 lr = f2lg2(f2add(c.r, mkf2(1.0f))), lg = f2lg2(f2add(c.g, mkf2(1.0f))), lb = f2lg2(f2add(c.b, mkf2(1.0f)));
    const f2 dl = f2sub(lumc, cp_lum2(lr, lg, lb));
    const f2 lumaDiff = mkf2(fminf(fabsf(f2lo(dl)), 0.5f), fminf(fabsf(f2hi(dl)), 0.5f));
    const f2 wl = f2ex2(f2fma(lumaDiff, nlphi2, f2add(sargp, mkf2(A2))));         // w * lumaFactor
    const f2 wm = f2mul(f2fma(agewd, mkf2(wdA), f2mul(wl, oma)), age);            // mix(w * lumaFactor, pow(w, 0.1), age) * age
    const f2 w = mkf2(f2lo(wm) < 0.0001f ? 0.0f : f2lo(wm), f2hi(wm) < 0.0001f ? 0.0f : f2hi(wm));
    accr = f2fma(w, lr, accr); accg = f2fma(w, lg, accg); accb = f2fma(w, lb, accb);
    tw = f2add(tw, w);
  }
  const f2 inv = mkf2(fx_rcp(f2lo(tw)), fx_rcp(f2hi(tw)));
  const f2 orr = f2sub(f2ex2(f2mul(accr, inv)), mkf2(1.0f)), og = f2sub(f2ex2(f2mul(accg, inv)), mkf2(1.0f)), ob = f2sub(f2ex2(f2mul(accb, inv)), mkf2(1.0f));
  uint4 q;
  q.x = pack_h2(f2lo(orr), f2lo(og)); q.y = pack_h2(f2lo(ob), f2lo(alpha)); q.z = pack_h2(f2hi(orr), f2hi(og)); q.w = pack_h2(f2hi(ob), f2hi(alpha));
  *((uint4*)(a.out.p + ((unsigned)y * (unsigned)a.out.pitch + (unsigned)x * 16u))) = q;
  if (COMPOSE) {
    if (y >= a.crow0 && y < a.crow1) {  // K4 reads the fp16 texel just stored (DenoiserComposePass.js:66-67)
      const float4 g = ld_f4(a.gb, x, y);
      const float4 c = c_compose(a.cam, x, y, a.W, a.H, g, roughness, depth, mk3(h_lo(q.x), h_hi(q.x), h_lo(q.y)), mk3(h_lo(q.z), h_hi(q.z), h_lo(q.w)));
      st_f4(a.composed.p, a.composed.pitch, x, y, c);
      if (IMAGE) st_h4(a.k5.out.p, a.k5.out.pitch, x, y, ssgi_compose_lit(a.k5, x, y, depth, [&] { return c; }));  // K5 of the texel just stored
    }
  }
}

// K5 of a discarded (background: depth 1) pixel, which reads the scene texel only
RFX_D v4 k5_background(const SsgiComposeArgs& k5, int x, int y) {
  return ssgi_compose_lit(k5, x, y, 1.0f, [] { return make_float4(0.0f, 0.0f, 0.0f, 0.0f); });
}

// IMAGE (with COMPOSE): the composing pixels also store K5 of their composed texel into a.k5.out (the chain's compose stage)
template <bool FIRST, bool COMPOSE, bool IMAGE = false>
__global__ void __launch_bounds__(kThreads, 4) cpoisson_kernel(const __grid_constant__ CPoissonArgs a) {
  int x, y;
  const bool in_rows = range_pixel(a.row0, a.row1, x, y);
  const bool active = x < a.W && y < a.H && in_rows;
  const int xc = min(x, a.W - 1), yc = min(y, a.H - 1);
  const float4 nc = ld_f4(a.nrdz, xc, yc);
  const float depth = nc.w;
  const float fwd = fwidth_f(depth);
  const float fwn = fx_length(fwidth_3(mk3(nc.x, nc.y, nc.z)));
  if (!active) return;
  if (depth == 1.0f && fwd == 0.0f) {  // discard :129-132: the target keeps its texel (double-buffered targets: carry it forward)
    if (a.carry.local.p) {
      const unsigned off = (unsigned)y * (unsigned)a.carry.local.pitch + (unsigned)x * 16u;
      *((uint4*)(a.out.p + ((unsigned)y * (unsigned)a.out.pitch + (unsigned)x * 16u))) = *((const uint4*)(peer_row_base(a.carry, y) + off));
    }
    if (COMPOSE && a.composed_carry.local.p && y >= a.crow0 && y < a.crow1) {
      const unsigned off = (unsigned)y * (unsigned)a.composed_carry.local.pitch + (unsigned)x * 16u;
      st_f4(a.composed.p, a.composed.pitch, x, y, *((const float4*)(peer_row_base(a.composed_carry, y) + off)));
    }
    if (IMAGE && y >= a.crow0 && y < a.crow1) st_h4(a.k5.out.p, a.k5.out.pitch, x, y, k5_background(a.k5, x, y));
    return;
  }
  // block-uniform: can any tap of this 16x16 tile leave the image?
  int lx, ly;
  lane_to_pixel(threadIdx.x & 31, lx, ly);
  const int bx0 = blockIdx.x * kTileW, by0 = y - ((int)((threadIdx.x >> 6) << 2) + ly);
  const bool interior = bx0 - a.reach_x >= 0 && bx0 + kTileW - 1 + a.reach_x <= a.W - 1 && by0 - a.reach_y >= 0 && by0 + kTileH - 1 + a.reach_y <= a.H - 1;
  if (interior) cpoisson_body<FIRST, COMPOSE, IMAGE, true>(a, x, y, nc, fwn);
  else cpoisson_body<FIRST, COMPOSE, IMAGE, false>(a, x, y, nc, fwn);
}

template <bool FIRST>
static void cpoisson_go(const CPoissonArgs& a, dim3 grid, cudaStream_t s) {
  if (!a.compose) cpoisson_kernel<FIRST, false><<<grid, kThreads, 0, s>>>(a);
  else if (a.k5.out.p) cpoisson_kernel<FIRST, true, true><<<grid, kThreads, 0, s>>>(a);
  else cpoisson_kernel<FIRST, true><<<grid, kThreads, 0, s>>>(a);
}
cudaError_t launch_cpoisson(const CPoissonArgs& a, cudaStream_t s) {
  dim3 grid((a.W + kTileW - 1) / kTileW, row_tiles(a.row0, a.row1));
  if (a.first) cpoisson_go<true>(a, grid, s);
  else cpoisson_go<false>(a, grid, s);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------------------------
// K3 passes >= 1 with TMA staging (the experiment BASELINE.json's north_star asks for): an interior block stages the
// (16 + 2 reach_x) x (16 + 2 reach_y) texel tiles of `in` and `nrdz` its taps can touch into shared memory with two
// cp.async.bulk.tensor.2d loads completing on one mbarrier, then every tap reads LDS.128 instead of LDG.128.  Border blocks
// (TMA fills out-of-range texels with zeros, the samplers clamp to the edge) take the global path.  Same arithmetic, same
// bytes out.  Selected with RFX_K3_TMA=1 (the default).
// ------------------------------------------------------------------------------------------------------------------
RFX_D unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
RFX_D void mbar_init(unsigned long long* bar, unsigned count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count)); }
RFX_D void mbar_expect_tx(unsigned long long* bar, unsigned bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory"); }
RFX_D void mbar_wait(unsigned long long* bar, unsigned phase) {
  unsigned ok;
  do {
    asm volatile("{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}" : "=r"(ok) : "r"(smem_u32(bar)), "r"(phase) : "memory");
  } while (!ok);
}
RFX_D void tma_load_2d(void* dst, const CUtensorMap* map, int c0, int c1, unsigned long long* bar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(smem_u32(dst)), "l"(map), "r"(c0), "r"(c1),
               "r"(smem_u32(bar))
               : "memory");
}

template <bool COMPOSE, bool IMAGE = false>
__global__ void __launch_bounds__(kThreads, 4) cpoisson_tma_kernel(const __grid_constant__ CPoissonTmaArgs t) {
  extern __shared__ __align__(1024) unsigned char tile[];
  __shared__ unsigned long long bar;
  const CPoissonArgs& a = t.a;
  int x, y;
  const bool in_rows = range_pixel(a.row0, a.row1, x, y);
  const bool active = x < a.W && y < a.H && in_rows;
  int lx, ly;
  lane_to_pixel(threadIdx.x & 31, lx, ly);
  const int bx0 = blockIdx.x * kTileW, by0 = y - ((int)((threadIdx.x >> 6) << 2) + ly);
  // block-uniform: every texel of the staged tile exists (no clamping anywhere in this block); box_w may exceed 16 + 2 reach_x by
  // one texel: an ODD row pitch (in 16-byte texels) spreads the rows of the tile over the shared-memory banks
  const bool interior = bx0 - a.reach_x >= 0 && bx0 - a.reach_x + t.box_w - 1 <= a.W - 1 && by0 - a.reach_y >= 0 && by0 + kTileH - 1 + a.reach_y <= a.H - 1;
  SmemTile st{};
  if (interior) {
    const unsigned tile_bytes = (unsigned)t.box_w * (unsigned)t.box_h * 16u;
    const unsigned off2 = (tile_bytes + 127u) & ~127u;  // TMA destinations are 128-byte aligned
    st.in = tile; st.nrdz = tile + off2; st.x0 = bx0 - a.reach_x; st.y0 = by0 - a.reach_y; st.bw = t.box_w;
    if (threadIdx.x == 0) {
      mbar_init(&bar, 1);
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      mbar_expect_tx(&bar, 2u * tile_bytes);
      tma_load_2d(tile, &t.map_in, st.x0 * 4, st.y0, &bar);                  // coordinates in 4-byte elements: 4 per 16-byte texel
      tma_load_2d(tile + off2, &t.map_nrdz, st.x0 * 4, st.y0, &bar);
    }
  }
  const int xc = min(x, a.W - 1), yc = min(y, a.H - 1);
  const float4 nc = ld_f4(a.nrdz, xc, yc);
  const float depth = nc.w;
  const float fwd = fwidth_f(depth);
  const float fwn = fx_length(fwidth_3(mk3(nc.x, nc.y, nc.z)));
  if (interior) mbar_wait(&bar, 0);  // every thread waits (also the ones that leave below): the tile must have landed before the block can retire
  if (!active) return;
  if (depth == 1.0f && fwd == 0.0f) {
    if (a.carry.local.p) {
      const unsigned off = (unsigned)y * (unsigned)a.carry.local.pitch + (unsigned)x * 16u;
      *((uint4*)(a.out.p + ((unsigned)y * (unsigned)a.out.pitch + (unsigned)x * 16u))) = *((const uint4*)(peer_row_base(a.carry, y) + off));
    }
    if (COMPOSE && a.composed_carry.local.p && y >= a.crow0 && y < a.crow1) {
      const unsigned off = (unsigned)y * (unsigned)a.composed_carry.local.pitch + (unsigned)x * 16u;
      st_f4(a.composed.p, a.composed.pitch, x, y, *((const float4*)(peer_row_base(a.composed_carry, y) + off)));
    }
    if (IMAGE && y >= a.crow0 && y < a.crow1) st_h4(a.k5.out.p, a.k5.out.pitch, x, y, k5_background(a.k5, x, y));
    return;
  }
  if (interior) cpoisson_body<false, COMPOSE, IMAGE, true, true>(a, x, y, nc, fwn, st);
  else cpoisson_body<false, COMPOSE, IMAGE, false, false>(a, x, y, nc, fwn);
}

static constexpr size_t kTmaSmemCap = 100 * 1024;  // dynamic shared memory cpoisson_tma_kernel may take
static size_t cpoisson_tma_smem(int box_w, int box_h) {  // the `in` tile, then the `nrdz` tile at the next 128-byte boundary
  const size_t tile_bytes = (size_t)box_w * box_h * 16;
  return ((tile_bytes + 127) & ~(size_t)127) + tile_bytes;
}

bool cpoisson_tma_fits(int box_w, int box_h) {
  return box_w * 4 <= 256 && box_h <= 256 && cpoisson_tma_smem(box_w, box_h) <= kTmaSmemCap;  // box rows count 4-byte elements, 4 per texel
}

cudaError_t launch_cpoisson_tma(const CPoissonTmaArgs& t, cudaStream_t s) {
  if (!cpoisson_tma_fits(t.box_w, t.box_h)) return cudaErrorInvalidValue;
  dim3 grid((t.a.W + kTileW - 1) / kTileW, row_tiles(t.a.row0, t.a.row1));
  const size_t smem = cpoisson_tma_smem(t.box_w, t.box_h);
  // the shared-memory limit is an attribute of the kernel on the CURRENT device: raise it once on every device that launches it
  static bool attr_set[64] = {};
  int dev = 0;
  const cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  if (dev >= 64 || !attr_set[dev]) {
    cudaFuncSetAttribute(cpoisson_tma_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kTmaSmemCap);
    cudaFuncSetAttribute(cpoisson_tma_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kTmaSmemCap);
    cudaFuncSetAttribute(cpoisson_tma_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kTmaSmemCap);
    if (dev < 64) attr_set[dev] = true;
  }
  if (!t.a.compose) cpoisson_tma_kernel<false><<<grid, kThreads, smem, s>>>(t);
  else if (t.a.k5.out.p) cpoisson_tma_kernel<true, true><<<grid, kThreads, smem, s>>>(t);
  else cpoisson_tma_kernel<true><<<grid, kThreads, smem, s>>>(t);
  return cudaGetLastError();
}

// stand-alone K4 (denoiseIterations == 0: no Poisson pass to ride on); IMAGE as cpoisson_kernel's
template <bool IMAGE>
__global__ void __launch_bounds__(kThreads) ccompose_kernel(const __grid_constant__ CComposeArgs a) {
  int x, y;
  const bool in_rows = range_pixel(a.row0, a.row1, x, y);
  const bool active = x < a.W && y < a.H && in_rows;
  const int xc = min(x, a.W - 1), yc = min(y, a.H - 1);
  const float4 nc = ld_f4(a.nrdz, xc, yc);
  const float fwd = fwidth_f(nc.w);
  if (!active) return;
  if (nc.w == 1.0f && fwd == 0.0f) {
    if (a.composed_carry.local.p) {
      const unsigned off = (unsigned)y * (unsigned)a.composed_carry.local.pitch + (unsigned)x * 16u;
      st_f4(a.composed.p, a.composed.pitch, x, y, *((const float4*)(peer_row_base(a.composed_carry, y) + off)));
    }
    if (IMAGE) st_h4(a.k5.out.p, a.k5.out.pitch, x, y, k5_background(a.k5, x, y));
    return;
  }
  const uint4 q = __ldg((const uint4*)(a.dn.p + ((unsigned)y * (unsigned)a.dn.pitch + (unsigned)x * 16u)));
  const float4 g = ld_f4(a.gb, x, y);
  const float4 c = c_compose(a.cam, x, y, a.W, a.H, g, nrdz_roughness(nc), nc.w, mk3(h_lo(q.x), h_hi(q.x), h_lo(q.y)), mk3(h_lo(q.z), h_hi(q.z), h_lo(q.w)));
  st_f4(a.composed.p, a.composed.pitch, x, y, c);
  if (IMAGE) st_h4(a.k5.out.p, a.k5.out.pitch, x, y, ssgi_compose_lit(a.k5, x, y, nc.w, [&] { return c; }));
}
cudaError_t launch_ccompose(const CComposeArgs& a, cudaStream_t s) {
  dim3 grid((a.W + kTileW - 1) / kTileW, row_tiles(a.row0, a.row1));
  if (a.k5.out.p) ccompose_kernel<true><<<grid, kThreads, 0, s>>>(a);
  else ccompose_kernel<false><<<grid, kThreads, 0, s>>>(a);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------------------------
// chain_output() views: interleaved -> the reference's plane formats
// ------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) split_tr_kernel(PV tr, OutV o0, OutV o1, int W, int H) {
  const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (x >= W || y >= H) return;
  const float4* p = (const float4*)(tr.p + ((unsigned)y * (unsigned)tr.pitch + (unsigned)x * 32u));
  st_f4(o0.p, o0.pitch, x, y, p[0]);
  st_f4(o1.p, o1.pitch, x, y, p[1]);
}
__global__ void __launch_bounds__(256) split_dn_kernel(PV dn, OutV o0, OutV o1, int W, int H) {
  const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (x >= W || y >= H) return;
  const uint4 q = *((const uint4*)(dn.p + ((unsigned)y * (unsigned)dn.pitch + (unsigned)x * 16u)));
  *((uint2*)(o0.p + ((unsigned)y * (unsigned)o0.pitch + (unsigned)x * 8u))) = make_uint2(q.x, q.y);
  *((uint2*)(o1.p + ((unsigned)y * (unsigned)o1.pitch + (unsigned)x * 8u))) = make_uint2(q.z, q.w);
}
cudaError_t launch_split_tr(PV tr, OutV o0, OutV o1, int W, int H, cudaStream_t s) {
  split_tr_kernel<<<dim3((W + 31) / 32, (H + 7) / 8), 256, 0, s>>>(tr, o0, o1, W, H);
  return cudaGetLastError();
}
cudaError_t launch_split_dn(PV dn, OutV o0, OutV o1, int W, int H, cudaStream_t s) {
  split_dn_kernel<<<dim3((W + 31) / 32, (H + 7) / 8), 256, 0, s>>>(dn, o0, o1, W, H);
  return cudaGetLastError();
}

}  // namespace rfx
