// k_temporal.cu — K2 temporal reprojection / accumulation (sm_90a).
//
// Replaces the fullscreen draw of reference src/temporal-reproject/TemporalReprojectPass.js:192-193
// (shader src/temporal-reproject/shader/temporal_reproject.frag:178-208 + reproject.frag).
// Used with 2 planes (SSGI: diffuse + specular, packed fp16x8 input) and with 1 plane (TRAA).
//
// Structure vs the shader: the two per-plane neighbourhood-AABB loops (reproject.frag:53-81) read the
// same packed texels, so they are merged into ONE 5x5 sweep that unpacks each texel once and feeds both
// planes' min/max (the specular plane only inside its 3x3 / 5x5 radius) — same values, half the loads.
// FAST = true moves log/exp/pow to the SFU pipe (lg2/ex2.approx).
#include "rfx_kernels.h"

namespace rfx {

RFX_D float t_lg2a(float x) { float r; asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
RFX_D float t_ex2a(float x) { float r; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
#define T_LN2 0.69314718055994530942f
#define T_LOG2E 1.44269504088896340736f

struct TState {  // the shader's invocation globals (reproject.frag:3-7)
  v2 vUv, velocity;
  v3 worldNormal, worldPos;
  float depth, curvature, viewAngle, rayLength, roughness, moveFactor;
};

RFX_D v3 screenSpaceToWorldSpace(v2 uv, float depth, const M4& world, const M4& projInv) {  // reproject.frag:21-28
  const v4 ndc = mk4((uv.x - 0.5f) * 2.0f, (uv.y - 0.5f) * 2.0f, (depth - 0.5f) * 2.0f, 1.0f);
  const v4 clip = mul(projInv, ndc);
  const v4 view = mul(world, clip / clip.w);
  return xyz(view);
}

template <bool LOG, bool FAST>
RFX_D v3 transformColor(v3 c) {  // reproject.frag:42
  if (!LOG) return c;
  if (FAST) return mk3(t_lg2a(c.x + 1.0f) * T_LN2, t_lg2a(c.y + 1.0f) * T_LN2, t_lg2a(c.z + 1.0f) * T_LN2);
  return mk3(logcr(c.x + 1.0f), logcr(c.y + 1.0f), logcr(c.z + 1.0f));
}
template <bool LOG, bool FAST>
RFX_D v3 undoColorTransform(v3 c) {  // :43
  if (!LOG) return c;
  if (FAST) return mk3(t_ex2a(c.x * T_LOG2E) - 1.0f, t_ex2a(c.y * T_LOG2E) - 1.0f, t_ex2a(c.z * T_LOG2E) - 1.0f);
  return mk3(expcr(c.x) - 1.0f, expcr(c.y) - 1.0f, expcr(c.z) - 1.0f);
}
template <bool FAST>
RFX_D float tpow(float x, float p) { return FAST ? t_ex2a(p * t_lg2a(x)) : powcr(x, p); }

RFX_D float getViewZ(const TemporalArgs& a, float d) {
  return a.cam.perspective ? perspectiveDepthToViewZ(d, a.cam.near_plane, a.cam.far_plane) : orthographicDepthToViewZ(d, a.cam.near_plane, a.cam.far_plane);
}

// validateReprojectedUV  reproject.frag:130-167
template <bool FAST>
RFX_D float validateReprojectedUV(const TemporalArgs& a, const TState& s, v2 ruv, float distFactor) {
  if (ruv.x > 1.0f || ruv.x < 0.0f || ruv.y > 1.0f || ruv.y < 0.0f) return 0.0f;
  const float4 t = tex_f4_nearest(a.velocity, ruv);
  const v3 lastWorldNormal = unpackNormal(t.z);
  const float lastDepth = t.w;
  const v3 lastWorldPos = screenSpaceToWorldSpace(ruv, lastDepth, a.prev_world, a.prev_proj_inv);
  // (lastViewAngle / angleMix are computed by the shader but never used)
  const v3 dpos = s.worldPos - lastWorldPos;
  float disoccl = 0.0f;
  if (FAST) {
    disoccl += length(dpos) * 0.1f * distFactor;
    disoccl += fabsf(dot(dpos, s.worldNormal)) * 0.05f * distFactor;
  } else {
    disoccl += length(dpos) / 10.0f * distFactor;
    disoccl += fabsf(dot(dpos, s.worldNormal)) / 20.0f * distFactor;
  }
  disoccl += fminf(1.0f - dot(s.worldNormal, lastWorldNormal), 1.0f) / 1.0f * distFactor;
  float confidence = 1.0f - fminf(disoccl, 1.0f);
  confidence = fmaxf(confidence, 0.0f);
  return tpow<FAST>(confidence, a.confidence_power);
}

// reprojectHitPoint  reproject.frag:169-193
RFX_D v2 reprojectHitPoint(const TemporalArgs& a, const TState& s) {
  if (s.curvature > 0.05f || s.rayLength < 0.01f) return mk2(-1.0f, -1.0f);
  const v3 cameraPos = mk3(a.camera_pos[0], a.camera_pos[1], a.camera_pos[2]);
  const v3 cameraRay = normalize(s.worldPos - cameraPos);
  const v3 hit = cameraPos + cameraRay * s.rayLength;
  const v4 rh = mul(a.prev_proj_view, mk4(hit, 1.0f));
  const v2 q = mk2(rh.x, rh.y) / rh.w;
  return mk2(q.x * 0.5f + 0.5f, q.y * 0.5f + 0.5f);
}

template <bool HLIN>
RFX_D v4 fetch_hist(const TemporalArgs& a, const PV& t, v2 uv) {
  if (a.hist_f32) return HLIN ? tex_f4_linear(t, uv) : f4v(tex_f4_nearest(t, uv));  // block-uniform: the FloatType FramebufferTexture history
  return HLIN ? tex_h4_linear(t, uv) : tex_h4_nearest(t, uv);
}
template <bool HLIN>
RFX_D v4 fetch_hist(const TemporalArgs&, const PeerPV& t, v2 uv) {  // the fused TRAA tail: RGBA16F LINEAR, rows on their owners
  static_assert(HLIN, "the TRAA history is sampled LINEAR");
  return peer_h4_linear(t, uv);
}

// the per-pass chain in a row-sharded group: its history (RGBA16F `dn`, or the RGBA32F temporal target) with rows on their owners
struct PeerHist {
  const PeerPV& p;
};
template <bool HLIN>
RFX_D v4 fetch_hist(const TemporalArgs& a, const PeerHist& t, v2 uv) {
  static_assert(HLIN, "the chain's history is sampled LINEAR");
  return a.hist_f32 ? peer_f4_linear(t.p, uv) : peer_h4_linear(t.p, uv);
}

// BiCubicCatmullRom5Tap  reproject.frag:212-255
template <bool HLIN, class Hist>
RFX_D v4 catmull5(const TemporalArgs& a, const Hist& tex, v2 P) {
  const v2 inv = mk2(a.inv_w, a.inv_h);
  const v2 UV = P / inv;
  const v2 tc = mk2(floorf(UV.x - 0.5f) + 0.5f, floorf(UV.y - 0.5f) + 0.5f);
  const v2 f = UV - tc;
  const v2 f2 = f * f;
  const v2 f3 = f2 * f;
  const v2 w0 = f2 - 0.5f * (f3 + f);
  const v2 w1 = 1.5f * f3 - 2.5f * f2 + mk2(1.0f, 1.0f);
  const v2 w3 = 0.5f * (f3 - f2);
  const v2 w2 = mk2(1.0f, 1.0f) - w0 - w1 - w3;
  const v2 W0 = w0, W1 = w1 + w2, W2 = w3;
  const v2 S0 = (tc - mk2(1.0f, 1.0f)) * inv, S1 = (tc + w2 / W1) * inv, S2 = (tc + mk2(2.0f, 2.0f)) * inv;
  const float sw0 = W1.x * W0.y, sw1 = W0.x * W1.y, sw2 = W1.x * W1.y, sw3 = W2.x * W1.y, sw4 = W1.x * W2.y;
  const v4 Ct = fetch_hist<HLIN>(a, tex, mk2(S1.x, S0.y)), Cl = fetch_hist<HLIN>(a, tex, mk2(S0.x, S1.y)), Cc = fetch_hist<HLIN>(a, tex, mk2(S1.x, S1.y)),
           Cr = fetch_hist<HLIN>(a, tex, mk2(S2.x, S1.y)), Cb = fetch_hist<HLIN>(a, tex, mk2(S1.x, S2.y));
  const float wm = 1.0f / (sw0 + sw1 + sw2 + sw3 + sw4);
  v4 r;
  r.x = fmaxf(((((Ct.x * sw0 + Cl.x * sw1) + Cc.x * sw2) + Cr.x * sw3) + Cb.x * sw4) * wm, 0.0f);
  r.y = fmaxf(((((Ct.y * sw0 + Cl.y * sw1) + Cc.y * sw2) + Cr.y * sw3) + Cb.y * sw4) * wm, 0.0f);
  r.z = fmaxf(((((Ct.z * sw0 + Cl.z * sw1) + Cc.z * sw2) + Cr.z * sw3) + Cb.z * sw4) * wm, 0.0f);
  r.w = fmaxf(((((Ct.w * sw0 + Cl.w * sw1) + Cc.w * sw2) + Cr.w * sw3) + Cb.w * sw4) * wm, 0.0f);
  return r;
}

// getVelocityNormalDepth  reproject.frag:97-105 (the quad derivatives of depth / normal are taken by the caller)
RFX_D void temporal_state(const TemporalArgs& a, int x, int y, int xc, int yc, TState& s) {
  s.vUv = pixel_uv(x, y, a.W, a.H);
  s.roughness = 1.0f; s.moveFactor = 0.0f; s.rayLength = 0.0f;
  const float4 vt = ld_f4(a.velocity, xc, yc);
  s.velocity = mk2(vt.x, vt.y);
  s.worldNormal = unpackNormal(vt.z);
  s.depth = vt.w;
}

// output of plane i at (x, y) into out0 / out1
struct PlaneStore {
  const TemporalArgs& a;
  int x, y;
  RFX_D void operator()(int i, v4 v) const {
    const OutV& o = i == 0 ? a.out0 : a.out1;
    if (a.out_half) st_h4(o.p, o.pitch, x, y, v);
    else st_f4(o.p, o.pitch, x, y, make_float4(v.x, v.y, v.z, v.w));
  }
};

// K2 of one pixel once its quad derivatives are known (fwd = fwidth(depth), s.curvature; the TRAA form, ITYPE DIFFUSE, reads
// neither).  `in` samples the RGBA16F input, h0 / h1 are the history planes, store(i, v) receives plane i.  temporal_kernel and
// the fused TRAA tail (ctraa_kernel) both run this code, so their arithmetic cannot differ.
template <int TC, int ITYPE, bool LOG, bool HLIN, bool FAST, class In, class Hist, class Store>
RFX_D void temporal_px(const TemporalArgs& a, const In& in, const Hist& h0, const Hist& h1, TState& s, float fwd, int x, int y, const Store& store) {
  // getTexels + preprocessInput  temporal_reproject.frag:124-145
  v4 inp[2];
  bool sampled[2] = {false, false};
  if (ITYPE == RFX_INPUT_DIFFUSE_SPECULAR) {
    unpackTwoVec4(a.in_scaled ? tex_f4_nearest(a.input, s.vUv) : ld_f4(a.input, x, y), inp[0], inp[1]);
  } else if (a.input_half) {
    inp[0] = in.linear(s.vUv);  // composer buffer: LINEAR, fetched at the pixel centre
  } else {
    inp[0] = f4v(a.in_scaled ? tex_f4_nearest(a.input, s.vUv) : ld_f4(a.input, x, y));
  }
  constexpr int NIN = ITYPE == RFX_INPUT_DIFFUSE_SPECULAR ? 2 : 1;
#pragma unroll
  for (int i = 0; i < NIN; i++) {
    sampled[i] = inp[i].x >= 0.0f;
    const v3 c = transformColor<LOG, FAST>(vmax(xyz(inp[i]), mk3(0.0f)));
    inp[i] = mk4(c, inp[i].w);
  }
  if (ITYPE != RFX_INPUT_DIFFUSE) {
    if (s.depth == 1.0f && fwd == 0.0f) return;  // discard :188-193
  }
  // computeGVariables :147-153 (viewDir / viewAngle only feed the unused angleMix)
  s.worldPos = screenSpaceToWorldSpace(s.vUv, s.depth, a.cam.camera_matrix_world, a.cam.projection_inverse);
  // getRoughnessRayLength :167-176
  if (ITYPE == RFX_INPUT_DIFFUSE_SPECULAR) {
    s.rayLength = inp[1].w;
    s.roughness = clampf(inp[0].w, 0.0f, 1.0f);
  } else if (ITYPE == RFX_INPUT_SPECULAR) {
    const v2 d = unpackHalf2x16(__float_as_uint(inp[0].w));
    s.rayLength = d.x;
    s.roughness = clampf(d.y, 0.0f, 1.0f);
  }
  // computeReprojectedUv :155-165
  v3 ruvD, ruvS;
  {
    const float viewZ = fabsf(getViewZ(a, s.depth));
    const float distFactor = 1.0f + 1.0f / (viewZ + 1.0f);
    const v2 r = s.vUv - s.velocity;
    ruvD = mk3(r.x, r.y, validateReprojectedUV<FAST>(a, s, r, distFactor));
    ruvS = mk3(-1.0f);
    if (ITYPE != RFX_INPUT_DIFFUSE) {
      const v2 h = reprojectHitPoint(a, s);
      ruvS = mk3(h.x, h.y, validateReprojectedUV<FAST>(a, s, h, distFactor));
      if (ruvS.x == -1.0f) ruvS = ruvD;
    }
  }
  s.moveFactor = fminf(dot(s.velocity, s.velocity) * 10000.0f, 1.0f);

  const int rs[2] = {a.rs0, a.rs1};
  // ---- neighbourhood AABBs (clampNeighborhood / getNeighborhoodAABB, reproject.frag:53-95), one merged sweep
  v3 mn[2], mx[2];
  int radius[2];
  bool need_sweep = false;
#pragma unroll
  for (int i = 0; i < TC; i++) {
    const v3 inLin = undoColorTransform<LOG, FAST>(xyz(inp[i]));
    mn[i] = inLin; mx[i] = inLin;
    radius[i] = (rs[i] != 0 && s.roughness < 0.25f) ? 1 : 2;
    need_sweep = need_sweep || sampled[i];
  }
  if (need_sweep) {
    if (ITYPE == RFX_INPUT_DIFFUSE_SPECULAR) {
      // neighborUv = vUv + (dx,dy)*invTexSize lands on texel (x+dx, y+dy) (clamped): direct addressing.  The packed texel holds
      // fp16 pairs and x -> fl(x - 1e-4) is monotonic, so min/max run on the packed halves (HMNMX2) and the offset is removed
      // once at the end — same values as unpacking every texel to fp32 first, a third of the instructions.
      const __half2 pinf = __floats2half2_rn(INFINITY, INFINITY), ninf = __floats2half2_rn(-INFINITY, -INFINITY);
      __half2 mn_rg[2] = {pinf, pinf}, mn_ba[2] = {pinf, pinf}, mx_rg[2] = {ninf, ninf}, mx_ba[2] = {ninf, ninf};
      for (int dy = -2; dy <= 2; dy++) {
        const int ty = clampi(y + dy, a.H);
#pragma unroll
        for (int dx = -2; dx <= 2; dx++) {
          const int tx = clampi(x + dx, a.W);
          // a smaller SSGI target (resolutionScale < 1): the shader's literal NEAREST fetch at vUv + (dx, dy) * invTexSize
          const float4 e = a.in_scaled ? tex_f4_nearest(a.input, mk2(s.vUv.x + (float)dx * a.inv_w, s.vUv.y + (float)dy * a.inv_h)) : ld_f4(a.input, tx, ty);
#pragma unroll
          for (int i = 0; i < TC; i++) {
            const unsigned urg = __float_as_uint(rs[i] != 0 ? e.z : e.x), uba = __float_as_uint(rs[i] != 0 ? e.w : e.y);
            const __half2 rg = *reinterpret_cast<const __half2*>(&urg), ba = *reinterpret_cast<const __half2*>(&uba);
            const bool inside = abs(dx) <= radius[i] && abs(dy) <= radius[i];
            if (inside && (__low2float(rg) - RFX_NON_ZERO_OFFSET) >= 0.0f) {  // neighborTexel.r >= 0.
              mn_rg[i] = __hmin2(mn_rg[i], rg); mx_rg[i] = __hmax2(mx_rg[i], rg);
              mn_ba[i] = __hmin2(mn_ba[i], ba); mx_ba[i] = __hmax2(mx_ba[i], ba);
            }
          }
        }
      }
#pragma unroll
      for (int i = 0; i < TC; i++) {
        const v3 lo = mk3(__low2float(mn_rg[i]) - RFX_NON_ZERO_OFFSET, __high2float(mn_rg[i]) - RFX_NON_ZERO_OFFSET, __low2float(mn_ba[i]) - RFX_NON_ZERO_OFFSET);
        const v3 hi = mk3(__low2float(mx_rg[i]) - RFX_NON_ZERO_OFFSET, __high2float(mx_rg[i]) - RFX_NON_ZERO_OFFSET, __low2float(mx_ba[i]) - RFX_NON_ZERO_OFFSET);
        mn[i] = vmin(lo, mn[i]);
        mx[i] = vmax(hi, mx[i]);
      }
    } else {
      for (int dx = -radius[0]; dx <= radius[0]; dx++)
        for (int dy = -radius[0]; dy <= radius[0]; dy++) {
          const v2 nuv = mk2(s.vUv.x + (float)dx * a.inv_w, s.vUv.y + (float)dy * a.inv_h);
          const v4 nt = a.input_half ? in.linear(nuv) : f4v(tex_f4_nearest(a.input, nuv));
          if (nt.x >= 0.0f) { mn[0] = vmin(xyz(nt), mn[0]); mx[0] = vmax(xyz(nt), mx[0]); }
        }
    }
  }

#pragma unroll
  for (int i = 0; i < TC; i++) {
    const bool spec = rs[i] != 0;
    const v3 uvc = spec ? ruvS : ruvD;
    const Hist& hist = i == 0 ? h0 : h1;
    // reproject()  temporal_reproject.frag:83-122
    const v4 acc = catmull5<HLIN>(a, hist, mk2(uvc.x, uvc.y));
    v3 accRgb = transformColor<LOG, FAST>(xyz(acc));
    float accA = acc.w;
    v3 inRgb = xyz(inp[i]);
    if (!sampled[i]) {
      inRgb = accRgb;
    } else {
      accA += 1.0f;
      const v3 lo = transformColor<LOG, FAST>(mn[i]), hi = transformColor<LOG, FAST>(mx[i]);
      const v3 clamped = mk3(clampf(accRgb.x, lo.x, hi.x), clampf(accRgb.y, lo.y, hi.y), clampf(accRgb.z, lo.z, hi.z));
      const float r = spec ? s.roughness : 1.0f;
      const float clampAggressiveness = fminf(1.0f, uvc.z * r);
      const float clampIntensity = mixf(0.0f, fminf(1.0f, s.moveFactor * 50.0f + a.clamp_intensity), clampAggressiveness);
      const v3 newColor = mix(accRgb, clamped, clampIntensity);
      const float colorDiff = fminf(length(newColor - accRgb), 1.0f);
      accA *= 1.0f - colorDiff;
      accRgb = newColor;
    }
    // accumulate()  temporal_reproject.frag:42-79
    const float confidence = tpow<FAST>(uvc.z, a.confidence_power);
    float accumBlend = 1.0f - 1.0f / (accA + 1.0f);
    accumBlend = mixf(0.0f, accumBlend, confidence);
    float maxValue = (a.full_accumulate ? 1.0f : a.max_blend) * a.keep_data;
    if (ITYPE != RFX_INPUT_DIFFUSE) {
      if (spec && s.roughness >= 0.0f && s.roughness < 0.1f) {
        const float maxRoughnessValue = mixf(0.0f, maxValue, s.roughness / 0.1f);
        maxValue = mixf(maxValue, maxRoughnessValue, fminf(100.0f * s.moveFactor, 1.0f));
      }
    }
    const float tmix = fminf(accumBlend, maxValue);
    float oa = 1.0f / (1.0f - tmix) - 1.0f;
    oa = fminf(65536.0f, oa);
    const v3 orgb = undoColorTransform<LOG, FAST>(mix(inRgb, accRgb, tmix));
    store(i, mk4(orgb, oa));
  }
}

template <int TC, int ITYPE, bool LOG, bool HLIN, bool FAST>
#ifndef RFX_K2_MIN_BLOCKS
#define RFX_K2_MIN_BLOCKS 4  // tools/sweep_occupancy.sh sweeps it
#endif
__global__ void __launch_bounds__(kThreads, RFX_K2_MIN_BLOCKS) temporal_kernel(const __grid_constant__ TemporalArgs a) {
  int x, y;
  const bool in_rows = range_pixel(a.row0, a.row1, x, y);
  const bool active = x < a.W && y < a.H && in_rows;
  TState s;
  temporal_state(a, x, y, min(x, a.W - 1), min(y, a.H - 1), s);
  const float fwd = fwidth_f(s.depth);
  s.curvature = length(fwidth_3(s.worldNormal));  // getCurvature :265-269
  if (!active) return;
  temporal_px<TC, ITYPE, LOG, HLIN, FAST>(a, PlaneH4{a.input}, a.hist0, a.hist1, s, fwd, x, y, PlaneStore{a, x, y});
}

// K2 with the history read on the owners and the carry of discarded pixels (TemporalPeer).  temporal_px returns without a store
// exactly where the shader discards, so a pixel whose planes were not stored copies last frame's texels of out0 / out1.
struct StoreSeen {
  PlaneStore s;
  bool* seen;
  RFX_D void operator()(int i, v4 v) const { *seen = true; s(i, v); }
};
template <int TC, int ITYPE, bool LOG>
__global__ void __launch_bounds__(kThreads, RFX_K2_MIN_BLOCKS) temporal_peer_kernel(const __grid_constant__ TemporalArgs a, const __grid_constant__ TemporalPeer p) {
  int x, y;
  const bool in_rows = range_pixel(a.row0, a.row1, x, y);
  const bool active = x < a.W && y < a.H && in_rows;
  TState s;
  temporal_state(a, x, y, min(x, a.W - 1), min(y, a.H - 1), s);
  const float fwd = fwidth_f(s.depth);
  s.curvature = length(fwidth_3(s.worldNormal));
  if (!active) return;
  bool seen = false;
  temporal_px<TC, ITYPE, LOG, true, true>(a, PlaneH4{a.input}, PeerHist{p.hist0}, PeerHist{p.hist1}, s, fwd, x, y, StoreSeen{PlaneStore{a, x, y}, &seen});
  if (ITYPE != RFX_INPUT_DIFFUSE && !seen) {
    if (a.out_half) { carry_texel<8>(p.carry.p[0], a.out0, x, y); if (TC == 2) carry_texel<8>(p.carry.p[1], a.out1, x, y); }
    else { carry_texel<16>(p.carry.p[0], a.out0, x, y); if (TC == 2) carry_texel<16>(p.carry.p[1], a.out1, x, y); }
  }
}

cudaError_t launch_temporal_peer(const TemporalArgs& a, const TemporalPeer& p, cudaStream_t s) {
  if (!a.history_linear || !a.fast || a.in_scaled) return cudaErrorNotSupported;
  dim3 grid((a.W + kTileW - 1) / kTileW, row_tiles(a.row0, a.row1));
#define RFX_LTP(TC, IT) do { if (a.log_transform) temporal_peer_kernel<TC, IT, true><<<grid, kThreads, 0, s>>>(a, p); else temporal_peer_kernel<TC, IT, false><<<grid, kThreads, 0, s>>>(a, p); } while (0)
  if (a.input_type == RFX_INPUT_DIFFUSE_SPECULAR && a.texture_count == 2) RFX_LTP(2, RFX_INPUT_DIFFUSE_SPECULAR);
  else if (a.input_type == RFX_INPUT_DIFFUSE && a.texture_count == 1) RFX_LTP(1, RFX_INPUT_DIFFUSE);
  else if (a.input_type == RFX_INPUT_SPECULAR && a.texture_count == 1) RFX_LTP(1, RFX_INPUT_SPECULAR);
  else return cudaErrorNotSupported;
#undef RFX_LTP
  return cudaGetLastError();
}

template <int TC, int IT, bool FAST>
static void launch_temporal_t(const TemporalArgs& a, dim3 grid, cudaStream_t s) {
  if (a.log_transform) {
    if (a.history_linear) temporal_kernel<TC, IT, true, true, FAST><<<grid, kThreads, 0, s>>>(a);
    else temporal_kernel<TC, IT, true, false, FAST><<<grid, kThreads, 0, s>>>(a);
  } else {
    if (a.history_linear) temporal_kernel<TC, IT, false, true, FAST><<<grid, kThreads, 0, s>>>(a);
    else temporal_kernel<TC, IT, false, false, FAST><<<grid, kThreads, 0, s>>>(a);
  }
}

cudaError_t launch_temporal(const TemporalArgs& a, cudaStream_t s) {
  dim3 grid((a.W + kTileW - 1) / kTileW, row_tiles(a.row0, a.row1));
#define RFX_LT(TC, IT) do { if (a.fast) launch_temporal_t<TC, IT, true>(a, grid, s); else launch_temporal_t<TC, IT, false>(a, grid, s); } while (0)
  if (a.input_type == RFX_INPUT_DIFFUSE_SPECULAR && a.texture_count == 2) RFX_LT(2, RFX_INPUT_DIFFUSE_SPECULAR);
  else if (a.input_type == RFX_INPUT_DIFFUSE && a.texture_count == 1) RFX_LT(1, RFX_INPUT_DIFFUSE);
  else if (a.input_type == RFX_INPUT_SPECULAR && a.texture_count == 1) RFX_LT(1, RFX_INPUT_SPECULAR);
  else return cudaErrorNotSupported;
#undef RFX_LT
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------------------------
// TRAA frame tail of the fast chain: K5 ssgi_compose -> K2 (TRAA form) -> K9 traa_compose in one launch per frame.
// K9 fetches the accumulated plane LINEAR at the pixel centre, which touches texels x +- 1 / y +- 1 wherever
// ((x + .5) / W) * W - .5 is not exactly x, so a block runs K2 on its 16x16 tile plus a ring of one texel (18 x 18).  K2 fetches
// K5 LINEAR at vUv + (dx, dy) / size with |dx|, |dy| <= 2, i.e. texels up to 3 away, so K5 is staged for the tile plus 4 texels on
// each side (24 x 24), rounded to RGBA16F as ssgi_compose_kernel stores it.  K2 and K9 read those fp16 texels from shared memory
// with tex_h4_linear's arithmetic, and K2 / K5 / K9 are the per-pass kernels' own device functions: the bytes are those of the
// three per-pass launches, and the K5 plane never reaches memory.
// ------------------------------------------------------------------------------------------------------------------
constexpr int kTraaTileW = 64;  // a block covers 64 x 16 output pixels: the ring and the K5 halo are recomputed on 16 % / 69 % extra texels
constexpr int kTraaRing = 1, kTraaK5Halo = 3 + kTraaRing;
constexpr int kTraaAccW = kTraaTileW + 2 * kTraaRing, kTraaAccH = kTileH + 2 * kTraaRing;
constexpr int kTraaK5W = kTraaTileW + 2 * kTraaK5Halo, kTraaK5H = kTileH + 2 * kTraaK5Halo;

struct TileH4 {  // RGBA16F texels of a W x H plane held in shared memory: texel (x, y) at s[(y - y0) * w + (x - x0)]
  const uint2* s;
  int x0, y0, w, W, H;
  RFX_D v4 tex(int x, int y) const { return half4_to_v4(s[(y - y0) * w + (x - x0)]); }
  RFX_D v4 linear(v2 uv) const {
    const Bilin b = bilin_setup(uv, W, H);
    return bilin_blend4(b, tex(b.x0, b.y0), tex(b.x1, b.y0), tex(b.x0, b.y1), tex(b.x1, b.y1));
  }
};
RFX_D uint2 pack_h4(v4 v) {  // st_h4's rounding
  uint2 u;
  u.x = packHalf2x16(v.x, v.y);
  u.y = packHalf2x16(v.z, v.w);
  return u;
}
struct TraaStore {  // K2's output: into the shared tile for K9, and into the accumulated plane for the block's own output pixels
  uint2* slot;
  const OutV& acc;
  int x, y;
  bool own;
  RFX_D void operator()(int, v4 v) const {
    const uint2 u = pack_h4(v);
    *slot = u;
    if (own) *((uint2*)(acc.p + ((unsigned)y * (unsigned)acc.pitch + (unsigned)x * 8u))) = u;
  }
};

#ifndef RFX_TRAA_MIN_BLOCKS
#define RFX_TRAA_MIN_BLOCKS 3
#endif
template <bool LOG, bool FAST>
__global__ void __launch_bounds__(kThreads, RFX_TRAA_MIN_BLOCKS) ctraa_kernel(const __grid_constant__ CTraaArgs a) {
  __shared__ uint2 k5s[kTraaK5W * kTraaK5H];
  __shared__ uint2 accs[kTraaAccW * kTraaAccH];
  const TemporalArgs& t = a.t;
  const int W = t.W, H = t.H;
  const int x0 = blockIdx.x * kTraaTileW, y0 = (t.row0 & ~1) + (int)blockIdx.y * kTileH;  // tile rows laid out as range_pixel does
  const int r0 = t.row0, r1 = t.row1;
  for (int i = threadIdx.x; i < kTraaK5W * kTraaK5H; i += kThreads)  // slots outside the image hold a clamped duplicate, never read
    k5s[i] = pack_h4(ssgi_compose_px(a.k5, clampi(x0 - kTraaK5Halo + i % kTraaK5W, W), clampi(y0 - kTraaK5Halo + i / kTraaK5W, H)));
  __syncthreads();
  const TileH4 k5{k5s, x0 - kTraaK5Halo, y0 - kTraaK5Halo, kTraaK5W, W, H};
  for (int i = threadIdx.x; i < kTraaAccW * kTraaAccH; i += kThreads) {
    const int x = x0 - kTraaRing + i % kTraaAccW, y = y0 - kTraaRing + i / kTraaAccW;
    if (x < 0 || x >= W || y < 0 || y >= H) continue;
    const bool own = x >= x0 && x < x0 + kTraaTileW && y >= y0 && y < y0 + kTileH && y >= r0 && y < r1;
    TState s;
    temporal_state(t, x, y, x, y, s);
    s.curvature = 0.0f;  // the TRAA form takes no derivative (fwidth feeds only the discard / hit-point tests of the other forms)
    temporal_px<1, RFX_INPUT_DIFFUSE, LOG, true, FAST>(t, k5, a.hist, a.hist, s, 0.0f, x, y, TraaStore{&accs[i], a.acc, x, y, own});
  }
  __syncthreads();
  const TileH4 acc{accs, x0 - kTraaRing, y0 - kTraaRing, kTraaAccW, W, H};
  for (int i = threadIdx.x; i < kTraaTileW * kTileH; i += kThreads) {
    const int x = x0 + i % kTraaTileW, y = y0 + i / kTraaTileW;
    if (x < W && y < H && y >= r0 && y < r1) st_h4(a.out.p, a.out.pitch, x, y, traa_compose_px(acc, x, y, W, H));
  }
}

cudaError_t launch_ctraa(const CTraaArgs& a, cudaStream_t s) {
  const TemporalArgs& t = a.t;
  if (t.texture_count != 1 || t.input_type != RFX_INPUT_DIFFUSE || !t.input_half || !t.out_half || !t.history_linear || t.hist_f32 || t.in_scaled)
    return cudaErrorNotSupported;
  dim3 grid((t.W + kTraaTileW - 1) / kTraaTileW, row_tiles(t.row0, t.row1));
  if (t.fast) {
    if (t.log_transform) ctraa_kernel<true, true><<<grid, kThreads, 0, s>>>(a);
    else ctraa_kernel<false, true><<<grid, kThreads, 0, s>>>(a);
  } else {
    if (t.log_transform) ctraa_kernel<true, false><<<grid, kThreads, 0, s>>>(a);
    else ctraa_kernel<false, false><<<grid, kThreads, 0, s>>>(a);
  }
  return cudaGetLastError();
}

}  // namespace rfx
