// k_fx.cu — the plugin surface's cosmetic effects (SURVEY.md §8f row 3) as ONE tail kernel, plus TAAPass.
//
// The reference runs SharpnessEffect / LensDistortionEffect / GradualBackgroundEffect / SparkleEffect as postprocessing `Effect`s:
// an EffectPass merges the effects of a pass into one fullscreen shader in which every effect samples the same input buffer and
// the colour is handed from one mainImage() to the next.  effects_kernel is that merged shader, selected at run time: up to four
// effects in caller order, one read of the frame, one write — instead of one full-frame round trip per effect.  HBM traffic is
// 8 B/px in + 8 B/px out (+ 4 depth / + 16 velocity when used); the 3x3 and bilinear taps of the input are L1 / L2 hits.
// Arithmetic is IEEE fp32, and every transcendental of the effects is evaluated in double and rounded once (rfx_device.cuh's sincr /
// expcr / powcr, what "correctly rounded" means for the parity oracle), so effects_kernel is bit-equal to the oracle.  A libm fp32 call
// 1-2 ulp off would not stay small here: the hash of SparkleEffect (fract(sin(x) * 43758.5)) and pow(noise, 500 * spread) turn a one-ulp
// difference of sin() into a different sparkle pattern.  TAAPass takes its sRGB curve on the SFU and re-evaluates it in double only for
// the ~0.4 % of texels whose 8-bit rounding is within 2e-3 of a tie.
#include "rfx_device.cuh"
#include "rfx_kernels.h"

namespace rfx {

namespace {

RFX_D v4 add4(v4 a, v4 b) { return mk4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); }
// powcr(x, 4.) without the double pow: x * x is exact in double, so d * d is x^4 rounded once to double, as pow returns it
RFX_D float pow4cr(float x) { const double d = (double)x * (double)x; return (float)(d * d); }

// SharpnessEffect.js:8-29
RFX_D v4 fx_sharpness(const PV& in, v4 inputColor, v2 uv, v2 ts, float sharp) {
  v4 blurred = tex_h4_linear(in, uv - 1.0f * ts);
  blurred = add4(blurred, tex_h4_linear(in, uv + mk2(0.0f, -1.0f) * ts));
  blurred = add4(blurred, tex_h4_linear(in, uv + mk2(1.0f, -1.0f) * ts));
  blurred = add4(blurred, tex_h4_linear(in, uv + mk2(-1.0f, 0.0f) * ts));
  blurred = add4(blurred, inputColor);
  blurred = add4(blurred, tex_h4_linear(in, uv + mk2(1.0f, 0.0f) * ts));
  blurred = add4(blurred, tex_h4_linear(in, uv + mk2(-1.0f, 1.0f) * ts));
  blurred = add4(blurred, tex_h4_linear(in, uv + mk2(0.0f, 1.0f) * ts));
  blurred = add4(blurred, tex_h4_linear(in, uv + 1.0f * ts));
  blurred = blurred / 9.0f;
  const v4 s = mk4(inputColor.x + (inputColor.x - blurred.x) * sharp, inputColor.y + (inputColor.y - blurred.y) * sharp,
                   inputColor.z + (inputColor.z - blurred.z) * sharp, inputColor.w + (inputColor.w - blurred.w) * sharp);
  return mk4(fmaxf(s.x, 0.0f), fmaxf(s.y, 0.0f), fmaxf(s.z, 0.0f), s.w);
}
// LensDistortionEffect.js:14-45
RFX_D v4 fx_lens(const PV& in, v2 vUv, float W, float H, float alphax, float alphay, float aberration) {
  const float x = __fdiv_rn(2.0f * vUv.x - 1.0f, 1.0f), y = __fdiv_rn(2.0f * vUv.y - 1.0f, 1.0f);
  const float r = x * x + y * y;
  const float x3 = __fdiv_rn(x, 1.0f - alphax * r), y3 = __fdiv_rn(y, 1.0f - alphay * r);
  const float q = x3 * x3 + y3 * y3;
  const float x2 = __fdiv_rn(x, 1.0f - alphax * q), y2 = __fdiv_rn(y, 1.0f - alphay * q);
  const v2 duv = mk2(__fdiv_rn((x2 + 1.0f) * 1.0f, 2.0f), __fdiv_rn((y2 + 1.0f) * 1.0f, 2.0f));
  const float ox = __fdiv_rn(1.0f, W), oy = __fdiv_rn(1.0f, H);
  const v4 rv = tex_h4_linear(in, duv - aberration * mk2(ox, 0.0f));
  const v4 gv = tex_h4_linear(in, duv - aberration * mk2(0.0f, oy));
  const v4 bv = tex_h4_linear(in, duv - aberration * mk2(ox, oy));
  return mk4(rv.x, gv.y, bv.z, 1.0f);
}
// getViewPosition  GradualBackgroundEffect.js:22-29 / SparkleEffect.js:29-36
RFX_D v3 view_position(const CamD& cam, v2 vUv, float viewZ) {
  const float clipW = cam.projection.m[2 * 4 + 3] * viewZ + cam.projection.m[3 * 4 + 3];
  v4 clip = mk4((vUv.x - 0.5f) * 2.0f, (vUv.y - 0.5f) * 2.0f, (viewZ - 0.5f) * 2.0f, 1.0f);
  clip = mk4(clip.x * clipW, clip.y * clipW, clip.z * clipW, clip.w * clipW);
  v3 p = xyz(mul(cam.projection_inverse, clip));
  p.z = viewZ;
  return p;
}
RFX_D float view_z(const CamD& cam, bool perspective, float depth) {
  return perspective ? perspectiveDepthToViewZ(depth, cam.near_plane, cam.far_plane) : orthographicDepthToViewZ(depth, cam.near_plane, cam.far_plane);
}
// GradualBackgroundEffect.js:31-46
RFX_D v4 fx_gradual_background(const EffectsArgs& a, v4 inputColor, int x, int y, v2 uv) {
  const float depth = ld_r32f(a.depth, x, y);  // textureLod(depthTexture, uv, 0.) at the pixel centre of a NEAREST texture
  const v3 viewPos = view_position(a.cam, uv, view_z(a.cam, a.cam.perspective != 0, depth));
  const v3 worldPos = xyz(mul(a.cam.camera_matrix_world, mk4(viewPos, 1.0f)));
  const float distToCenter = length(mk2(worldPos.x, worldPos.z)) + fmaxf(0.0f, -worldPos.y);
  // pow(distToCenter, 0.1) is taken in double (powcr) only where the clamp may not saturate: elsewhere the fp32 powf (a few ulps, far
  // inside the 1e-5 margin) already puts the fade at 0 or 1, and so would the exact value
  const float p15 = powf(distToCenter, 0.1f) * 15.0f, margin = 1e-5f * (p15 + fabsf(a.max_distance));
  float g = p15 - a.max_distance;
  if (g > -margin && g < 1.0f + margin) g = powcr(distToCenter, 0.1f) * 15.0f - a.max_distance;
  const float fade = clampf(g, 0.0f, 1.0f);
  const v3 c = mix(xyz(inputColor), mk3(a.bg[0], a.bg[1], a.bg[2]), fade);
  return mk4(c, 1.0f);
}
// three <common> rand()
RFX_D float rand2(v2 uv) {
  const float dt = dot(uv, mk2(12.9898f, 78.233f)), sn = mod_gl(dt, 3.141592653589793f);
  const float v = sincr(sn) * 43758.5453f;
  return v - floorf(v);
}
// SparkleEffect.js:38-43
RFX_D float nn(v2 n) {
  const v2 b = mk2(floorf(n.x), floorf(n.y));
  const v2 f = mk2(smoothstepf(0.0f, 1.0f, n.x - floorf(n.x)), smoothstepf(0.0f, 1.0f, n.y - floorf(n.y)));
  return mixf(mixf(rand2(b), rand2(b + mk2(1.0f, 0.0f)), f.x), mixf(rand2(b + mk2(0.0f, 1.0f)), rand2(b + mk2(1.0f, 1.0f)), f.x), f.y);
}
// SparkleEffect.js:45-99
RFX_D v4 fx_sparkle(const EffectsArgs& a, v4 inputColor, int x, int y, v2 uv) {
  const float4 vt = ld_f4(a.velocity, x, y);
  const float depth = vt.w;
  if (depth == 0.0f || depth == 1.0f) return inputColor;
  const v3 normal = unpackNormal(vt.z);
  const v3 viewNormal = normalize(xyz(mul(a.cam.view_matrix, mk4(normal, 0.0f))));
  const v3 viewPos = view_position(a.cam, uv, view_z(a.cam, a.sparkle_perspective != 0, depth));
  const v3 viewDir = normalize(viewPos);
  const v3 worldPos = xyz(mul(a.cam.camera_matrix_world, mk4(viewPos, 1.0f)));
  if (worldPos.y < 0.01f) return inputColor;
  const v3 cameraPos = xyz(mul(a.cam.camera_matrix_world, mk4(0.0f, 0.0f, 0.0f, 1.0f)));
  const float dist = length(worldPos - cameraPos);
  const float distFactor = expcr(-dist * 0.005f);
  float facing = fmaxf(dot(-viewDir, viewNormal), 0.0f);
  facing = pow4cr(facing);
  const v3 nw = normalize(worldPos);
  const v2 offset = mk2(nw.x, nw.z) * 1000.0f + mk2(normal.x, normal.z) * 500.0f;
  float noise = nn(offset);
  noise = powcr(noise, 500.0f * a.spread);
  float lum = dot(xyz(inputColor), mk3(0.299f, 0.587f, 0.114f));
  lum = smoothstepf(0.15f, 1.0f, lum);
  const float sparkleFactor = noise * lum * facing * distFactor * 5000.0f * a.intensity;
  const v3 c = xyz(inputColor);
  const v3 color = c + mk3(pow4cr(c.x), pow4cr(c.y), pow4cr(c.z)) * sparkleFactor;
  return mk4(color, 1.0f);
}

__global__ void __launch_bounds__(256) effects_kernel(const __grid_constant__ EffectsArgs a) {
  const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = a.row0 + blockIdx.y * 8 + (threadIdx.x >> 5);
  if (x >= a.W || y >= a.row1) return;
  const v2 uv = pixel_uv(x, y, a.W, a.H);
  v4 c = tex_h4_linear(a.input, uv);  // EffectPass: texture2D(inputBuffer, vUv)
  for (int e = 0; e < a.n_effects; e++) {
    switch (a.effects[e]) {
      case RFX_FX_SHARPNESS: c = fx_sharpness(a.input, c, uv, mk2(a.texel_x, a.texel_y), a.sharpness); break;
      case RFX_FX_LENS_DISTORTION: c = fx_lens(a.input, uv, (float)a.W, (float)a.H, a.alphax, a.alphay, a.aberration); break;
      case RFX_FX_GRADUAL_BACKGROUND: c = fx_gradual_background(a, c, x, y, uv); break;
      case RFX_FX_SPARKLE: c = fx_sparkle(a, c, x, y, uv); break;
      default: break;
    }
  }
  st_h4(a.out.p, a.out.pitch, x, y, c);
}

// three r151 LinearTosRGB (encodings_pars_fragment)
// EXACT = false: v^0.41666 on the SFU (ex2(0.41666 * lg2(v)), relative error ~1e-6, i.e. < 3e-4 of an 8-bit step — two orders inside the
// tie window that triggers the exact re-evaluation below).  As pow, it is NaN for a negative v (lg2 of a negative number is NaN) and 0
// for +-0 (lg2 gives -inf, ex2 of it 0); mix() carries the NaN even where v <= 0.0031308 selects the linear segment, so a negative
// channel ends at 0 after the clamp whatever the history holds.
template <bool EXACT>
RFX_D float linear_to_srgb(float v) {
  const float pw = EXACT ? powcr(v, 0.41666f) : fx_ex2(0.41666f * fx_lg2(v));
  const float hi = pw * 1.055f - 0.055f, lo = v * 12.92f;
  return mixf(hi, lo, v <= 0.0031308f ? 1.0f : 0.0f);
}
template <bool EXACT>
RFX_D v4 taa_value(const TaaArgs& a, v4 color, v4 acc, float t) {
  if (a.srgb_output) color = mk4(linear_to_srgb<EXACT>(color.x), linear_to_srgb<EXACT>(color.y), linear_to_srgb<EXACT>(color.z), color.w);
  if (a.camera_not_moved_frames == 0.0f) return color;
  return mk4(mixf(acc.x, color.x, t), mixf(acc.y, color.y, t), mixf(acc.z, color.z, t), mixf(acc.w, color.w, t));
}
RFX_D bool near_tie(float v) { const float s = clampf(v, 0.0f, 1.0f) * 255.0f; return fabsf((s - floorf(s)) - 0.5f) < 2e-3f; }
RFX_D unsigned to_unorm8(float v) { return (unsigned)lroundf(clampf(v, 0.0f, 1.0f) * 255.0f); }  // round to nearest, ties away from zero

// taa.frag:6-18 rendered to the canvas (RGBA8)
__global__ void __launch_bounds__(256) taa_kernel(const __grid_constant__ TaaArgs a) {
  const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = a.row0 + blockIdx.y * 8 + (threadIdx.x >> 5);
  if (x >= a.W || y >= a.row1) return;
  const v4 color = tex_h4_linear(a.input, pixel_uv(x, y, a.W, a.H));
  v4 acc = mk4(0.0f, 0.0f, 0.0f, 0.0f);
  float t = 1.0f;
  if (!(a.camera_not_moved_frames == 0.0f)) {
    const uchar4 h = __ldg((const uchar4*)(a.history.p + pv_off(a.history, x, y, 4)));
    acc = mk4(__fdiv_rn((float)h.x, 255.0f), __fdiv_rn((float)h.y, 255.0f), __fdiv_rn((float)h.z, 255.0f), __fdiv_rn((float)h.w, 255.0f));
    t = __fdiv_rn(1.0f, a.camera_not_moved_frames + 1.0f);
  }
  v4 o = taa_value<false>(a, color, acc, t);
  if (a.srgb_output && (near_tie(o.x) || near_tie(o.y) || near_tie(o.z))) o = taa_value<true>(a, color, acc, t);  // the libm pow may sit on the other side of the tie
  uchar4 q;
  q.x = (unsigned char)to_unorm8(o.x); q.y = (unsigned char)to_unorm8(o.y); q.z = (unsigned char)to_unorm8(o.z); q.w = (unsigned char)to_unorm8(o.w);
  *((uchar4*)(a.out.p + ((unsigned)y * (unsigned)a.out.pitch + (unsigned)x * 4u))) = q;
}

}  // namespace

cudaError_t launch_effects(const EffectsArgs& a, cudaStream_t s) {
  dim3 grid((a.W + 31) / 32, (a.row1 - a.row0 + 7) / 8);
  effects_kernel<<<grid, 256, 0, s>>>(a);
  return cudaGetLastError();
}
cudaError_t launch_taa(const TaaArgs& a, cudaStream_t s) {
  dim3 grid((a.W + 31) / 32, (a.row1 - a.row0 + 7) / 8);
  taa_kernel<<<grid, 256, 0, s>>>(a);
  return cudaGetLastError();
}

}  // namespace rfx
