// k_post.cu — K6 HBAO, K6h horizon-march AO, K7 AO compose, K8 motion blur, K9 TRAA compose, env mip downsample (sm_90a).
//
// K6 replaces reference src/ao/AOPass.js:108-109 running src/hbao/shader/hbao.frag:64-96 (+ hbao_utils.glsl,
// whose stale line-1 include is dropped, SURVEY.md D3); K7 src/ao/shader/ao_compose.frag:6-16;
// K8 src/motion-blur/shader/motion_blur.frag:11-44; K9 src/traa/shader/traa_compose.frag:3-6.
// Debug views: GBufferDebugPass (src/gbuffer/debug/GBufferDebugPass.js) and K5's isDebug branch (ssgi_compose.frag:21-24) for
// the views ssgi_compose_kernel does not fetch.
#include "rfx_kernels.h"

namespace rfx {

// K6 and K6h share the world position and the world normal of hbao_utils.glsl (A: HbaoArgs or HbaoHorizonArgs; both carry
// depth, normal, projection_inverse, camera_matrix_world and view_matrix).
template <class A>
RFX_D v3 hbao_world_pos(const A& a, float depth, v2 coord) {  // hbao_utils.glsl:19-29
  const float z = depth * 2.0f - 1.0f;
  const v4 clip = mk4(coord.x * 2.0f - 1.0f, coord.y * 2.0f - 1.0f, z, 1.0f);
  const v4 vs = mul(a.projection_inverse, clip);
  const v4 ws = mul(a.camera_matrix_world, vs);
  return xyz(ws) / ws.w;
}
// getWorldNormal (hbao_utils.glsl:46-79): from the normal plane when `use_normal_plane`, else rebuilt from 9 depth taps
template <class A>
RFX_D v3 hbao_world_normal(const A& a, v2 vUv, bool use_normal_plane) {
  if (use_normal_plane) {  // useNormalTexture  hbao_utils.glsl:70-79: RGBA8 NEAREST, unpackRGBToNormal, (vec4(n, 1.) * viewMatrix).xyz
    const uchar4 t = __ldg((const uchar4*)(a.normal.p + pv_off(a.normal, nearest_i(vUv.x, a.normal.w), nearest_i(vUv.y, a.normal.h), 4)));
    const v3 n = mk3(2.0f * ((float)t.x / 255.0f) - 1.0f, 2.0f * ((float)t.y / 255.0f) - 1.0f, 2.0f * ((float)t.z / 255.0f) - 1.0f);
    return normalize(xyz(mul(mk4(n, 1.0f), a.view_matrix)));
  }
  // computeWorldNormal  hbao_utils.glsl:46-68: in depth texels (textureSize(depthTexture)); texelFetch clamps at the border
  const int DW = a.depth.w, DH = a.depth.h;
  const float sx = (float)DW, sy = (float)DH;
  const int ix = (int)(vUv.x * sx), iy = (int)(vUv.y * sy);
  auto D = [&](int dx, int dy) { return ld_r32f(a.depth, clampi(ix + dx, DW), clampi(iy + dy, DH)); };
  const float c0 = D(0, 0), l2 = D(-2, 0), l1 = D(-1, 0), r1 = D(1, 0), r2 = D(2, 0), b2 = D(0, -2), b1 = D(0, -1), t1 = D(0, 1), t2 = D(0, 2);
  const float dl = fabsf((2.0f * l1 - l2) - c0), dr = fabsf((2.0f * r1 - r2) - c0);
  const float db = fabsf((2.0f * b1 - b2) - c0), dt = fabsf((2.0f * t1 - t2) - c0);
  const v3 ce = hbao_world_pos(a, c0, vUv);
  const v3 dpdx = (dl < dr) ? ce - hbao_world_pos(a, l1, mk2(vUv.x - 1.0f / sx, vUv.y)) : -ce + hbao_world_pos(a, r1, mk2(vUv.x + 1.0f / sx, vUv.y));
  const v3 dpdy = (db < dt) ? ce - hbao_world_pos(a, b1, mk2(vUv.x, vUv.y - 1.0f / sy)) : -ce + hbao_world_pos(a, t1, mk2(vUv.x, vUv.y + 1.0f / sy));
  return normalize(cross(dpdx, dpdy));
}

// GENERAL = false: the target has the depth plane's size, `resolution` is that size and the normal is rebuilt from depth, so the
// pixel itself addresses the depth texel and the blue noise.  GENERAL = true: the target may be smaller than the depth plane
// (AOEffect.setSize scales the AO pass by resolutionScale, src/ao/AOEffect.js:126-146) and `resolution` may be fractional; the
// depth is fetched NEAREST by uv, the blue-noise pixel is ivec2(vUv * resolution) and the normal may come from a normal texture.
// CARRY (row-sharded AO chain): `out` is double-buffered and a discarded pixel copies last frame's texel from its owner (`c`)
template <bool GENERAL, bool CARRY>
__global__ void __launch_bounds__(256) hbao_kernel(const __grid_constant__ HbaoArgs a, const __grid_constant__ PeerPV c) {
  const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = a.row0 + blockIdx.y * 8 + (threadIdx.x >> 5);
  if (x >= a.W || y >= a.row1) return;
  const v2 vUv = pixel_uv(x, y, a.W, a.H);
  const float depth = GENERAL ? tex_r32f_nearest(a.depth, vUv) : ld_r32f(a.depth, x, y);
  if (depth == 1.0f) {  // discard: target keeps its texel
    if (CARRY) carry_texel<8>(c, a.out, x, y);
    return;
  }
  const v4 cp = mul(a.camera_matrix_world, mk4(0.0f, 0.0f, 0.0f, 1.0f));
  const v3 cameraPosition = xyz(cp);
  const v3 worldPos = hbao_world_pos(a, depth, vUv);
  const v3 worldNormal = hbao_world_normal(a, vUv, GENERAL && a.normal.p);
  // getOcclusion: blueNoise() is re-evaluated with the same index for every sample (A9), so the
  // `spp` samples are identical; the loop is kept (it is what the shader executes) but the sample
  // itself is computed once.
  const int bx = GENERAL ? (int)(vUv.x * a.res_x) : x, by = GENERAL ? (int)(vUv.y * a.res_y) : y;  // ivec2(vUv * resolution)
  const uchar4 bn = __ldg(a.blue.tex + ((by + a.blue.shift.sy) % a.blue.size) * a.blue.size + ((bx + a.blue.shift.sx) % a.blue.size));
  const float2 sc = __ldg(a.rot_table + bn.y);
  const float ux = (float)bn.x / 255.0f, bz = (float)bn.z / 255.0f;
  v3 sampleWorldDir;
  {
    const float r = sqrtf(ux);
    const v3 b = normalize(cross(worldNormal, mk3(0.0f, 1.0f, 1.0f)));
    const v3 t = cross(b, worldNormal);
    sampleWorldDir = normalize(r * sc.x * b + sqrtf(1.0f - ux) * worldNormal + r * sc.y * t);
  }
  // pow(blueNoise.z, distancePower + 1.): at the default distancePower = 1, bz * bz is powcr(bz, 2) bit for bit (the square of an fp32
  // value is exact in double, so both round it to fp32 once) without the double pow
  const float dp = a.distance_power + 1.0f;
  const v3 sampleWorldPos = worldPos + a.ao_distance * (dp == 2.0f ? bz * bz : powcr(bz, dp)) * sampleWorldDir;
  const v4 suv4 = mul(a.projection_view, mk4(sampleWorldPos, 1.0f));
  const v2 sq = mk2(suv4.x, suv4.y) / suv4.w;
  const v2 suv = mk2(sq.x * 0.5f + 0.5f, sq.y * 0.5f + 0.5f);
  const float sampleDepth = tex_r32f_nearest(a.depth, suv);
  float deltaDepth = depth - sampleDepth;
  const float d = length(sampleWorldPos - cameraPosition);
  deltaDepth *= 0.001f * d * d;
  const float th = a.thickness * 0.01f;
  const float theta = dot(worldNormal, sampleWorldDir);
  float occ1 = 0.0f;
  if (deltaDepth < th) {
    const float horizon = sampleDepth + deltaDepth * a.bias * 1000.0f;
    float occlusion = fmaxf(0.0f, horizon - depth) * theta;
    const float m = fmaxf(0.0f, 1.0f - deltaDepth / th);
    occlusion = 10.0f * occlusion * m / d;
    occ1 = sqrtf(occlusion);
  }
  float ao = 0.0f, totalWeight = 0.0f;
  for (int i = 0; i < a.spp; i++) { totalWeight += theta; ao += occ1; }
  if (totalWeight > 0.0f) ao /= totalWeight;
  ao = clampf(1.0f - ao, 0.0f, 1.0f);
  st_h4(a.out.p, a.out.pitch, x, y, mk4(worldNormal, ao));
}
cudaError_t launch_hbao(const HbaoArgs& a, cudaStream_t s, const PeerPV* carry) {
  dim3 grid((a.W + 31) / 32, (a.row1 - a.row0 + 7) / 8);
  const PeerPV c = carry ? *carry : PeerPV{};
  if (a.general) { if (carry) hbao_kernel<true, true><<<grid, 256, 0, s>>>(a, c); else hbao_kernel<true, false><<<grid, 256, 0, s>>>(a, c); }
  else { if (carry) hbao_kernel<false, true><<<grid, 256, 0, s>>>(a, c); else hbao_kernel<false, false><<<grid, 256, 0, s>>>(a, c); }
  return cudaGetLastError();
}

// K6h: horizon-march AO (DESIGN.md §1 K6h; Bavoil, Sainz and Dimitrov 2008, per-sample form).  One thread per pixel walks its D x S
// taps in order (direction-major), so the sum has the oracle's order.  Texel snapping, the projected radius and the step size are
// IEEE in both variants; FAST puts the per-tap 1/sqrt(vv) and 1/distance^2 on the SFU.
// CARRY: as hbao_kernel's
template <bool FAST, bool CARRY>
__global__ void __launch_bounds__(256) hbao_horizon_kernel(const __grid_constant__ HbaoHorizonArgs a, const __grid_constant__ PeerPV c) {
  const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = a.row0 + blockIdx.y * 8 + (threadIdx.x >> 5);
  if (x >= a.W || y >= a.row1) return;
  const v2 vUv = pixel_uv(x, y, a.W, a.H);
  const float depth = tex_r32f_nearest(a.depth, vUv);
  if (depth == 1.0f) {  // background: the target keeps its texel
    if (CARRY) carry_texel<8>(c, a.out, x, y);
    return;
  }
  const v3 P = hbao_world_pos(a, depth, vUv);
  const v3 N = hbao_world_normal(a, vUv, a.normal.p != nullptr);
  // projected radius: distance * 0.5 * resolution.y * projection[5] / w_clip of the view position (perspective and orthographic)
  const v4 vs = mul(a.projection_inverse, mk4(vUv.x * 2.0f - 1.0f, vUv.y * 2.0f - 1.0f, depth * 2.0f - 1.0f, 1.0f));
  const v3 Pv = xyz(vs) / vs.w;
  const float w_clip = mul(a.projection, mk4(Pv, 1.0f)).w;
  const float r_px = a.distance * 0.5f * a.res_y * a.projection.m[5] / w_clip;
  float ao = 1.0f;
  if (r_px >= 1.0f) {
    const float delta = fminf(r_px, a.max_radius_pixels) / (float)(a.steps + 1);
    const int bx = (int)(vUv.x * a.res_x), by = (int)(vUv.y * a.res_y);  // ivec2(vUv * resolution), K6's blue-noise texel
    const uchar4 bn = __ldg(a.blue.tex + ((by + a.blue.shift.sy) % a.blue.size) * a.blue.size + ((bx + a.blue.shift.sx) % a.blue.size));
    const float j = (float)bn.y / 255.0f;
    const float2* dirs = a.dirs + bn.x;
    float sum = 0.0f;
    for (int d = 0; d < a.directions; d++) {
      const float2 dir = __ldg(dirs + d * 256);
#pragma unroll 4
      for (int k = 0; k < a.steps; k++) {
        const float t = 1.0f + ((float)k + j) * delta;
        const float ox = floorf(dir.x * t + 0.5f), oy = floorf(dir.y * t + 0.5f);
        const v2 uv = mk2(vUv.x + ox / a.res_x, vUv.y + oy / a.res_y);
        const float sd = tex_r32f_nearest(a.depth, uv);
        const v3 V = hbao_world_pos(a, sd, uv) - P;
        const float vv = dot(V, V);
        if (vv > 0.0f) {
          const float c = (FAST ? dot(N, V) * fx_rsqrt(vv) : dot(N, V) / sqrtf(vv)) - a.angle_bias;
          const float f = 1.0f - (FAST ? vv * a.inv_dist2 : vv / a.dist2);
          sum += clampf(c, 0.0f, 1.0f) * clampf(f, 0.0f, 1.0f);
        }
      }
    }
    ao = clampf(1.0f - a.intensity * sum / (float)(a.directions * a.steps), 0.0f, 1.0f);
  }
  st_h4(a.out.p, a.out.pitch, x, y, mk4(N, ao));
}
cudaError_t launch_hbao_horizon(const HbaoHorizonArgs& a, cudaStream_t s, const PeerPV* carry) {
  dim3 grid((a.W + 31) / 32, (a.row1 - a.row0 + 7) / 8);
  const PeerPV c = carry ? *carry : PeerPV{};
  if (a.fast) { if (carry) hbao_horizon_kernel<true, true><<<grid, 256, 0, s>>>(a, c); else hbao_horizon_kernel<true, false><<<grid, 256, 0, s>>>(a, c); }
  else { if (carry) hbao_horizon_kernel<false, true><<<grid, 256, 0, s>>>(a, c); else hbao_horizon_kernel<false, false><<<grid, 256, 0, s>>>(a, c); }
  return cudaGetLastError();
}

__global__ void __launch_bounds__(256) ao_compose_kernel(const __grid_constant__ AoComposeArgs a) {
  const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = a.row0 + blockIdx.y * 8 + (threadIdx.x >> 5);
  if (x >= a.W || y >= a.row1) return;
  const v2 uv = pixel_uv(x, y, a.W, a.H);
  const float unpackedDepth = ld_r32f(a.depth, x, y);
  float ao = unpackedDepth > 0.9999f ? 1.0f : tex_h4_linear(a.ao, uv).w;
  ao = a.power == 2.0f ? ao * ao : powcr(ao, a.power);  // the default power 2: ao * ao is powcr(ao, 2) bit for bit, as in hbao_kernel
  const v3 aoColor = mix(mk3(a.color[0], a.color[1], a.color[2]), mk3(1.0f), ao);
  const v4 in = tex_h4_linear(a.input, uv);
  st_h4(a.out.p, a.out.pitch, x, y, mk4(aoColor * xyz(in), in.w));
}
cudaError_t launch_ao_compose(const AoComposeArgs& a, cudaStream_t s) {
  dim3 grid((a.W + 31) / 32, (a.row1 - a.row0 + 7) / 8);
  ao_compose_kernel<<<grid, 256, 0, s>>>(a);
  return cudaGetLastError();
}

// K8 for pixel (x, y) given the effect's inputColor: motion_blur.frag's mainImage, velocity NEAREST at the pixel, the samples + 1 taps
// LINEAR through `tap` (the input buffer).  Shared by motion_blur_kernel and traa_motion_blur_kernel.
template <class S>
RFX_D v4 motion_blur_px(const MotionBlurArgs& a, const S& tap, v4 inputColor, v2 vUv, int x, int y) {
  const float4 vt = ld_f4(a.velocity, x, y);
  v2 velocity = mk2(vt.x, vt.y);
  if (!(dot(velocity, velocity) > 0.000000001f)) return inputColor;
  velocity = velocity * a.intensity;
  // blueNoise(vUv, frame) with `resolution` = window size (MotionBlurEffect.js:94): blue_noise.glsl:37-45
  v2 bnv;
  {
    const v2 p = mk2(vUv.x * a.res_x, vUv.y * a.res_y);
    int tx, ty;
    if (a.blue.index == 0) {  // textureLod(blueNoiseTexture, uv * resolution / blueNoiseSize, 0.)  NEAREST + REPEAT
      const float cx = p.x / (float)a.blue.size, cy = p.y / (float)a.blue.size;
      tx = (int)floorf(cx * (float)a.blue.size) % a.blue.size;
      ty = (int)floorf(cy * (float)a.blue.size) % a.blue.size;
      if (tx < 0) tx += a.blue.size;
      if (ty < 0) ty += a.blue.size;
    } else {
      tx = ((int)p.x + a.blue.shift.sx) % a.blue.size;
      ty = ((int)p.y + a.blue.shift.sy) % a.blue.size;
    }
    const uchar4 t = __ldg(a.blue.tex + ty * a.blue.size + tx);
    bnv = mk2((float)t.x / 255.0f, (float)t.y / 255.0f);
  }
  const v2 jitterOffset = a.jitter * velocity * bnv;
  const float frameSpeed = (1.0f / 100.0f) / a.delta_time;
  v2 startUv = vUv + (jitterOffset - velocity * 0.5f) * frameSpeed;
  v2 endUv = vUv + (jitterOffset + velocity * 0.5f) * frameSpeed;
  startUv = mk2(fmaxf(0.0f, startUv.x), fmaxf(0.0f, startUv.y));
  endUv = mk2(fminf(1.0f, endUv.x), fminf(1.0f, endUv.y));
  const float samplesFloat = (float)a.samples;
  v3 c = xyz(inputColor);
  for (float i = 0.0f; i <= samplesFloat; i++) {
    const v2 ruv = mix(startUv, endUv, i / samplesFloat);
    c = c + xyz(tap.linear(ruv));
  }
  c = c / (samplesFloat + 2.0f);
  return mk4(c, inputColor.w);
}
__global__ void __launch_bounds__(256) motion_blur_kernel(const __grid_constant__ MotionBlurArgs a) {
  const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = a.row0 + blockIdx.y * 8 + (threadIdx.x >> 5);
  if (x >= a.W || y >= a.row1) return;
  const v2 vUv = pixel_uv(x, y, a.W, a.H);
  st_h4(a.out.p, a.out.pitch, x, y, motion_blur_px(a, PlaneH4{a.input}, tex_h4_linear(a.input, vUv), vUv, x, y));
}
cudaError_t launch_motion_blur(const MotionBlurArgs& a, cudaStream_t s) {
  dim3 grid((a.W + 31) / 32, (a.row1 - a.row0 + 7) / 8);
  motion_blur_kernel<<<grid, 256, 0, s>>>(a);
  return cudaGetLastError();
}

// TRAAEffect + MotionBlurEffect in one EffectPass: inputColor = K9's colour of the accumulated plane (kept in fp32, as in the merged
// shader), then K8 with its taps on the input buffer.  PEER: the input buffer's rows are read on the ranks that own them.
template <bool PEER>
__global__ void __launch_bounds__(256) traa_motion_blur_kernel(const __grid_constant__ TraaMotionBlurArgs a, const __grid_constant__ PeerPV in) {
  const MotionBlurArgs& m = a.mb;
  const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = m.row0 + blockIdx.y * 8 + (threadIdx.x >> 5);
  if (x >= m.W || y >= m.row1) return;
  const v2 vUv = pixel_uv(x, y, m.W, m.H);
  const v4 inputColor = traa_compose_px(a.acc, x, y, m.W, m.H);
  v4 c;
  if constexpr (PEER) c = motion_blur_px(m, PeerH4{in}, inputColor, vUv, x, y);
  else c = motion_blur_px(m, PlaneH4{m.input}, inputColor, vUv, x, y);
  st_h4(m.out.p, m.out.pitch, x, y, c);
}
cudaError_t launch_traa_motion_blur(const TraaMotionBlurArgs& a, cudaStream_t s, const PeerPV* peer) {
  dim3 grid((a.mb.W + 31) / 32, (a.mb.row1 - a.mb.row0 + 7) / 8);
  if (peer) traa_motion_blur_kernel<true><<<grid, 256, 0, s>>>(a, *peer);
  else traa_motion_blur_kernel<false><<<grid, 256, 0, s>>>(a, PeerPV{});
  return cudaGetLastError();
}

__global__ void __launch_bounds__(256) traa_compose_kernel(const __grid_constant__ TraaComposeArgs a) {
  const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = a.row0 + blockIdx.y * 8 + (threadIdx.x >> 5);
  if (x >= a.W || y >= a.row1) return;
  st_h4(a.out.p, a.out.pitch, x, y, traa_compose_px(a.acc, x, y, a.W, a.H));
}
cudaError_t launch_traa_compose(const TraaComposeArgs& a, cudaStream_t s) {
  dim3 grid((a.W + 31) / 32, (a.row1 - a.row0 + 7) / 8);
  traa_compose_kernel<<<grid, 256, 0, s>>>(a);
  return cudaGetLastError();
}

// box-filter mip level (generateMipmaps of the env map, reference src/ssgi/SSGIEffect.js:324-329)
__global__ void env_downsample_kernel(PV src, OutV dst, int w1, int h1) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= w1 || y >= h1) return;
  const int x0 = min(2 * x, src.w - 1), x1 = min(2 * x + 1, src.w - 1), y0 = min(2 * y, src.h - 1), y1 = min(2 * y + 1, src.h - 1);
  const v4 a = ld_h4(src, x0, y0), b = ld_h4(src, x1, y0), d = ld_h4(src, x0, y1), e = ld_h4(src, x1, y1);
  st_h4(dst.p, dst.pitch, x, y,
        mk4(((a.x + b.x) + (d.x + e.x)) * 0.25f, ((a.y + b.y) + (d.y + e.y)) * 0.25f, ((a.z + b.z) + (d.z + e.z)) * 0.25f,
            ((a.w + b.w) + (d.w + e.w)) * 0.25f));
}
cudaError_t launch_env_downsample(PV src, OutV dst, int w1, int h1, cudaStream_t s) {
  dim3 block(16, 16), grid((w1 + 15) / 16, (h1 + 15) / 16);
  env_downsample_kernel<<<grid, block, 0, s>>>(src, dst, w1, h1);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------------------------------
// Env-map importance-sampling tables on the device (SURVEY.md §8f row 1): restates `gatherData`
// (src/ssgi/utils/EquirectHdrInfoUniform.js:149-245) with the SAME summation order as the JS loops — every accumulator is a JS
// double advanced pixel after pixel — so the tables are bit-identical to the worker's: one thread walks one row (rows are
// independent), one thread walks the global sums (two dependent chains of W*H and H doubles: ~5 ms for 1024x512, once per
// environment change; the reference spends ~100 ms in a Web Worker), then every inverse-CDF entry is an independent binary search.
// flipY: the reference "un-flips" IN PLACE (row y -> row h-1-y for y = 0..h-1), which mirrors the top half over the bottom half
// (SURVEY.md A4): the source row of row r is min(r, h-1-r).
// ------------------------------------------------------------------------------------------------------------------------
RFX_D double env_weight(const PV& map, int x, int row) {  // colorToLuminance on the fp16 texel widened to fp32 (DataUtils.fromHalfFloat)
  const uint2 t = __ldg((const uint2*)(map.p + ((long long)row * map.pitch + (long long)x * 8)));
  const double r = (double)h_lo(t.x), g = (double)h_hi(t.x), b = (double)h_lo(t.y);
  return __dadd_rn(__dadd_rn(__dmul_rn(0.2126, r), __dmul_rn(0.7152, g)), __dmul_rn(0.0722, b));
}
__global__ void env_row_scan_kernel(PV map, int flip_y, float* cdf_c, double* row_sum) {
  const int y = blockIdx.x * blockDim.x + threadIdx.x;
  if (y >= map.h) return;
  const int src = flip_y ? min(y, map.h - 1 - y) : y;
  double cum = 0.0;
  float* out = cdf_c + (size_t)y * map.w;
  for (int x = 0; x < map.w; x++) {
    cum = __dadd_rn(cum, env_weight(map, x, src));
    out[x] = (float)cum;                                   // cdfConditional[i] = cumulativeRowWeight (Float32Array store)
  }
  row_sum[y] = cum;
  if (cum != 0.0)
    for (int x = 0; x < map.w; x++) out[x] = (float)((double)out[x] / cum);   // cdfConditional[i] /= cumulativeRowWeight
}
__global__ void env_totals_kernel(PV map, int flip_y, const double* row_sum, float* cdf_m, double* total_out) {
  if (blockIdx.x || threadIdx.x) return;
  double total = 0.0;
  for (int y = 0; y < map.h; y++) {                         // totalSumValue += weight, pixel after pixel in row-major order
    const int src = flip_y ? min(y, map.h - 1 - y) : y;
    for (int x = 0; x < map.w; x++) total = __dadd_rn(total, env_weight(map, x, src));
  }
  *total_out = total;
  double cum = 0.0;
  for (int y = 0; y < map.h; y++) { cum = __dadd_rn(cum, row_sum[y]); cdf_m[y] = (float)cum; }
  if (cum != 0.0)
    for (int y = 0; y < map.h; y++) cdf_m[y] = (float)((double)cdf_m[y] / cum);
}
RFX_D int env_closest(const float* a, double target, int count) {  // binarySearchFindClosestIndexOf :130-147
  int lower = 0, upper = count - 1;
  while (lower < upper) {
    const int mid = (lower + upper) >> 1;
    if ((double)a[mid] < target) lower = mid + 1; else upper = mid;
  }
  return lower;
}
__global__ void env_inverse_cdf_kernel(const float* cdf_m, const float* cdf_c, int W, int H, float* marginal, float* conditional) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < H) marginal[i] = (float)(((double)env_closest(cdf_m, (double)(i + 1) / (double)H, H) + 0.5) / (double)H);
  if (i < W * H) {
    const int y = i / W, x = i - y * W;
    conditional[i] = (float)(((double)env_closest(cdf_c + (size_t)y * W, (double)(x + 1) / (double)W, W) + 0.5) / (double)W);
  }
}
cudaError_t launch_env_cdf(PV map, int flip_y, float* cdf_c, float* cdf_m, double* row_sum, double* total, float* marginal, float* conditional, cudaStream_t s) {
  env_row_scan_kernel<<<(map.h + 63) / 64, 64, 0, s>>>(map, flip_y, cdf_c, row_sum);
  env_totals_kernel<<<1, 1, 0, s>>>(map, flip_y, row_sum, cdf_m, total);
  env_inverse_cdf_kernel<<<(map.w * map.h + 255) / 256, 256, 0, s>>>(cdf_m, cdf_c, map.w, map.h, marginal, conditional);
  return cudaGetLastError();
}

// GBufferDebugPass: getMaterial (gbuffer_packing.glsl:181-196) at the pixel's own texel (target and G-buffer have one size, NEAREST).
// `depth` is gBuffer.r: the shader's depthTexture is not among the material's uniforms, so its sampler stays on unit 0, gBufferTexture's.
__global__ void __launch_bounds__(256) gbuffer_debug_kernel(const __grid_constant__ GbufferDebugArgs a) {
  const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = a.row0 + blockIdx.y * 8 + (threadIdx.x >> 5);
  if (x >= a.W || y >= a.row1) return;
  const float4 g = ld_f4(a.gb, x, y);
  float4 o = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
  if (g.x != 0.0f) {
    v3 c;
    switch (a.mode) {
      case 0: c = xyz(floatToVec4(g.x)); break;
      case 1: c = mk3(floatToVec4(g.x).w); break;
      case 2: c = unpackNormal(g.y); break;
      case 3: c = mk3(gb_roughness(g.z)); break;
      case 4: c = mk3(gb_metalness(g.z)); break;
      default: c = decodeRGBE8<true>(floatToVec4(g.w)); break;
    }
    o = make_float4(c.x, c.y, c.z, 1.0f);
  }
  st_f4(a.out.p, a.out.pitch, x, y, o);
}
cudaError_t launch_gbuffer_debug(const GbufferDebugArgs& a, cudaStream_t s) {
  dim3 grid((a.W + 31) / 32, (a.row1 - a.row0 + 7) / 8);
  gbuffer_debug_kernel<<<grid, 256, 0, s>>>(a);
  return cudaGetLastError();
}

// K5 with isDebug: textureLod(inputTexture, vUv, 0.) rounded to the RGBA16F composer buffer.  A depth texture reads (d, 0, 0, 1)
// (GLES 3.0 depth-texture swizzle).  NEAREST and LINEAR are those of every other pass (nearest_i, bilin_setup), so a source of
// another size is resampled exactly as the reference's sampler would.
__global__ void __launch_bounds__(256) ssgi_compose_debug_kernel(const __grid_constant__ SsgiComposeDebugArgs a) {
  const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = a.row0 + blockIdx.y * 8 + (threadIdx.x >> 5);
  if (x >= a.W || y >= a.row1) return;
  const v2 uv = pixel_uv(x, y, a.W, a.H);
  v4 c;
  if (a.gi_fmt == RFX_FMT_R32F) c = mk4(tex_r32f_nearest(a.gi, uv), 0.0f, 0.0f, 1.0f);
  else if (a.gi_fmt == RFX_FMT_RGBA16F) c = tex_h4_linear(a.gi, uv);
  else c = f4v(tex_f4_nearest(a.gi, uv));
  st_h4(a.out.p, a.out.pitch, x, y, c);
}
cudaError_t launch_ssgi_compose_debug(const SsgiComposeDebugArgs& a, cudaStream_t s) {
  dim3 grid((a.W + 31) / 32, (a.row1 - a.row0 + 7) / 8);
  ssgi_compose_debug_kernel<<<grid, 256, 0, s>>>(a);
  return cudaGetLastError();
}

}  // namespace rfx
