// rfx_kernels.h — internal launch interface between the C-ABI layer (rfx_api.cu) and the
// sm_90a kernels (k_*.cu).  Everything here is plain structs of device pointers + uniforms.
#pragma once
#include <cuda.h>  // CUtensorMap (type only; the encode entry point is resolved at run time)

#include "rfx_device.cuh"
#include "../../include/rfx.h"

namespace rfx {

struct OutV {  // writable plane view
  unsigned char* p;
  long long pitch;
};

#define RFX_MAX_PEERS 8
struct PeerPV {
  PV local;                                    // this rank's allocation (full-frame sized); rows [own0, own1) are valid here
  const unsigned char* base[RFX_MAX_PEERS];    // every rank's allocation of the same plane (peer-mapped), same pitch
  int bound[RFX_MAX_PEERS + 1];                // rank k owns rows [bound[k], bound[k+1]) of the data being read
  int n;                                       // ranks; <= 1: single GPU (local only)
  int own0, own1;
};
RFX_D const unsigned char* peer_row_base(const PeerPV& p, int y) {
  if (p.n <= 1 || (y >= p.own0 && y < p.own1)) return p.local.p;
  int k = 0;
#pragma unroll
  for (int i = 1; i < RFX_MAX_PEERS; i++) k += (i < p.n && y >= p.bound[i]) ? 1 : 0;
  return p.base[k];
}
// LINEAR fetch of an RGBA16F plane whose rows live on their owners: tex_h4_linear's arithmetic, each row from peer_row_base
RFX_D v4 peer_h4_linear(const PeerPV& p, v2 uv) {
  const Bilin b = bilin_setup(uv, p.local.w, p.local.h);
  const unsigned char* r0 = peer_row_base(p, b.y0) + (unsigned)b.y0 * (unsigned)p.local.pitch;
  const unsigned char* r1 = peer_row_base(p, b.y1) + (unsigned)b.y1 * (unsigned)p.local.pitch;
  auto ld = [](const unsigned char* r, int x) { return half4_to_v4(__ldg((const uint2*)(r + (unsigned)x * 8u))); };
  return bilin_blend4(b, ld(r0, b.x0), ld(r0, b.x1), ld(r1, b.x0), ld(r1, b.x1));
}

// LINEAR fetch of an RGBA32F plane whose rows live on their owners: tex_f4_linear's arithmetic, each row from peer_row_base
RFX_D v4 peer_f4_linear(const PeerPV& p, v2 uv) {
  const Bilin b = bilin_setup(uv, p.local.w, p.local.h);
  const unsigned char* r0 = peer_row_base(p, b.y0) + (unsigned)b.y0 * (unsigned)p.local.pitch;
  const unsigned char* r1 = peer_row_base(p, b.y1) + (unsigned)b.y1 * (unsigned)p.local.pitch;
  auto ld = [](const unsigned char* r, int x) { return f4v(__ldg((const float4*)(r + (unsigned)x * 16u))); };
  return bilin_blend4(b, ld(r0, b.x0), ld(r0, b.x1), ld(r1, b.x0), ld(r1, b.x1));
}
// Carry on discard (per-pass chain in a row-sharded group): a target is double-buffered by frame parity, and a pixel the shader
// `discard`s (the reference's "target keeps its texel") copies last frame's texel of each target plane from the rank that owns the row.
struct PeerCarry {
  PeerPV p[2];  // last frame's planes of target 0 / 1 (p[1] unused with one plane)
};
template <int BYTES>
RFX_D void carry_texel(const PeerPV& src, const OutV& dst, int x, int y) {
  const size_t off = (size_t)y * (size_t)dst.pitch + (size_t)x * BYTES;  // src and dst: the same format and width, hence the same pitch
  const unsigned char* s = peer_row_base(src, y) + off;
  if (BYTES == 16) *(uint4*)(dst.p + off) = __ldg((const uint4*)s);
  else *(uint2*)(dst.p + off) = __ldg((const uint2*)s);
}

struct CamD {  // device copy of rfx_camera
  M4 projection, projection_inverse, camera_matrix_world, view_matrix;
  float near_plane, far_plane;
  int perspective;
};

struct BlueD {
  const uchar4* tex;  // size x size RGBA8, GL texel order
  int size;
  BlueShift shift;    // (pcg4d(seed(index)).xy % 0x0fffffff) % size, computed on the host
  int index;          // raw index (0 selects the tiled lookup of blue_noise.glsl:38-39)
  int mask;           // size - 1 when size is a power of two (the shipped 128 x 128 texture), else 0
};
RFX_D int blue_index(const BlueD& b, int x, int y) {
  if (b.mask) return ((y + b.shift.sy) & b.mask) * b.size + ((x + b.shift.sx) & b.mask);
  return ((y + b.shift.sy) % b.size) * b.size + ((x + b.shift.sx) % b.size);
}

struct EnvD {
  PV mip[16];  // RGBA16F levels
  int levels;
  PV marginal, conditional;  // R32F
  float size_x, size_y, total_sum_whole, total_sum_decimal;
};

// ---- K3 ----------------------------------------------------------------------------------
struct PoissonArgs {
  PV depth, gb, in0, in1;
  OutV out0, out1;
  int W, H, row0, row1;
  float radius, phi, luma_phi, depth_phi, normal_phi, roughness_phi, specular_phi;
  int texture_count, spec0, spec1, gbuffer_texture, input_linear, in_half;
  BlueD blue;
  const float2* rot_table;  // [256] (sin, cos) of (k/255)*2*pi, correctly rounded
  // fast variant only:
  PV nrd;                       // float4 (normal.xyz, roughness) from the decode prepass
  float tap_ox[8], tap_oy[8];   // POISSON[i] / resolution
};
// carry != nullptr: the carry-on-discard instantiation (out0 / out1 double-buffered in a row-sharded group, see PeerCarry)
cudaError_t launch_poisson(const PoissonArgs& a, cudaStream_t s, const PeerCarry* carry = nullptr);       // exact-libm variant (any configuration)
cudaError_t launch_poisson_fast(const PoissonArgs& a, cudaStream_t s, const PeerCarry* carry = nullptr);  // SFU variant (GBUFFER_TEXTURE configurations)
cudaError_t launch_gbuffer_decode(PV gb, OutV nrd, int W, int H, int gbuffer_texture, int row0, int row1, int halo, cudaStream_t s);

// ---- K4 / K5 -------------------------------------------------------------------------------
struct ComposeArgs {
  PV depth, gb, diffuse, specular, scene;  // diffuse / specular / scene: p == nullptr = not bound (null sampler)
  OutV out;
  int W, H, row0, row1;
  CamD cam;
  int input_type;
  int gi_f32;  // diffuse / specular are RGBA32F NEAREST (denoiseMode "full_temporal": the temporal pass's targets)
  int fast;
};
cudaError_t launch_gi_compose(const ComposeArgs& a, cudaStream_t s, const PeerPV* carry = nullptr);  // carry: as launch_poisson's, `out`

struct SsgiComposeArgs {
  PV depth, gi, scene;
  OutV out;
  int W, H, row0, row1;
  int use_fog, fog_exp2, perspective, is_debug;
  float fog_color[3], fog_near, fog_far, fog_density, camera_near, camera_far;
};
cudaError_t launch_ssgi_compose(const SsgiComposeArgs& a, cudaStream_t s);
// K5 without isDebug for pixel (x, y) of depth `depth`; gi() returns the pixel's GI texel and is called for a foreground pixel only.
// Shared with the compose stage fused into the fast chain's K4 (k_chain.cu), which passes the texel it just composed.
template <class GI>
RFX_D v4 ssgi_compose_lit(const SsgiComposeArgs& a, int x, int y, float depth, const GI& gi) {
  v3 c;
  if (depth == 1.0f) {
    c = xyz(tex_h4_linear(a.scene, pixel_uv(x, y, a.W, a.H)));
  } else {
    c = xyz(f4v(gi()));
    if (a.use_fog) {  // :34-41 + three.js <fog_fragment>
      const float gz = a.perspective ? perspectiveDepthToViewZ(depth, a.camera_near, a.camera_far) : orthographicDepthToViewZ(depth, a.camera_near, a.camera_far);
      const float vFogDepth = -(gz * 0.4f);
      const float fogFactor = a.fog_exp2 ? 1.0f - expcr(-a.fog_density * a.fog_density * vFogDepth * vFogDepth) : smoothstepf(a.fog_near, a.fog_far, vFogDepth);
      c = mix(c, mk3(a.fog_color[0], a.fog_color[1], a.fog_color[2]), fogFactor);
    }
  }
  return mk4(c, 1.0f);
}
// K5 for pixel (x, y): the texel ssgi_compose_kernel stores (RGBA16F)
RFX_D v4 ssgi_compose_px(const SsgiComposeArgs& a, int x, int y) {
  if (a.is_debug) {  // ssgi_compose.frag:21-24
    const float4 t = ld_f4(a.gi, x, y);
    return mk4(t.x, t.y, t.z, t.w);
  }
  return ssgi_compose_lit(a, x, y, ld_r32f(a.depth, x, y), [&] { return ld_f4(a.gi, x, y); });
}
// K5 with isDebug for the views ssgi_compose_kernel does not fetch (its debug branch reads an RGBA32F plane of the output's size):
// `gi` of any size and format, sampled at the pixel centre with its own sampler.
struct SsgiComposeDebugArgs {
  PV gi;
  int gi_fmt;  // RFX_FMT_R32F (a depth texture: (d, 0, 0, 1)), RFX_FMT_RGBA16F (LINEAR), RFX_FMT_RGBA32F (NEAREST)
  OutV out;
  int W, H, row0, row1;
};
cudaError_t launch_ssgi_compose_debug(const SsgiComposeDebugArgs& a, cudaStream_t s);

// GBufferDebugPass (k_post.cu)
struct GbufferDebugArgs {
  PV gb;
  OutV out;
  int W, H, row0, row1;
  int mode;
};
cudaError_t launch_gbuffer_debug(const GbufferDebugArgs& a, cudaStream_t s);

// ---- K2 ----------------------------------------------------------------------------------
struct TemporalArgs {
  PV input, velocity, hist0, hist1;
  OutV out0, out1;
  int W, H, row0, row1;
  CamD cam;
  M4 prev_view, prev_world, prev_proj, prev_proj_inv;
  M4 prev_proj_view;  // prevProjectionMatrix * prevViewMatrix (reproject.frag:183), fma-lowered on the host
  float camera_pos[3];
  float max_blend, clamp_intensity, keep_data, confidence_power;
  float inv_w, inv_h;  // invTexSize
  int full_accumulate, texture_count, input_type, log_transform, rs0, rs1, history_linear;
  int input_half, out_half;
  int in_scaled;  // inputTexture (the SSGI target) is smaller than the output (resolutionScale < 1): NEAREST fetch by uv
  int hist_f32;  // history planes are RGBA32F (denoiseMode "full_temporal" / "temporal")
  int fast;  // SFU variants of log/exp/pow
};
cudaError_t launch_temporal(const TemporalArgs& a, cudaStream_t s);
// K2 of the per-pass chain in a row-sharded group: the history planes are read on the rank that owns each row (RGBA16F through
// peer_h4_linear, RGBA32F through peer_f4_linear), and a discarded pixel carries last frame's texel of out0 / out1 (double-buffered)
// from the owner.  a.hist0 / a.hist1 are ignored; history_linear must be on, and fast too except for the TRAA form (texture_count 1,
// input_type DIFFUSE), which also has an exact instantiation.
struct TemporalPeer {
  PeerPV hist0, hist1;
  PeerCarry carry;
};
cudaError_t launch_temporal_peer(const TemporalArgs& a, const TemporalPeer& p, cudaStream_t s);

// ---- K1 ----------------------------------------------------------------------------------
struct SsgiArgs {
  PV depth, gb, velocity, direct, accumulated;  // velocity/direct/accumulated may have p == nullptr
  OutV out;
  int W, H, row0, row1;
  CamD cam;
  float ray_distance, thickness, env_blur, max_env_mip;
  float near_minus_far, near_mul_far, far_minus_near;
  int steps, refine_steps, mode;
  unsigned flags;
  BlueD blue;
  EnvD env;
  const float2* rot_table;   // [256] (sin, cos)
  const float* step_table;   // [steps][256]  cs(i, b) = 1 - exp(-0.25 (i + b - 0.5)^2), row i-1 for step i
  PV viewz;                  // R32F: getViewZ(depth) per texel (launch_viewz prepass)
  int proj_sparse;           // projection matrix has the perspective sparsity pattern (exact-zero terms dropped)
  int fast;                  // SFU variants of the continuous transcendentals
  // fast fused kernel (ssgi_fast_kernel)
  float ps_x0, ps_x2, ps_y1, ps_y2, ps_hw, ps_hh;  // projection rows scaled to texel units: tx = (ps_x0*x + ps_x2*z) / -z + ps_hw
  int vz_pitchw;             // viewZ pitch in 4-byte words
  int scaled;                // the render target (W x H) is smaller than the input planes (resolutionScale < 1): texels are fetched by uv
  PeerPV acc_peer;           // `accumulated` in a row-sharded group (n > 1): rows live on their owners
};
cudaError_t launch_ssgi(const SsgiArgs& a, cudaStream_t s);
cudaError_t launch_viewz(const SsgiArgs& a, OutV vz, cudaStream_t s);

// ---- K6 / K7 / K8 / K9 -----------------------------------------------------------------------
struct HbaoArgs {
  PV depth;
  PV normal;  // RGBA8 view-space normal (NormalPass layout) or p == nullptr: rebuilt from depth
  OutV out;
  int W, H, row0, row1;
  M4 projection_view, projection_inverse, camera_matrix_world;
  M4 view_matrix;       // normal texture only
  float res_x, res_y;   // uniform `resolution` (the target's unrounded size)
  int general;          // scaled target, a `resolution` other than W x H or a normal texture: hbao_kernel<true>
  float ao_distance, distance_power, bias, thickness;
  int spp;
  BlueD blue;
  const float2* rot_table;
};
cudaError_t launch_hbao(const HbaoArgs& a, cudaStream_t s, const PeerPV* carry = nullptr);  // carry: as launch_poisson's, `out`

// K6h: horizon-march AO (an extension; DESIGN.md §1)
struct HbaoHorizonArgs {
  PV depth;
  PV normal;  // RGBA8 view-space normal (NormalPass layout) or p == nullptr: rebuilt from depth
  OutV out;
  int W, H, row0, row1;
  M4 projection, projection_inverse, camera_matrix_world;
  M4 view_matrix;       // normal texture only
  float res_x, res_y;   // the target's unrounded size
  float distance, dist2, inv_dist2, angle_bias, intensity, max_radius_pixels;
  int directions, steps;
  int fast;             // SFU sqrt / reciprocal for the per-tap values
  BlueD blue;
  const float2* dirs;   // [directions][256] (cos, sin)
};
cudaError_t launch_hbao_horizon(const HbaoHorizonArgs& a, cudaStream_t s, const PeerPV* carry = nullptr);  // carry: as launch_hbao's

struct AoComposeArgs {
  PV depth, ao, input;
  OutV out;
  int W, H, row0, row1;
  float power, color[3];
};
cudaError_t launch_ao_compose(const AoComposeArgs& a, cudaStream_t s);

struct MotionBlurArgs {
  PV velocity, input;
  OutV out;
  int W, H, row0, row1;
  float intensity, jitter, delta_time, res_x, res_y;
  int samples;
  BlueD blue;
};
cudaError_t launch_motion_blur(const MotionBlurArgs& a, cudaStream_t s);

struct TraaComposeArgs {
  PV acc;
  OutV out;
  int W, H, row0, row1;
};
cudaError_t launch_traa_compose(const TraaComposeArgs& a, cudaStream_t s);
// LINEAR sampler of an RGBA16F plane in device memory (motion_blur_px's taps)
struct PlaneH4 {
  const PV& t;
  RFX_D v4 linear(v2 uv) const { return tex_h4_linear(t, uv); }
};
// the same over a plane whose rows live on their owners (a row-sharded group)
struct PeerH4 {
  const PeerPV& t;
  RFX_D v4 linear(v2 uv) const { return peer_h4_linear(t, uv); }
};

// TRAAEffect + MotionBlurEffect as one EffectPass (the reference README's SSGI frame): K9's colour is K8's inputColor, and K8's taps
// sample the pass's input buffer `mb.input` (the frame before TRAA).  `mb.out` gets every pixel of rows [mb.row0, mb.row1).
// peer != nullptr: `mb.input` is ignored and the taps read peer->local's rows on their owners.
struct TraaMotionBlurArgs {
  MotionBlurArgs mb;
  PV acc;  // TRAA accumulated plane of this frame
};
cudaError_t launch_traa_motion_blur(const TraaMotionBlurArgs& a, cudaStream_t s, const PeerPV* peer = nullptr);
// K9 for pixel (x, y) of the W x H target (traa_compose.frag:3-6): the accumulated plane fetched LINEAR at the pixel centre, a = 1
RFX_D v4 traa_compose_px(const PV& acc, int x, int y, int W, int H) {
  const v4 t = tex_h4_linear(acc, pixel_uv(x, y, W, H));
  return mk4(t.x, t.y, t.z, 1.0f);
}

// merged cosmetic effects + TAAPass (k_fx.cu)
struct EffectsArgs {
  PV input, depth, velocity;
  OutV out;
  CamD cam;
  int W, H, row0, row1;
  int n_effects, effects[4];
  float texel_x, texel_y;  // postprocessing's texelSize = 1 / size (a JS double rounded to fp32)
  float sharpness, alphax, alphay, aberration, bg[3], max_distance, spread, intensity;
  int sparkle_perspective;
};
cudaError_t launch_effects(const EffectsArgs& a, cudaStream_t s);
struct TaaArgs {
  PV input, history;
  OutV out;
  int W, H, row0, row1;
  float camera_not_moved_frames;
  int srgb_output;
};
cudaError_t launch_taa(const TaaArgs& a, cudaStream_t s);

// G-buffer ingest (k_ingest.cu)
struct IngestArgs {
  PV albedo, normal, material, emissive, motion, depth;  // emissive.p / motion.p may be null
  OutV out_gb, out_vel;                                  // either .p may be null
  int W, H, row0, row1;
  int albedo_half, material_half, normal_f32, motion_f32, normalize_normals;
  float motion_sx, motion_sy;
};
cudaError_t launch_gbuffer_ingest(const IngestArgs& a, cudaStream_t s);

// env mip chain: dst (w1 x h1) = box filter of src (w0 x h0), RGBA16F
cudaError_t launch_env_downsample(PV src, OutV dst, int w1, int h1, cudaStream_t s);
// importance-sampling tables of an equirect map on the device (gatherData, EquirectHdrInfoUniform.js:149-245); 3 launches
cudaError_t launch_env_cdf(PV map, int flip_y, float* cdf_c, float* cdf_m, double* row_sum, double* total, float* marginal, float* conditional, cudaStream_t s);


// ==========================================================================================
// fast chain (k_chain.cu): the SSGI-mode chain of rfx_ssgi_chain_* with fast_math on.  Same passes, same tap geometry and
// decisions as the per-pass kernels above, but chain-internal plane formats chosen for the tap loops:
//   nrdz  16 B  (n.xyz, depth) + roughness code in the low mantissa bits          (decode prepass, once per frame)
//   tr    32 B  {diffuse rgba fp32, specular rgba fp32}                            K2 -> K3 pass 0 (NEAREST)
//   dn    16 B  {diffuse rgba fp16, specular rgba fp16}                            K3 ping-pong (LINEAR), K2 history, K4 input
// and the last Poisson pass also does the GI compose for its pixel (K4 has no neighbourhood in the fast variant).
// Row-sharded multi-GPU frames read last frame's `composed` / `dn` rows owned by other ranks in place over NVLink (PeerPV).
// ==========================================================================================
struct CDecodeArgs { PV gb, depth; OutV nrdz; int W, H; };
cudaError_t launch_cdecode(const CDecodeArgs& a, int row0, int row1, int halo, cudaStream_t s);

struct CTemporalArgs {
  PV input, velocity;   // K1 output (packed), velocity plane
  PeerPV hist;          // dn of the previous frame
  OutV out;             // tr
  int W, H, row0, row1;
  CamD cam;
  M4 prev_world, prev_proj_inv, prev_proj_view;
  float camera_pos[3];
  float max_blend, clamp_intensity, keep_data, confidence_power;
  float inv_w, inv_h;
  int full_accumulate;
};
cudaError_t launch_ctemporal(const CTemporalArgs& a, cudaStream_t s);

struct CPoissonArgs {
  PV nrdz, in;          // in: tr (pass 0) or dn (passes >= 1)
  OutV out;             // dn
  int W, H, row0, row1;
  float radius, phi, luma_phi, depth_phi, normal_phi, roughness_phi, specular_phi;
  BlueD blue;
  const float2* rot_table;
  float tap_ox[8], tap_oy[8];
  int first;            // pass 0: `in` is tr, NEAREST
  int reach_x, reach_y; // pixels a tap (incl. its bilinear footprint) can lie from its pixel: blocks further than that from every border skip all clamping
  // `out` is double-buffered by frame parity when it is the history plane: a discarded pixel (the reference's "target keeps its
  // texel", SURVEY.md A2) then copies last frame's texel forward.  carry.local.p == nullptr: single-buffered target, no write.
  PeerPV carry;
  // fused GI compose (last pass): rows [crow0, crow1) also write `composed` (discarded pixels carry last frame's texel forward)
  int compose;
  int crow0, crow1;
  PV gb;
  OutV composed;
  PeerPV composed_carry;
  CamD cam;
  // the chain's compose stage fused into K4 (rfx_ssgi_chain_set_compose): k5.out.p != nullptr selects the instantiations whose composing
  // pixels also store K5 of the texel they composed (k5.gi is not read; a discarded pixel is background, whose K5 is the scene texel)
  SsgiComposeArgs k5;
};
cudaError_t launch_cpoisson(const CPoissonArgs& a, cudaStream_t s);
struct CPoissonTmaArgs {  // passes >= 1 with TMA-staged tiles (experiment, RFX_K3_TMA=1)
  CPoissonArgs a;
  CUtensorMap map_in, map_nrdz;  // 2-D maps over the 16-byte texel planes as rows of 4-byte elements; box = box_w*4 x box_h
  int box_w, box_h;              // texels: 16 + 2 * reach_x, 16 + 2 * reach_y
};
// Whether a box_w x box_h texel tile can be staged through TMA: each box dimension at most 256 elements, and both tiles within the
// kernel's dynamic shared memory.  When it cannot, the pass runs launch_cpoisson (same bytes out).
bool cpoisson_tma_fits(int box_w, int box_h);
cudaError_t launch_cpoisson_tma(const CPoissonTmaArgs& t, cudaStream_t s);  // cudaErrorInvalidValue unless cpoisson_tma_fits

struct CComposeArgs {   // stand-alone K4 over dn (denoiseIterations == 0)
  PV nrdz, gb, dn;
  OutV composed;
  PeerPV composed_carry;
  int W, H, row0, row1;
  CamD cam;
  SsgiComposeArgs k5;  // as CPoissonArgs::k5
};
cudaError_t launch_ccompose(const CComposeArgs& a, cudaStream_t s);

// chain_output() views of the interleaved planes in the reference's formats
cudaError_t launch_split_tr(PV tr, OutV o0, OutV o1, int W, int H, cudaStream_t s);   // 32 B -> 2 x RGBA32F
cudaError_t launch_split_dn(PV dn, OutV o0, OutV o1, int W, int H, cudaStream_t s);   // 16 B -> 2 x RGBA16F

// common launch geometry: 256-thread blocks, 8 warps as 2 x 4 warp tiles of 8x4 pixels => 16x16 pixel tile
constexpr int kTileW = 16, kTileH = 16, kThreads = 256;
RFX_D void block_pixel(int& x, int& y, int row_base) {
  int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, lx, ly;
  lane_to_pixel(lane, lx, ly);
  x = blockIdx.x * kTileW + ((warp & 1) << 3) + lx;
  y = row_base + blockIdx.y * kTileH + ((warp >> 1) << 2) + ly;
}
// A launch over output rows [row0, row1) covers them with 16-row tiles starting at row0 & ~1, so that quads stay aligned to
// even rows.  range_pixel: the pixel of this thread; returns whether its row lies inside the range.  row_tiles: gridDim.y.
RFX_D bool range_pixel(int row0, int row1, int& x, int& y) {
  block_pixel(x, y, row0 & ~1);
  return y >= row0 && y < row1;
}
inline int row_tiles(int row0, int row1) { return (row1 - (row0 & ~1) + kTileH - 1) / kTileH; }

}  // namespace rfx
