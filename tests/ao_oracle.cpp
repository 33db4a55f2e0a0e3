// tests/ao_oracle.cpp — TEST INFRASTRUCTURE ONLY.  The CPU oracle (oracle/rfx_oracle.cpp, compiled into this library with the
// same flags) extended by the reduced-resolution AO of AOEffect (src/ao/AOEffect.js:126-154) and the useNormalTexture branch of K6
// (hbao_utils.glsl:70-79).  Pinned bit for bit against the reference's own shaders by tests/test_reference_glsl_ao.py.
//
// AOEffect.setSize gives the AO pass a target of (int)(width * scale) x (int)(height * scale) whose `resolution` uniform is the
// unrounded product (AOPass.js:79-83; three keeps width * scale, GL truncates it for the texture).  hbao.frag runs on that grid: vUv
// comes from the target, depth is a NEAREST fetch of the full-size depth plane and computeWorldNormal works in depth texels
// (textureSize(depthTexture)), which HbaoShader already does once its planes have their own sizes.  The denoiser keeps the full size
// and its first pass samples the AO target LINEAR; with no denoise iteration ao_compose samples the AO target itself LINEAR.
#include "../oracle/rfx_oracle.cpp"

namespace {

// hbao.frag:64-96 with getWorldNormal's useNormalTexture branch (hbao_utils.glsl:70-79): the world normal is
// normalize((vec4(unpackRGBToNormal(texture(normalTexture, vUv).rgb), 1.) * viewMatrix).xyz), normalTexture RGBA8 NEAREST
struct HbaoNormalTextureShader : HbaoShader {
  Tex normalTexture;
  mat4 viewMatrix;

  vec3 getWorldNormal(vec2 uv) const {
    vec3 worldNormal = 2.0f * textureLod0(normalTexture, uv).xyz() - 1.0f;  // three <packing> unpackRGBToNormal
    worldNormal = (vec4(worldNormal, 1.0f) * viewMatrix).xyz();            // view-space to world-space
    return normalize(worldNormal);
  }
  bool mainPx(int px, int py, vec4& out) const {
    vec2 vUv = pixelUv(px, py, W, H);
    float depth = textureLod0(depthTexture, vUv).x;
    if (depth == 1.0f) return false;
    vec3 cameraPosition = (cameraMatrixWorld * vec4(0.0f, 0.0f, 0.0f, 1.0f)).xyz();
    vec3 worldPos = getWorldPos(depth, vUv);
    vec3 worldNormal = getWorldNormal(vUv);
    float ao = 0.0f, totalWeight = 0.0f;
    for (int i = 0; i < spp; i++) {  // getOcclusion :21-62 (same blue-noise value every iteration, A9)
      vec4 blueNoise = bn.sample(vUv, resolution, blueNoiseIndex);
      vec3 sampleWorldDir = SsgiShader::cosineSampleHemisphere(worldNormal, vec2(blueNoise.x, blueNoise.y));
      vec3 sampleWorldPos = worldPos + aoDistance * powcr(blueNoise.z, distancePower + 1.0f) * sampleWorldDir;
      vec4 sampleUv = projectionViewMatrix * vec4(sampleWorldPos, 1.0f);
      vec2 suv = vec2(sampleUv.x, sampleUv.y) / sampleUv.w;
      suv = suv * 0.5f + 0.5f;
      float sampleDepth = textureLod0(depthTexture, suv).x;
      float deltaDepth = depth - sampleDepth;
      float d = distance(sampleWorldPos, cameraPosition);
      deltaDepth *= 0.001f * d * d;
      float th = thickness * 0.01f;
      float theta = dot(worldNormal, sampleWorldDir);
      totalWeight += theta;
      if (deltaDepth < th) {
        float horizon = sampleDepth + deltaDepth * bias * 1000.0f;
        float occlusion = gmax(0.0f, horizon - depth) * theta;
        float m = gmax(0.0f, 1.0f - deltaDepth / th);
        occlusion = 10.0f * occlusion * m / d;
        occlusion = std::sqrt(occlusion);
        ao += occlusion;
      }
    }
    if (totalWeight > 0.0f) ao /= totalWeight;
    ao = clampf(1.0f - ao, 0.0f, 1.0f);
    out = vec4(worldNormal, ao);
    return true;
  }
};

template <class S>
void hbao_setup(S& s, const rfx_hbao_params* p, int W, int H, float res_x, float res_y, const float* depth, int DW, int DH, const uint8_t* blue_noise,
                int bn_w, int bn_h) {
  s.W = W; s.H = H;
  s.projectionViewMatrix = load_mat4(p->projection_view);
  s.projectionMatrixInverse = load_mat4(p->projection_inverse);
  s.cameraMatrixWorld = load_mat4(p->camera_matrix_world);
  s.depthTexture = mk(depth, DW, DH, F_R32F);
  s.bn.tex = mk(blue_noise, bn_w, bn_h, F_RGBA8, false, true);
  s.resolution = vec2(res_x, res_y);
  s.aoDistance = p->ao_distance; s.distancePower = p->distance_power; s.bias = p->bias; s.thickness = p->thickness;
  s.spp = p->spp; s.blueNoiseIndex = p->blue_noise_index;
}

template <class S>
void hbao_run(const S& s, uint16_t* out) {
#pragma omp parallel for schedule(dynamic, 4)
  for (int y = 0; y < s.H; y++)
    for (int x = 0; x < s.W; x++) {
      vec4 o;
      if (s.mainPx(x, y, o)) store_rgba16f(out, s.W, x, y, o);
    }
}

}  // namespace

extern "C" {

// K6.  out RGBA16F W x H (the AO target); depth R32F DW x DH (>= W x H); resolution = the target's unrounded size;
// normal: RGBA8 NW x NH view-space normals (useNormalTexture) or NULL; p->view_matrix is read only with it.  Discarded pixels untouched.
void orc_ao_hbao(const rfx_hbao_params* p, int W, int H, float res_x, float res_y, const float* depth, int DW, int DH, const uint8_t* normal, int NW,
                 int NH, const uint8_t* blue_noise, int bn_w, int bn_h, uint16_t* out) {
  if (!normal) {
    HbaoShader s;
    hbao_setup(s, p, W, H, res_x, res_y, depth, DW, DH, blue_noise, bn_w, bn_h);
    hbao_run(s, out);
    return;
  }
  HbaoNormalTextureShader s;
  hbao_setup(s, p, W, H, res_x, res_y, depth, DW, DH, blue_noise, bn_w, bn_h);
  s.normalTexture = mk(normal, NW, NH, F_RGBA8);
  s.viewMatrix = load_mat4(p->view_matrix);
  hbao_run(s, out);
}

// K3 (one AO denoiser pass): as orc_poisson_denoise, with in0 / in1 of IW x IH (sampled by uv; LINEAR for the AO target)
void orc_ao_poisson_denoise(const rfx_poisson_params* p, int W, int H, const float* depth, const float* gbuffer_or_normal, const void* in0,
                            const void* in1, int in_half, int IW, int IH, const uint8_t* blue_noise, int bn_w, int bn_h, uint16_t* out0, uint16_t* out1) {
  PoissonShader s;
  s.W = W; s.H = H;
  s.depthTexture = mk(depth, W, H, F_R32F);
  s.GBUFFER_TEXTURE = p->gbuffer_texture != 0;
  if (s.GBUFFER_TEXTURE) s.gBufferTexture = mk(gbuffer_or_normal, W, H, F_RGBA32F); else s.normalTexture = mk(gbuffer_or_normal, W, H, F_RGBA32F);
  int fmt = in_half ? F_RGBA16F : F_RGBA32F;
  s.inputTexture = mk(in0, IW, IH, fmt, p->input_linear != 0);
  s.inputTexture2 = mk(in1, IW, IH, fmt, p->input_linear != 0);
  s.bn.tex = mk(blue_noise, bn_w, bn_h, F_RGBA8, false, true);
  s.radius = p->radius; s.phi = p->phi; s.lumaPhi = p->luma_phi; s.depthPhi = p->depth_phi; s.normalPhi = p->normal_phi;
  s.roughnessPhi = p->roughness_phi; s.specularPhi = p->specular_phi;
  s.resolution = vec2((float)W, (float)H);  // PoissonDenoisePass.setSize: the pass's own (full) size
  s.textureCount = p->texture_count; s.blueNoiseIndex = p->blue_noise_index;
  s.isTextureSpecular[0] = p->is_texture_specular[0]; s.isTextureSpecular[1] = p->is_texture_specular[1];
  uint16_t* outs[2] = {out0, out1};
#pragma omp parallel for schedule(dynamic, 4)
  for (int y = 0; y < H; y++)
    for (int x = 0; x < W; x++) {
      vec4 o[2];
      if (!s.mainPx(x, y, o)) continue;
      for (int i = 0; i < p->texture_count; i++) store_rgba16f(outs[i], W, x, y, o[i]);
    }
}

// K7.  ao_compose.frag:6-16 with the ao plane AW x AH (sampled LINEAR by uv), depth / input / out W x H
void orc_ao_ao_compose(const rfx_ao_compose_params* p, int W, int H, const float* depth, const uint16_t* ao, int AW, int AH, const uint16_t* input,
                       uint16_t* out) {
  Tex d = mk(depth, W, H, F_R32F), a = mk(ao, AW, AH, F_RGBA16F, true), in = mk(input, W, H, F_RGBA16F, true);
  vec3 color(p->color[0], p->color[1], p->color[2]);
#pragma omp parallel for
  for (int y = 0; y < H; y++)
    for (int x = 0; x < W; x++) {
      vec2 uv = pixelUv(x, y, W, H);
      float unpackedDepth = textureLod0(d, uv).x;
      float aov = unpackedDepth > 0.9999f ? 1.0f : textureLod0(a, uv).w;
      aov = powcr(aov, p->power);
      vec3 aoColor = mix(color, vec3(1.0f), aov);
      vec4 inputColor = textureLod0(in, uv);
      aoColor *= inputColor.xyz();
      store_rgba16f(out, W, x, y, vec4(aoColor, inputColor.w));
    }
}

}  // extern "C"
