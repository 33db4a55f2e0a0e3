// tests/horizon_oracle.cpp — TEST INFRASTRUCTURE ONLY.  CPU oracle of K6h, the horizon-march AO pass (DESIGN.md §1 K6h).
//
// K6h is an extension: the reference has no direction x step loop (SURVEY.md D1), so there is no reference shader to pin this
// against.  It follows the written definition of rfx_hbao_horizon_launch (include/rfx.h) and reuses K6's pinned pieces for
// everything K6 already defines: getWorldPos, computeWorldNormal, the normal-texture branch (tests/ao_oracle.cpp) and the blue-noise
// texel.  tests/test_horizon_ao_cpu.py holds it to an independent numpy restatement of the same definition.
#include "ao_oracle.cpp"

#include <cmath>

namespace {

// theta = 2 pi (d + b / 255) / D in double, rounded to float: (cos, sin) at [2 * (d * 256 + b)]
void horizon_directions(int D, float* out) {
  for (int d = 0; d < D; d++)
    for (int b = 0; b < 256; b++) {
      const double theta = 2.0 * 3.14159265358979323846 * ((double)d + (double)b / 255.0) / (double)D;
      out[2 * (d * 256 + b)] = (float)std::cos(theta);
      out[2 * (d * 256 + b) + 1] = (float)std::sin(theta);
    }
}

struct HorizonShader : HbaoNormalTextureShader {
  mat4 projectionMatrix;
  bool useNormalTexture = false;
  float distance_ = 0, angleBias = 0, intensity = 0, maxRadiusPixels = 0;
  int directions = 0, steps = 0;
  std::vector<float> dirs;

  bool mainPx(int px, int py, vec4& out) const {
    vec2 vUv = pixelUv(px, py, W, H);
    float depth = textureLod0(depthTexture, vUv).x;
    if (depth == 1.0f) return false;
    vec3 P = getWorldPos(depth, vUv);
    vec3 N = useNormalTexture ? HbaoNormalTextureShader::getWorldNormal(vUv) : computeWorldNormal(vUv);
    vec4 vs = projectionMatrixInverse * vec4(vUv.x * 2.0f - 1.0f, vUv.y * 2.0f - 1.0f, depth * 2.0f - 1.0f, 1.0f);
    vec3 Pv = vs.xyz() / vs.w;
    float wClip = (projectionMatrix * vec4(Pv, 1.0f)).w;
    float rPx = distance_ * 0.5f * resolution.y * projectionMatrix.m[5] / wClip;
    float ao = 1.0f;
    if (rPx >= 1.0f) {
      float delta = gmin(rPx, maxRadiusPixels) / (float)(steps + 1);
      vec4 blue = bn.sample(vUv, resolution, blueNoiseIndex);  // K6's texel: (byte) / 255
      int br = (int)std::lround(blue.x * 255.0f);
      float j = blue.y;
      float dist2 = distance_ * distance_;
      float sum = 0.0f;
      for (int d = 0; d < directions; d++) {
        float dx = dirs[2 * (d * 256 + br)], dy = dirs[2 * (d * 256 + br) + 1];
        for (int k = 0; k < steps; k++) {
          float t = 1.0f + ((float)k + j) * delta;
          float ox = std::floor(dx * t + 0.5f), oy = std::floor(dy * t + 0.5f);
          vec2 uv(vUv.x + ox / resolution.x, vUv.y + oy / resolution.y);
          float sampleDepth = textureLod0(depthTexture, uv).x;  // NEAREST, clamp to edge
          vec3 V = getWorldPos(sampleDepth, uv) - P;
          float vv = dot(V, V);
          if (vv > 0.0f) sum += clampf(dot(N, V) / std::sqrt(vv) - angleBias, 0.0f, 1.0f) * clampf(1.0f - vv / dist2, 0.0f, 1.0f);
        }
      }
      ao = clampf(1.0f - intensity * sum / (float)(directions * steps), 0.0f, 1.0f);
    }
    out = vec4(N, ao);
    return true;
  }
};

}  // namespace

extern "C" {

void orc_horizon_directions(int D, float* out) { horizon_directions(D, out); }

// K6h.  out RGBA16F W x H (the AO target); depth R32F DW x DH (>= W x H); normal: RGBA8 DW x DH view-space normals or NULL;
// p->resolution {0, 0} = (W, H).  Background pixels untouched.
void orc_ao_hbao_horizon(const rfx_hbao_horizon_params* p, int W, int H, const float* depth, int DW, int DH, const uint8_t* normal,
                         const uint8_t* blue_noise, int bn_w, int bn_h, uint16_t* out) {
  HorizonShader s;
  s.W = W; s.H = H;
  s.projectionMatrix = load_mat4(p->projection);
  s.projectionMatrixInverse = load_mat4(p->projection_inverse);
  s.cameraMatrixWorld = load_mat4(p->camera_matrix_world);
  s.viewMatrix = load_mat4(p->view_matrix);
  s.depthTexture = mk(depth, DW, DH, F_R32F);
  s.useNormalTexture = normal != nullptr;
  if (normal) s.normalTexture = mk(normal, DW, DH, F_RGBA8);
  s.bn.tex = mk(blue_noise, bn_w, bn_h, F_RGBA8, false, true);
  const bool res_default = p->resolution[0] == 0.0f && p->resolution[1] == 0.0f;
  s.resolution = res_default ? vec2((float)W, (float)H) : vec2(p->resolution[0], p->resolution[1]);
  s.blueNoiseIndex = p->blue_noise_index;
  s.distance_ = p->distance; s.angleBias = p->angle_bias; s.intensity = p->intensity; s.maxRadiusPixels = p->max_radius_pixels;
  s.directions = p->directions; s.steps = p->steps;
  s.dirs.resize((size_t)p->directions * 512);
  horizon_directions(p->directions, s.dirs.data());
  hbao_run(s, out);
}

}  // extern "C"
