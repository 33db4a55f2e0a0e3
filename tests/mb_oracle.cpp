// tests/mb_oracle.cpp — TEST INFRASTRUCTURE ONLY.  The CPU oracle (oracle/rfx_oracle.cpp, compiled into this library with the same flags)
// extended by TRAAEffect and MotionBlurEffect merged into one EffectPass, `new EffectPass(camera, traaEffect, motionBlur)` as the
// reference README wires the SSGI frame (readme.md:141-151).  Pinned bit for bit against the reference's own shaders by
// tests/test_traa_motion_blur_cpu.py.
//
// postprocessing merges the two effects' mainImage()s into one program: traa_compose.frag's outputColor (fp32, alpha 1) is
// motion_blur.frag's inputColor, and MotionBlurEffect.update binds inputTexture to the pass's input buffer (MotionBlurEffect.js:87-90),
// the frame before TRAA, so the taps read that plane, not the TRAA result.  The per-pixel arithmetic is orc_motion_blur's (K8) with
// orc_traa_compose's colour (K9) as inputColor.
#include "../oracle/rfx_oracle.cpp"

extern "C" {

// velocity RGBA32F nearest, accumulated and input RGBA16F linear, out RGBA16F
void orc_traa_motion_blur(const rfx_motion_blur_params* p, int W, int H, const float* velocity, const uint16_t* accumulated, const uint16_t* input,
                          const uint8_t* blue_noise, int bn_w, int bn_h, uint16_t* out) {
  Tex vel = mk(velocity, W, H, F_RGBA32F), acc = mk(accumulated, W, H, F_RGBA16F, true), in = mk(input, W, H, F_RGBA16F, true);
  BlueNoise bn; bn.tex = mk(blue_noise, bn_w, bn_h, F_RGBA8, false, true);
  vec2 resolution(p->resolution[0], p->resolution[1]);
  float samplesFloat = (float)p->samples;
#pragma omp parallel for schedule(dynamic, 4)
  for (int y = 0; y < H; y++)
    for (int x = 0; x < W; x++) {
      vec2 vUv = pixelUv(x, y, W, H);
      vec4 inputColor = vec4(textureLod0(acc, vUv).xyz(), 1.0f);  // traa_compose.frag:3-6
      vec4 vt = textureLod0(vel, vUv);                              // motion_blur.frag:11-44 from here on
      vec2 velocityv(vt.x, vt.y);
      bool didMove = dot(velocityv, velocityv) > 0.000000001f;
      if (!didMove) { store_rgba16f(out, W, x, y, inputColor); continue; }
      velocityv = velocityv * p->intensity;
      vec4 blueNoise = bn.sample(vUv, resolution, p->frame);
      vec2 jitterOffset = p->jitter * velocityv * vec2(blueNoise.x, blueNoise.y);
      float frameSpeed = (1.0f / 100.0f) / p->delta_time;
      vec2 startUv = vUv + (jitterOffset - velocityv * 0.5f) * frameSpeed;
      vec2 endUv = vUv + (jitterOffset + velocityv * 0.5f) * frameSpeed;
      startUv = vec2(gmax(0.0f, startUv.x), gmax(0.0f, startUv.y));
      endUv = vec2(gmin(1.0f, endUv.x), gmin(1.0f, endUv.y));
      vec3 motionBlurredColor = inputColor.xyz();
      for (float i = 0.0f; i <= samplesFloat; i++) {
        vec2 reprojectedUv = mix(startUv, endUv, i / samplesFloat);
        motionBlurredColor += textureLod0(in, reprojectedUv).xyz();
      }
      motionBlurredColor /= samplesFloat + 2.0f;
      store_rgba16f(out, W, x, y, vec4(motionBlurredColor, inputColor.w));
    }
}

}  // extern "C"
