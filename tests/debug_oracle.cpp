// tests/debug_oracle.cpp — TEST INFRASTRUCTURE ONLY.  The CPU oracle (oracle/rfx_oracle.cpp, compiled into this library with the
// same flags) extended by the debug views of SSGIEffect's `outputTexture` (src/ssgi/SSGIEffect.js:228-251): GBufferDebugPass
// (src/gbuffer/debug/GBufferDebugPass.js) and K5's isDebug branch (ssgi_compose.frag:21-24) on a view of any format and size.
// Pinned bit for bit against the reference's own shaders by tests/test_debug_views_cpu.py.
#include "../oracle/rfx_oracle.cpp"

extern "C" {

// GBufferDebugPass on a W x H target over a W x H packed G-buffer (RGBA32F, NEAREST), out RGBA32F.  The shader's `depthTexture` is not
// in the material's uniforms, so three never binds it and its sampler keeps unit 0 = gBufferTexture: depth is gBuffer.r.
void orc_dbg_gbuffer_debug(int mode, int W, int H, const float* gbuffer, float* out) {
  const Tex g = mk(gbuffer, W, H, F_RGBA32F);
  for (int y = 0; y < H; y++)
    for (int x = 0; x < W; x++) {
      const vec2 vUv = pixelUv(x, y, W, H);
      const float depth = textureLod0(g, vUv).x;
      if (depth == 0.0f) { store_rgba32f(out, W, x, y, vec4(0.0f, 0.0f, 0.0f, 0.0f)); continue; }
      const Material mat = getMaterial(g, vUv);
      vec3 c;
      if (mode == 0) c = mat.diffuse.xyz();
      else if (mode == 1) c = vec3(mat.diffuse.w, mat.diffuse.w, mat.diffuse.w);
      else if (mode == 2) c = mat.normal;
      else if (mode == 3) c = vec3(mat.roughness, mat.roughness, mat.roughness);
      else if (mode == 4) c = vec3(mat.metalness, mat.metalness, mat.metalness);
      else c = mat.emissive;
      store_rgba32f(out, W, x, y, vec4(c, 1.0f));
    }
}

// K5 with isDebug: out (W x H RGBA16F) = textureLod(inputTexture, vUv, 0.) for a view of format fmt (F_R32F a depth texture, read as
// (d, 0, 0, 1); F_RGBA16F LINEAR; F_RGBA32F NEAREST) and size sw x sh
void orc_dbg_ssgi_compose_debug(int W, int H, int fmt, const void* view, int sw, int sh, uint16_t* out) {
  const Tex t = mk(view, sw, sh, fmt, fmt == F_RGBA16F);
  for (int y = 0; y < H; y++)
    for (int x = 0; x < W; x++) store_rgba16f(out, W, x, y, textureLod0(t, pixelUv(x, y, W, H)));
}

}  // extern "C"
