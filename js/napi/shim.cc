// js/napi/shim.cc — N-API binding of include/rfx.h for a box that has Node + node_api.h.
//
// NOT BUILT IN THIS IMAGE: there is no `node`, no Node headers and no JS engine here (SURVEY.md D5); it is syntax-checked against
// a stub of the N-API prototypes it uses (tools/check_shim.sh).  This is the reference-side binding a maintainer adds, kept thin:
// every exported function forwards 1:1 to one `rfx_*` entry point of librfx.so and throws a JS Error carrying rfx_last_error() on a
// non-zero status.  Build (on such a box):
//   c++ -std=c++17 -shared -fPIC -I<node prefix>/include/node -I../../include shim.cc -L../../realism_effects_b200/csrc -lrfx -o rfx_napi.node
//
// JS-side types: ctx / chain / plane are externals; matrices are Float32Array(16); planes travel as externals created by planeAlloc
// (device memory) — host typed arrays cross only in planeUpload / planeDownload / envBuild / chainRenderHost.
#include <node_api.h>

#include <cstring>
#include <string>

#include "rfx.h"

namespace {

#define NAPI_OK(call) do { if ((call) != napi_ok) { napi_throw_error(env, nullptr, "N-API call failed: " #call); return nullptr; } } while (0)
#define ARGS(n) size_t argc = n; napi_value argv[n]; NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr))
#define CHECK(ctx, st, what) do { if ((st) != RFX_OK) return throw_status(env, ctx, st, what); } while (0)

napi_value throw_status(napi_env env, rfx_ctx* ctx, rfx_status st, const char* what) {
  std::string msg = std::string(what) + ": rfx status " + std::to_string((int)st) + " — " + (ctx ? rfx_last_error(ctx) : "no context");
  napi_throw_error(env, nullptr, msg.c_str());
  return nullptr;
}
template <class T>
T* unwrap(napi_env env, napi_value v) {
  napi_valuetype t;
  if (napi_typeof(env, v, &t) != napi_ok || t != napi_external) return nullptr;  // null / undefined => NULL (an unbound sampler)
  void* p = nullptr;
  napi_get_value_external(env, v, &p);
  return (T*)p;
}
napi_value external(napi_env env, void* p) { napi_value v; napi_create_external(env, p, nullptr, nullptr, &v); return v; }
napi_value undefined(napi_env env) { napi_value v; napi_get_undefined(env, &v); return v; }

void* typed_ptr(napi_env env, napi_value v, size_t* bytes = nullptr) {
  napi_valuetype vt;
  napi_typeof(env, v, &vt);
  if (vt == napi_null || vt == napi_undefined) return nullptr;
  napi_typedarray_type t; size_t len; void* data; napi_value ab; size_t off;
  if (napi_get_typedarray_info(env, v, &t, &len, &data, &ab, &off) != napi_ok) return nullptr;
  if (bytes) { const size_t es = (t == napi_float32_array || t == napi_uint32_array || t == napi_int32_array) ? 4 : (t == napi_uint16_array || t == napi_int16_array) ? 2 : (t == napi_float64_array) ? 8 : 1; *bytes = len * es; }
  return data;
}
bool read_f32(napi_env env, napi_value v, float* dst, size_t n) {
  napi_typedarray_type t; size_t len; void* data; napi_value ab; size_t off;
  if (napi_get_typedarray_info(env, v, &t, &len, &data, &ab, &off) != napi_ok || t != napi_float32_array || len < n) return false;
  std::memcpy(dst, data, n * sizeof(float));
  return true;
}
struct Obj {  // named-property reader with defaults
  napi_env env; napi_value o;
  bool has(const char* k) const { bool h = false; napi_has_named_property(env, o, k, &h); return h; }
  napi_value get(const char* k) const { napi_value v; napi_get_named_property(env, o, k, &v); return v; }
  double num(const char* k, double d) const { if (!has(k)) return d; double x = d; napi_valuetype t; napi_value v = get(k); napi_typeof(env, v, &t);
                                              if (t == napi_boolean) { bool b; napi_get_value_bool(env, v, &b); return b ? 1.0 : 0.0; }
                                              napi_get_value_double(env, v, &x); return x; }
  bool f32(const char* k, float* dst, size_t n) const { return has(k) && read_f32(env, get(k), dst, n); }
  void pair(const char* k, int32_t* dst) const {  // [a, b] numbers
    if (!has(k)) return;
    napi_value arr = get(k);
    for (uint32_t i = 0; i < 2; i++) { napi_value e; double d = 0; if (napi_get_element(env, arr, i, &e) == napi_ok) napi_get_value_double(env, e, &d); dst[i] = (int32_t)d; }
  }
  void floats(const char* k, float* dst, uint32_t n) const {  // plain JS array or Float32Array
    if (!has(k)) return;
    napi_value arr = get(k);
    if (read_f32(env, arr, dst, n)) return;
    for (uint32_t i = 0; i < n; i++) { napi_value e; double d = 0; if (napi_get_element(env, arr, i, &e) == napi_ok) napi_get_value_double(env, e, &d); dst[i] = (float)d; }
  }
};
bool read_camera(napi_env env, napi_value o, rfx_camera* c) {  // {projection, projectionInverse, matrixWorld, matrixWorldInverse, near, far, perspective}
  Obj b{env, o};
  if (!b.f32("projection", c->projection, 16) || !b.f32("projectionInverse", c->projection_inverse, 16) || !b.f32("matrixWorld", c->camera_matrix_world, 16) ||
      !b.f32("matrixWorldInverse", c->view_matrix, 16))
    return false;
  c->near_plane = (float)b.num("near", 0.1); c->far_plane = (float)b.num("far", 1000.0);
  c->perspective = (int32_t)b.num("perspective", 1);
  return true;
}
void read_chain_options(const Obj& b, rfx_ssgi_chain_options* o) {  // keys = src/ssgi/SSGIOptions.js names (+ width, height, flags, mode)
  o->width = (uint32_t)b.num("width", 0); o->height = (uint32_t)b.num("height", 0);
  o->denoise_iterations = (int32_t)b.num("denoiseIterations", 1); o->steps = (int32_t)b.num("steps", 20); o->refine_steps = (int32_t)b.num("refineSteps", 5);
  o->distance = (float)b.num("distance", 10); o->thickness = (float)b.num("thickness", 10); o->env_blur = (float)b.num("envBlur", 0.5);
  o->radius = (float)b.num("radius", 3); o->phi = (float)b.num("phi", 0.5); o->luma_phi = (float)b.num("lumaPhi", 5); o->depth_phi = (float)b.num("depthPhi", 2);
  o->normal_phi = (float)b.num("normalPhi", 50); o->roughness_phi = (float)b.num("roughnessPhi", 50); o->specular_phi = (float)b.num("specularPhi", 50);
  o->ssgi_flags = (uint32_t)b.num("flags", RFX_SSGI_USE_DIRECT_LIGHT); o->mode = (int32_t)b.num("mode", RFX_MODE_SSGI);
  o->blue_noise_start = (int32_t)b.num("blueNoiseStart", 1234567);
  o->resolution_scale = (float)b.num("resolutionScale", 1);
  o->denoise_mode = (int32_t)b.num("denoiseModeId", RFX_DENOISE_FULL);  // index of denoiseMode in ["full", "full_temporal", "temporal"]
}

// ---- context / planes -------------------------------------------------------------------------------------------------------
napi_value CtxCreate(napi_env env, napi_callback_info info) {  // ctxCreate(device) -> ctx
  ARGS(1);
  int32_t dev = 0; napi_get_value_int32(env, argv[0], &dev);
  rfx_ctx* ctx = nullptr;
  rfx_status st = rfx_ctx_create(dev, &ctx);
  CHECK(nullptr, st, "rfx_ctx_create");
  return external(env, ctx);
}
napi_value CtxDestroy(napi_env env, napi_callback_info info) { ARGS(1); rfx_ctx_destroy(unwrap<rfx_ctx>(env, argv[0])); return undefined(env); }
napi_value CtxSync(napi_env env, napi_callback_info info) { ARGS(1); rfx_ctx* c = unwrap<rfx_ctx>(env, argv[0]); CHECK(c, rfx_ctx_sync(c), "rfx_ctx_sync"); return undefined(env); }
napi_value SetFastMath(napi_env env, napi_callback_info info) {  // setFastMath(ctx, bool)
  ARGS(2); rfx_ctx* c = unwrap<rfx_ctx>(env, argv[0]); bool b = true; napi_get_value_bool(env, argv[1], &b);
  CHECK(c, rfx_ctx_set_fast_math(c, b), "rfx_ctx_set_fast_math"); return undefined(env);
}
napi_value BlueNoiseSet(napi_env env, napi_callback_info info) {  // blueNoiseSet(ctx, Uint8Array rgba, size)
  ARGS(3); rfx_ctx* ctx = unwrap<rfx_ctx>(env, argv[0]);
  uint32_t size = 0; napi_get_value_uint32(env, argv[2], &size);
  CHECK(ctx, rfx_blue_noise_set(ctx, (const uint8_t*)typed_ptr(env, argv[1]), size, size), "rfx_blue_noise_set");
  return undefined(env);
}
napi_value EnvBuild(napi_env env, napi_callback_info info) {  // envBuild(ctx, Uint16Array rgba16f, width, height[, flipY]) — CDF tables on the device
  ARGS(5); rfx_ctx* ctx = unwrap<rfx_ctx>(env, argv[0]);
  uint32_t w = 0, h = 0; napi_get_value_uint32(env, argv[2], &w); napi_get_value_uint32(env, argv[3], &h);
  bool flip = false; if (argc > 4) napi_get_value_bool(env, argv[4], &flip);
  CHECK(ctx, rfx_env_build(ctx, typed_ptr(env, argv[1]), w, h, flip), "rfx_env_build");
  return undefined(env);
}
napi_value EnvSet(napi_env env, napi_callback_info info) {  // envSet(ctx, map, width, height, marginal|null, conditional|null, totalSum) — host-built tables
  ARGS(7); rfx_ctx* ctx = unwrap<rfx_ctx>(env, argv[0]);
  rfx_env_desc e{};
  e.map_rgba16f = typed_ptr(env, argv[1]);
  napi_get_value_uint32(env, argv[2], &e.width); napi_get_value_uint32(env, argv[3], &e.height);
  e.marginal = (const float*)typed_ptr(env, argv[4]); e.conditional = (const float*)typed_ptr(env, argv[5]);
  double total = 0; napi_get_value_double(env, argv[6], &total);
  const double whole = (double)(int32_t)total;  // ~~totalSumValue (EquirectHdrInfoUniform.js:346-349)
  e.total_sum_whole = (float)whole; e.total_sum_decimal = (float)(total - whole);
  CHECK(ctx, rfx_env_set(ctx, &e), "rfx_env_set");
  return undefined(env);
}
napi_value EnvClear(napi_env env, napi_callback_info info) { ARGS(1); rfx_ctx* c = unwrap<rfx_ctx>(env, argv[0]); CHECK(c, rfx_env_clear(c), "rfx_env_clear"); return undefined(env); }

napi_value PlaneAlloc(napi_env env, napi_callback_info info) {  // planeAlloc(ctx, format, width, height) -> plane
  ARGS(4); rfx_ctx* ctx = unwrap<rfx_ctx>(env, argv[0]);
  int32_t fmt = 0; uint32_t w = 0, h = 0;
  napi_get_value_int32(env, argv[1], &fmt); napi_get_value_uint32(env, argv[2], &w); napi_get_value_uint32(env, argv[3], &h);
  rfx_plane* p = new rfx_plane();
  rfx_status st = rfx_plane_alloc(ctx, fmt, w, h, p);
  if (st != RFX_OK) { delete p; return throw_status(env, ctx, st, "rfx_plane_alloc"); }
  return external(env, p);
}
napi_value PlaneFree(napi_env env, napi_callback_info info) {  // planeFree(ctx, plane)
  ARGS(2); rfx_ctx* ctx = unwrap<rfx_ctx>(env, argv[0]); rfx_plane* p = unwrap<rfx_plane>(env, argv[1]);
  if (p) { rfx_plane_free(ctx, p); delete p; }
  return undefined(env);
}
napi_value PlaneUpload(napi_env env, napi_callback_info info) {  // planeUpload(ctx, plane, typedArray) — tightly packed rows
  ARGS(3); rfx_ctx* ctx = unwrap<rfx_ctx>(env, argv[0]); rfx_plane* p = unwrap<rfx_plane>(env, argv[1]);
  size_t bytes = 0; void* d = typed_ptr(env, argv[2], &bytes);
  if (!p || !d || bytes < (size_t)p->width * p->height * rfx_format_bytes(p->format)) { napi_throw_range_error(env, nullptr, "planeUpload: typed array smaller than the plane"); return nullptr; }
  CHECK(ctx, rfx_plane_upload(ctx, nullptr, p, d, 0), "rfx_plane_upload");
  return undefined(env);
}
napi_value PlaneDownload(napi_env env, napi_callback_info info) {  // planeDownload(ctx, plane, typedArray) — synchronous
  ARGS(3); rfx_ctx* ctx = unwrap<rfx_ctx>(env, argv[0]); rfx_plane* p = unwrap<rfx_plane>(env, argv[1]);
  size_t bytes = 0; void* d = typed_ptr(env, argv[2], &bytes);
  if (!p || !d || bytes < (size_t)p->width * p->height * rfx_format_bytes(p->format)) { napi_throw_range_error(env, nullptr, "planeDownload: typed array smaller than the plane"); return nullptr; }
  CHECK(ctx, rfx_plane_download(ctx, nullptr, p, d, 0), "rfx_plane_download");
  CHECK(ctx, rfx_ctx_sync(ctx), "rfx_ctx_sync");
  return undefined(env);
}

// ---- SSGI chain ---------------------------------------------------------------------------------------------------------------
napi_value ChainCreate(napi_env env, napi_callback_info info) {  // chainCreate(ctx, options) -> chain
  ARGS(2); rfx_ctx* ctx = unwrap<rfx_ctx>(env, argv[0]);
  rfx_ssgi_chain_options o{};
  read_chain_options(Obj{env, argv[1]}, &o);
  rfx_ssgi_chain* ch = nullptr;
  CHECK(ctx, rfx_ssgi_chain_create(ctx, &o, &ch), "rfx_ssgi_chain_create");
  return external(env, ch);
}
napi_value ChainSetOptions(napi_env env, napi_callback_info info) {  // chainSetOptions(ctx, chain, options) — reactive setters (reset the history)
  ARGS(3); rfx_ctx* ctx = unwrap<rfx_ctx>(env, argv[0]);
  rfx_ssgi_chain_options o{};
  read_chain_options(Obj{env, argv[2]}, &o);
  CHECK(ctx, rfx_ssgi_chain_set_options(unwrap<rfx_ssgi_chain>(env, argv[1]), &o), "rfx_ssgi_chain_set_options");
  return undefined(env);
}
napi_value ChainRender(napi_env env, napi_callback_info info) {  // chainRender(ctx, chain, camera, depth, gbuffer, velocity, direct|null, cameraPos, moved) — device planes
  ARGS(9); rfx_ctx* ctx = unwrap<rfx_ctx>(env, argv[0]);
  rfx_ssgi_frame f{};
  if (!read_camera(env, argv[2], &f.cam)) { napi_throw_type_error(env, nullptr, "camera: expected Float32Array(16) matrices"); return nullptr; }
  f.depth = unwrap<rfx_plane>(env, argv[3]); f.gbuffer = unwrap<rfx_plane>(env, argv[4]); f.velocity = unwrap<rfx_plane>(env, argv[5]);
  f.direct_light = unwrap<rfx_plane>(env, argv[6]);
  read_f32(env, argv[7], f.camera_pos, 3);
  bool moved = true; napi_get_value_bool(env, argv[8], &moved); f.camera_moved = moved;
  CHECK(ctx, rfx_ssgi_chain_render(unwrap<rfx_ssgi_chain>(env, argv[1]), nullptr, &f), "rfx_ssgi_chain_render");
  return undefined(env);
}
napi_value ChainOutput(napi_env env, napi_callback_info info) {  // chainOutput(ctx, chain, which) -> plane (borrowed: do not planeFree)
  ARGS(3); rfx_ctx* ctx = unwrap<rfx_ctx>(env, argv[0]);
  int32_t which = 0; napi_get_value_int32(env, argv[2], &which);
  rfx_plane* p = new rfx_plane();  // (a descriptor only; reclaimed with the JS object would need a finalizer: kept simple here)
  rfx_status st = rfx_ssgi_chain_output(unwrap<rfx_ssgi_chain>(env, argv[1]), which, p);
  if (st != RFX_OK) { delete p; return throw_status(env, ctx, st, "rfx_ssgi_chain_output"); }
  napi_value v;
  napi_create_external(env, p, [](napi_env, void* data, void*) { delete (rfx_plane*)data; }, nullptr, &v);
  return v;
}
// chainRenderHost(ctx, chain, camera, depth:Float32Array, gbuffer:Float32Array, velocity:Float32Array, direct:Uint16Array|null,
//                 cameraPos:Float32Array(3), cameraMoved:boolean, out:Float32Array[, sync:boolean = true])
napi_value ChainRenderHost(napi_env env, napi_callback_info info) {
  ARGS(11); rfx_ctx* ctx = unwrap<rfx_ctx>(env, argv[0]);
  rfx_ssgi_chain* ch = unwrap<rfx_ssgi_chain>(env, argv[1]);
  rfx_ssgi_host_frame f{};
  if (!read_camera(env, argv[2], &f.cam)) { napi_throw_type_error(env, nullptr, "camera: expected Float32Array(16) matrices"); return nullptr; }
  f.depth = (const float*)typed_ptr(env, argv[3]); f.gbuffer = (const float*)typed_ptr(env, argv[4]); f.velocity = (const float*)typed_ptr(env, argv[5]);
  f.direct_light = (const uint16_t*)typed_ptr(env, argv[6]);
  read_f32(env, argv[7], f.camera_pos, 3);
  bool moved = true; napi_get_value_bool(env, argv[8], &moved); f.camera_moved = moved;
  f.out_composed = (float*)typed_ptr(env, argv[9]);
  // `sync` selects the synchronous call; otherwise the frame is only enqueued (pipelined H2D / kernels / D2H) and the caller
  // pairs it with chainWaitHost(ctx, chain, 1) - the typed arrays of a frame must stay alive and untouched until it completed.
  bool sync = true;
  if (argc > 10) napi_get_value_bool(env, argv[10], &sync);
  rfx_status st = sync ? rfx_ssgi_chain_render_host(ch, &f) : rfx_ssgi_chain_submit_host(ch, &f);
  CHECK(ctx, st, sync ? "rfx_ssgi_chain_render_host" : "rfx_ssgi_chain_submit_host");
  return undefined(env);
}
napi_value ChainWaitHost(napi_env env, napi_callback_info info) {  // chainWaitHost(ctx, chain, maxInFlight)
  ARGS(3); rfx_ctx* ctx = unwrap<rfx_ctx>(env, argv[0]);
  int32_t n = 0; napi_get_value_int32(env, argv[2], &n);
  CHECK(ctx, rfx_ssgi_chain_wait_host(unwrap<rfx_ssgi_chain>(env, argv[1]), n), "rfx_ssgi_chain_wait_host");
  return undefined(env);
}
napi_value ChainReset(napi_env env, napi_callback_info info) { ARGS(1); rfx_ssgi_chain_reset(unwrap<rfx_ssgi_chain>(env, argv[0])); return undefined(env); }
napi_value ChainDestroy(napi_env env, napi_callback_info info) { ARGS(1); rfx_ssgi_chain_destroy(unwrap<rfx_ssgi_chain>(env, argv[0])); return undefined(env); }
// chainEnableTraa(ctx, chain, {maxBlend, neighborhoodClampIntensity, confidencePower, logTransform, fullAccumulate,
//                              fog: {color, near, far, density, isFogExp2}, near, far, perspective, isDebug} | null)
// null turns the TRAA tail off; the defaults are the values TRAAEffect forces
napi_value ChainEnableTraa(napi_env env, napi_callback_info info) {
  ARGS(3); rfx_ctx* ctx = unwrap<rfx_ctx>(env, argv[0]);
  napi_valuetype t = napi_undefined;
  napi_typeof(env, argv[2], &t);
  if (t != napi_object) { CHECK(ctx, rfx_ssgi_chain_enable_traa(unwrap<rfx_ssgi_chain>(env, argv[1]), nullptr), "rfx_ssgi_chain_enable_traa"); return undefined(env); }
  Obj b{env, argv[2]};
  rfx_traa_tail_options o{};
  o.max_blend = (float)b.num("maxBlend", 0.9); o.neighborhood_clamp_intensity = (float)b.num("neighborhoodClampIntensity", 1);
  o.confidence_power = (float)b.num("confidencePower", 4); o.log_transform = (int32_t)b.num("logTransform", 1); o.full_accumulate = (int32_t)b.num("fullAccumulate", 0);
  rfx_ssgi_compose_params& p = o.compose;
  p.camera_near = (float)b.num("near", 0.1); p.camera_far = (float)b.num("far", 1000); p.perspective = (int32_t)b.num("perspective", 1); p.is_debug = (int32_t)b.num("isDebug", 0);
  if (b.has("fog")) {
    Obj f{env, b.get("fog")};
    p.use_fog = 1; p.fog_exp2 = (int32_t)f.num("isFogExp2", 0); f.floats("color", p.fog_color, 3);
    p.fog_near = (float)f.num("near", 1); p.fog_far = (float)f.num("far", 1000); p.fog_density = (float)f.num("density", 0.00025);
  }
  CHECK(ctx, rfx_ssgi_chain_enable_traa(unwrap<rfx_ssgi_chain>(env, argv[1]), &o), "rfx_ssgi_chain_enable_traa");
  return undefined(env);
}

// ---- per-pass launches (one per reference fullscreen draw; whole planes) ------------------------------------------------------------
// ssgiCompose(ctx, depth, gi, scene, out[, {fog: {color, near, far, density, isFogExp2}, near, far, perspective, isDebug}]); with isDebug, gi is the
// debug view: any R32F / RGBA16F / RGBA32F plane of any size (depth / scene are not read then and may be null)
napi_value SsgiCompose(napi_env env, napi_callback_info info) {
  ARGS(6); rfx_ctx* c = unwrap<rfx_ctx>(env, argv[0]);
  rfx_ssgi_compose_params p{};
  napi_valuetype t = napi_undefined;
  if (argc > 5) napi_typeof(env, argv[5], &t);
  if (t == napi_object) {
    Obj b{env, argv[5]};
    p.camera_near = (float)b.num("near", 0.1); p.camera_far = (float)b.num("far", 1000); p.perspective = (int32_t)b.num("perspective", 1); p.is_debug = (int32_t)b.num("isDebug", 0);
    if (b.has("fog")) {
      Obj f{env, b.get("fog")};
      p.use_fog = 1; p.fog_exp2 = (int32_t)f.num("isFogExp2", 0); f.floats("color", p.fog_color, 3);
      p.fog_near = (float)f.num("near", 1); p.fog_far = (float)f.num("far", 1000); p.fog_density = (float)f.num("density", 0.00025);
    }
  }
  CHECK(c, rfx_ssgi_compose_launch(c, nullptr, t == napi_object ? &p : nullptr, unwrap<rfx_plane>(env, argv[1]), unwrap<rfx_plane>(env, argv[2]), unwrap<rfx_plane>(env, argv[3]),
                                   unwrap<rfx_plane>(env, argv[4]), 0, 0), "rfx_ssgi_compose_launch");
  return undefined(env);
}
napi_value TemporalReproject(napi_env env, napi_callback_info info) {  // temporalReproject(ctx, params, input, velocity, hist0, hist1|null, out0, out1|null)
  ARGS(8); rfx_ctx* c = unwrap<rfx_ctx>(env, argv[0]);
  Obj b{env, argv[1]};
  rfx_temporal_params p{};
  rfx_camera prev{};
  if (!read_camera(env, b.get("cam"), &p.cam) || !read_camera(env, b.get("prev"), &prev)) { napi_throw_type_error(env, nullptr, "temporalReproject: cam / prev camera blocks"); return nullptr; }
  std::memcpy(p.prev_view_matrix, prev.view_matrix, 64); std::memcpy(p.prev_camera_matrix_world, prev.camera_matrix_world, 64);
  std::memcpy(p.prev_projection, prev.projection, 64); std::memcpy(p.prev_projection_inverse, prev.projection_inverse, 64);
  b.f32("cameraPos", p.camera_pos, 3);
  p.max_blend = (float)b.num("maxBlend", 1); p.neighborhood_clamp_intensity = (float)b.num("neighborhoodClampIntensity", 1); p.keep_data = (float)b.num("keepData", 1);
  p.confidence_power = (float)b.num("confidencePower", 0.75); p.full_accumulate = (int32_t)b.num("fullAccumulate", 0); p.texture_count = (int32_t)b.num("textureCount", 1);
  p.input_type = (int32_t)b.num("inputType", RFX_INPUT_DIFFUSE); p.log_transform = (int32_t)b.num("logTransform", 0); p.history_linear = (int32_t)b.num("historyLinear", 1);
  b.pair("reprojectSpecular", p.reproject_specular);
  CHECK(c, rfx_temporal_reproject_launch(c, nullptr, &p, unwrap<rfx_plane>(env, argv[2]), unwrap<rfx_plane>(env, argv[3]), unwrap<rfx_plane>(env, argv[4]), unwrap<rfx_plane>(env, argv[5]),
                                         unwrap<rfx_plane>(env, argv[6]), unwrap<rfx_plane>(env, argv[7]), 0, 0), "rfx_temporal_reproject_launch");
  return undefined(env);
}
napi_value PoissonDenoise(napi_env env, napi_callback_info info) {  // poissonDenoise(ctx, params, depth, gbufferOrNormal, in0, in1|null, out0, out1|null)
  ARGS(8); rfx_ctx* c = unwrap<rfx_ctx>(env, argv[0]);
  Obj b{env, argv[1]};
  rfx_poisson_params p{};
  p.radius = (float)b.num("radius", 3); p.phi = (float)b.num("phi", 0.5); p.luma_phi = (float)b.num("lumaPhi", 5); p.depth_phi = (float)b.num("depthPhi", 2);
  p.normal_phi = (float)b.num("normalPhi", 3.25); p.roughness_phi = (float)b.num("roughnessPhi", 0); p.specular_phi = (float)b.num("specularPhi", 0);
  p.texture_count = (int32_t)b.num("textureCount", 1); b.pair("isTextureSpecular", p.is_texture_specular);
  p.gbuffer_texture = (int32_t)b.num("gbufferTexture", 0); p.input_linear = (int32_t)b.num("inputLinear", 1); p.blue_noise_index = (int32_t)b.num("blueNoiseIndex", 1);
  CHECK(c, rfx_poisson_denoise_launch(c, nullptr, &p, unwrap<rfx_plane>(env, argv[2]), unwrap<rfx_plane>(env, argv[3]), unwrap<rfx_plane>(env, argv[4]), unwrap<rfx_plane>(env, argv[5]),
                                      unwrap<rfx_plane>(env, argv[6]), unwrap<rfx_plane>(env, argv[7]), 0, 0), "rfx_poisson_denoise_launch");
  return undefined(env);
}
napi_value GiCompose(napi_env env, napi_callback_info info) {  // giCompose(ctx, {cam, inputType}, depth, gbuffer, diffuse|null, specular|null, scene|null, out)
  ARGS(8); rfx_ctx* c = unwrap<rfx_ctx>(env, argv[0]);
  Obj b{env, argv[1]};
  rfx_compose_params p{};
  if (!read_camera(env, b.get("cam"), &p.cam)) { napi_throw_type_error(env, nullptr, "giCompose: cam"); return nullptr; }
  p.input_type = (int32_t)b.num("inputType", RFX_INPUT_DIFFUSE_SPECULAR);
  CHECK(c, rfx_gi_compose_launch(c, nullptr, &p, unwrap<rfx_plane>(env, argv[2]), unwrap<rfx_plane>(env, argv[3]), unwrap<rfx_plane>(env, argv[4]), unwrap<rfx_plane>(env, argv[5]),
                                 unwrap<rfx_plane>(env, argv[6]), unwrap<rfx_plane>(env, argv[7]), 0, 0), "rfx_gi_compose_launch");
  return undefined(env);
}
napi_value Hbao(napi_env env, napi_callback_info info) {  // hbao(ctx, params, depth, out[, normal]); params.viewMatrix (with a normal plane), params.resolution
  ARGS(5); rfx_ctx* c = unwrap<rfx_ctx>(env, argv[0]);
  Obj b{env, argv[1]};
  rfx_hbao_params p{};
  if (!b.f32("projectionView", p.projection_view, 16) || !b.f32("projectionInverse", p.projection_inverse, 16) || !b.f32("matrixWorld", p.camera_matrix_world, 16)) {
    napi_throw_type_error(env, nullptr, "hbao: projectionView / projectionInverse / matrixWorld"); return nullptr; }
  p.ao_distance = (float)b.num("aoDistance", 2); p.distance_power = (float)b.num("distancePower", 1); p.bias = (float)b.num("bias", 40); p.thickness = (float)b.num("thickness", 0.075);
  p.spp = (int32_t)b.num("spp", 8); p.blue_noise_index = (int32_t)b.num("blueNoiseIndex", 1);
  b.floats("viewMatrix", p.view_matrix, 16); b.floats("resolution", p.resolution, 2);  // absent: unused / {0, 0} = the out plane's size
  CHECK(c, rfx_hbao_launch_ex(c, nullptr, &p, unwrap<rfx_plane>(env, argv[2]), unwrap<rfx_plane>(env, argv[4]), unwrap<rfx_plane>(env, argv[3]), 0, 0),
        "rfx_hbao_launch_ex");
  return undefined(env);
}
napi_value HbaoHorizon(napi_env env, napi_callback_info info) {  // hbaoHorizon(ctx, params, depth, out[, normal]); K6h, horizon-march AO
  ARGS(5); rfx_ctx* c = unwrap<rfx_ctx>(env, argv[0]);
  Obj b{env, argv[1]};
  rfx_hbao_horizon_params p{};
  if (!b.f32("projection", p.projection, 16) || !b.f32("projectionInverse", p.projection_inverse, 16) || !b.f32("matrixWorld", p.camera_matrix_world, 16)) {
    napi_throw_type_error(env, nullptr, "hbaoHorizon: projection / projectionInverse / matrixWorld"); return nullptr; }
  p.distance = (float)b.num("distance", 2); p.angle_bias = (float)b.num("angleBias", 0.1); p.intensity = (float)b.num("intensity", 1);
  p.max_radius_pixels = (float)b.num("maxRadiusPixels", 64);
  p.directions = (int32_t)b.num("directions", 8); p.steps = (int32_t)b.num("steps", 32); p.blue_noise_index = (int32_t)b.num("blueNoiseIndex", 1);
  b.floats("viewMatrix", p.view_matrix, 16); b.floats("resolution", p.resolution, 2);  // absent: unused / {0, 0} = the out plane's size
  CHECK(c, rfx_hbao_horizon_launch(c, nullptr, &p, unwrap<rfx_plane>(env, argv[2]), unwrap<rfx_plane>(env, argv[3]), unwrap<rfx_plane>(env, argv[4])),
        "rfx_hbao_horizon_launch");
  return undefined(env);
}
napi_value AoCompose(napi_env env, napi_callback_info info) {  // aoCompose(ctx, {power, color}, depth, ao, input, out)
  ARGS(6); rfx_ctx* c = unwrap<rfx_ctx>(env, argv[0]);
  Obj b{env, argv[1]};
  rfx_ao_compose_params p{};
  p.power = (float)b.num("power", 2); b.floats("color", p.color, 3);
  CHECK(c, rfx_ao_compose_launch(c, nullptr, &p, unwrap<rfx_plane>(env, argv[2]), unwrap<rfx_plane>(env, argv[3]), unwrap<rfx_plane>(env, argv[4]), unwrap<rfx_plane>(env, argv[5]), 0, 0),
        "rfx_ao_compose_launch");
  return undefined(env);
}
napi_value MotionBlur(napi_env env, napi_callback_info info) {  // motionBlur(ctx, params, velocity, input, out)
  ARGS(5); rfx_ctx* c = unwrap<rfx_ctx>(env, argv[0]);
  Obj b{env, argv[1]};
  rfx_motion_blur_params p{};
  p.intensity = (float)b.num("intensity", 1); p.jitter = (float)b.num("jitter", 1); p.delta_time = (float)b.num("deltaTime", 1.0 / 60); p.frame = (int32_t)b.num("frame", 0);
  p.samples = (int32_t)b.num("samples", 16); b.floats("resolution", p.resolution, 2);
  CHECK(c, rfx_motion_blur_launch(c, nullptr, &p, unwrap<rfx_plane>(env, argv[2]), unwrap<rfx_plane>(env, argv[3]), unwrap<rfx_plane>(env, argv[4]), 0, 0), "rfx_motion_blur_launch");
  return undefined(env);
}
napi_value TraaCompose(napi_env env, napi_callback_info info) {  // traaCompose(ctx, accumulated, out)
  ARGS(3); rfx_ctx* c = unwrap<rfx_ctx>(env, argv[0]);
  CHECK(c, rfx_traa_compose_launch(c, nullptr, unwrap<rfx_plane>(env, argv[1]), unwrap<rfx_plane>(env, argv[2]), 0, 0), "rfx_traa_compose_launch");
  return undefined(env);
}

napi_value GbufferDebug(napi_env env, napi_callback_info info) {  // gbufferDebug(ctx, mode, gbuffer, out): GBufferDebugPass (mode 0..5; other values show emissive)
  ARGS(4); rfx_ctx* c = unwrap<rfx_ctx>(env, argv[0]);
  int32_t mode = 0; napi_get_value_int32(env, argv[1], &mode);
  CHECK(c, rfx_gbuffer_debug_launch(c, nullptr, mode, unwrap<rfx_plane>(env, argv[2]), unwrap<rfx_plane>(env, argv[3]), 0, 0), "rfx_gbuffer_debug_launch");
  return undefined(env);
}
napi_value ChainSetDebugView(napi_env env, napi_callback_info info) {  // chainSetDebugView(ctx, chain, view): RFX_DEBUG_VIEW_* (the TRAA tail's K5)
  ARGS(3); rfx_ctx* c = unwrap<rfx_ctx>(env, argv[0]);
  int32_t view = RFX_DEBUG_VIEW_NONE; napi_get_value_int32(env, argv[2], &view);
  CHECK(c, rfx_ssgi_chain_set_debug_view(unwrap<rfx_ssgi_chain>(env, argv[1]), view), "rfx_ssgi_chain_set_debug_view");
  return undefined(env);
}

// ---- row-sharded groups inside one process (a Node host drives every GPU from one process: no NCCL, no CUDA IPC) ----------------------------
napi_value GroupCreateInprocess(napi_env env, napi_callback_info info) {  // groupCreateInprocess(ctx, rank, world) -> group
  ARGS(3); rfx_ctx* c = unwrap<rfx_ctx>(env, argv[0]);
  int32_t rank = 0, world = 1; napi_get_value_int32(env, argv[1], &rank); napi_get_value_int32(env, argv[2], &world);
  rfx_group* g = nullptr;
  CHECK(c, rfx_group_create_inprocess(c, rank, world, &g), "rfx_group_create_inprocess");
  return external(env, g);
}
napi_value GroupAttachChainsInprocess(napi_env env, napi_callback_info info) {  // groupAttachChainsInprocess(ctx, [groups], [chains])
  ARGS(3); rfx_ctx* c = unwrap<rfx_ctx>(env, argv[0]);
  rfx_group* gs[8] = {}; rfx_ssgi_chain* cs[8] = {};
  int32_t n = 0;
  for (uint32_t i = 0; i < 8; i++) {
    napi_value eg, ec;
    if (napi_get_element(env, argv[1], i, &eg) != napi_ok || napi_get_element(env, argv[2], i, &ec) != napi_ok) break;
    gs[i] = unwrap<rfx_group>(env, eg); cs[i] = unwrap<rfx_ssgi_chain>(env, ec);
    if (!gs[i] || !cs[i]) break;
    n++;
  }
  CHECK(c, rfx_group_attach_chains_inprocess(gs, cs, n), "rfx_group_attach_chains_inprocess");
  return undefined(env);
}
napi_value GroupSetBounds(napi_env env, napi_callback_info info) {  // groupSetBounds(ctx, group, [world + 1 ascending rows])
  ARGS(3); rfx_ctx* c = unwrap<rfx_ctx>(env, argv[0]);
  rfx_group* g = unwrap<rfx_group>(env, argv[1]);
  uint32_t b[9] = {};
  const int32_t n = rfx_group_world(g);
  for (int32_t i = 0; i <= n && i < 9; i++) { napi_value e; double d = 0; if (napi_get_element(env, argv[2], (uint32_t)i, &e) == napi_ok) napi_get_value_double(env, e, &d); b[i] = (uint32_t)d; }
  CHECK(c, rfx_group_set_bounds(g, b), "rfx_group_set_bounds");
  return undefined(env);
}
napi_value GroupDestroy(napi_env env, napi_callback_info info) { ARGS(1); rfx_group_destroy(unwrap<rfx_group>(env, argv[0])); return undefined(env); }
napi_value ChainRenderSharded(napi_env env, napi_callback_info info) {  // chainRenderSharded(ctx, chain, camera, depth, gbuffer, velocity, direct|null, cameraPos, moved): this member's band
  ARGS(9); rfx_ctx* ctx = unwrap<rfx_ctx>(env, argv[0]);
  rfx_ssgi_frame f{};
  if (!read_camera(env, argv[2], &f.cam)) { napi_throw_type_error(env, nullptr, "camera: expected Float32Array(16) matrices"); return nullptr; }
  f.depth = unwrap<rfx_plane>(env, argv[3]); f.gbuffer = unwrap<rfx_plane>(env, argv[4]); f.velocity = unwrap<rfx_plane>(env, argv[5]);
  f.direct_light = unwrap<rfx_plane>(env, argv[6]);
  read_f32(env, argv[7], f.camera_pos, 3);
  bool moved = true; napi_get_value_bool(env, argv[8], &moved); f.camera_moved = moved;
  CHECK(ctx, rfx_ssgi_chain_render_sharded(unwrap<rfx_ssgi_chain>(env, argv[1]), nullptr, &f), "rfx_ssgi_chain_render_sharded");
  return undefined(env);
}

napi_value Effects(napi_env env, napi_callback_info info) {  // effects(ctx, {cam, effects: [ids], sharpness, alphax, alphay, aberration, backgroundColor, maxDistance, spread, intensity, sparklePerspective}, input, depth|null, velocity|null, out)
  ARGS(6); rfx_ctx* c = unwrap<rfx_ctx>(env, argv[0]);
  Obj b{env, argv[1]};
  rfx_effects_params p{};
  if (!read_camera(env, b.get("cam"), &p.cam)) { napi_throw_type_error(env, nullptr, "effects: cam"); return nullptr; }
  float ids[4] = {0, 0, 0, 0};
  p.n_effects = (int32_t)b.num("count", 1);
  b.floats("effects", ids, 4);
  for (int i = 0; i < 4; i++) p.effects[i] = (int32_t)ids[i];
  p.sharpness = (float)b.num("sharpness", 1); p.alphax = (float)b.num("alphax", -0.05); p.alphay = (float)b.num("alphay", -0.05); p.aberration = (float)b.num("aberration", 1);
  b.floats("backgroundColor", p.background_color, 3);
  p.max_distance = (float)b.num("maxDistance", 5); p.spread = (float)b.num("spread", 1); p.intensity = (float)b.num("intensity", 1);
  p.sparkle_perspective = (int32_t)b.num("sparklePerspective", 0);
  CHECK(c, rfx_effects_launch(c, nullptr, &p, unwrap<rfx_plane>(env, argv[2]), unwrap<rfx_plane>(env, argv[3]), unwrap<rfx_plane>(env, argv[4]), unwrap<rfx_plane>(env, argv[5]), 0, 0),
        "rfx_effects_launch");
  return undefined(env);
}
napi_value Taa(napi_env env, napi_callback_info info) {  // taa(ctx, {cameraNotMovedFrames, srgbOutput}, input, history|null, out)
  ARGS(5); rfx_ctx* c = unwrap<rfx_ctx>(env, argv[0]);
  Obj b{env, argv[1]};
  rfx_taa_params p{};
  p.camera_not_moved_frames = (float)b.num("cameraNotMovedFrames", 0); p.srgb_output = (int32_t)b.num("srgbOutput", 1);
  CHECK(c, rfx_taa_launch(c, nullptr, &p, unwrap<rfx_plane>(env, argv[2]), unwrap<rfx_plane>(env, argv[3]), unwrap<rfx_plane>(env, argv[4]), 0, 0), "rfx_taa_launch");
  return undefined(env);
}
napi_value GbufferIngest(napi_env env, napi_callback_info info) {  // gbufferIngest(ctx, {motionScale, normalizeNormals}, albedo, normal, material, emissive|null, motion|null, depth, outGbuffer|null, outVelocity|null)
  ARGS(10); rfx_ctx* c = unwrap<rfx_ctx>(env, argv[0]);
  Obj b{env, argv[1]};
  rfx_ingest_params p{};
  p.motion_scale[0] = p.motion_scale[1] = 1.0f;
  b.floats("motionScale", p.motion_scale, 2);
  p.normalize_normals = (int32_t)b.num("normalizeNormals", 1);
  CHECK(c, rfx_gbuffer_ingest_launch(c, nullptr, &p, unwrap<rfx_plane>(env, argv[2]), unwrap<rfx_plane>(env, argv[3]), unwrap<rfx_plane>(env, argv[4]), unwrap<rfx_plane>(env, argv[5]),
                                     unwrap<rfx_plane>(env, argv[6]), unwrap<rfx_plane>(env, argv[7]), unwrap<rfx_plane>(env, argv[8]), unwrap<rfx_plane>(env, argv[9]), 0, 0),
        "rfx_gbuffer_ingest_launch");
  return undefined(env);
}

napi_value Init(napi_env env, napi_value exports) {
#define FN(name, f) {name, nullptr, f, nullptr, nullptr, nullptr, napi_default, nullptr}
  napi_property_descriptor d[] = {
      FN("ctxCreate", CtxCreate), FN("ctxDestroy", CtxDestroy), FN("ctxSync", CtxSync), FN("setFastMath", SetFastMath), FN("blueNoiseSet", BlueNoiseSet),
      FN("envBuild", EnvBuild), FN("envSet", EnvSet), FN("envClear", EnvClear), FN("planeAlloc", PlaneAlloc), FN("planeFree", PlaneFree),
      FN("planeUpload", PlaneUpload), FN("planeDownload", PlaneDownload), FN("chainCreate", ChainCreate), FN("chainSetOptions", ChainSetOptions),
      FN("chainRender", ChainRender), FN("chainOutput", ChainOutput), FN("chainRenderHost", ChainRenderHost), FN("chainWaitHost", ChainWaitHost),
      FN("chainReset", ChainReset), FN("chainDestroy", ChainDestroy), FN("chainEnableTraa", ChainEnableTraa), FN("ssgiCompose", SsgiCompose), FN("temporalReproject", TemporalReproject),
      FN("poissonDenoise", PoissonDenoise), FN("giCompose", GiCompose), FN("hbao", Hbao), FN("hbaoHorizon", HbaoHorizon), FN("aoCompose", AoCompose), FN("motionBlur", MotionBlur),
      FN("traaCompose", TraaCompose), FN("gbufferDebug", GbufferDebug), FN("chainSetDebugView", ChainSetDebugView), FN("gbufferIngest", GbufferIngest), FN("effects", Effects), FN("taa", Taa),
      FN("groupCreateInprocess", GroupCreateInprocess), FN("groupAttachChainsInprocess", GroupAttachChainsInprocess), FN("groupSetBounds", GroupSetBounds),
      FN("groupDestroy", GroupDestroy), FN("chainRenderSharded", ChainRenderSharded),
  };
#undef FN
  napi_define_properties(env, exports, sizeof d / sizeof d[0], d);
  return exports;
}

}  // namespace

NAPI_MODULE(NODE_GYP_MODULE_NAME, Init)
