// C-ABI plumbing: context, errors, and the field entry point's argument validation / dispatch.
#include <float.h>
#include <stdarg.h>
#include <string.h>

#include <vector>

#include "field_common.cuh"
#include "train_ws.h"
#include "../../include/onerf_ext.h"

static thread_local char g_err[512] = "";

void onerf_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

extern "C" int onerf_abi_version(void) { return ONERF_ABI_VERSION; }
extern "C" const char* onerf_last_error(void) { return g_err; }

extern "C" int onerf_ctx_create(int device, onerf_ctx** out) {
  ONERF_CHECK_ARG(out, "null out pointer");
  int count = 0;
  ONERF_CUDA(cudaGetDeviceCount(&count));
  ONERF_CHECK_ARG(device >= 0 && device < count, "no such CUDA device");
  cudaDeviceProp prop;
  ONERF_CUDA(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0) {
    onerf_set_error("onerf_ctx_create: device %d is sm_%d%d; this library is built for sm_90a only (no fallback)",
                    device, prop.major, prop.minor);
    return ONERF_ERR_UNSUPPORTED;
  }
  ONERF_CUDA(cudaSetDevice(device));
  onerf_ctx* c = new onerf_ctx();
  c->device = device;
  c->num_sms = prop.multiProcessorCount;
  c->launches = 0;
  c->pack_tables = nullptr;
  void* diag = nullptr;
  const cudaError_t e = cudaHostAlloc(&diag, 16, cudaHostAllocMapped);
  if (e != cudaSuccess) {
    delete c;
    onerf_set_error("onerf_ctx_create: cudaHostAlloc failed: %s", cudaGetErrorString(e));
    return ONERF_ERR_CUDA;
  }
  memset(diag, 0, 16);
  c->tc_diag = static_cast<uint32_t*>(diag);
  *out = c;
  return ONERF_OK;
}

extern "C" int onerf_ctx_destroy(onerf_ctx* ctx) {
  if (ctx) {
    onerf_free_pack_tables(ctx);
    if (ctx->tc_diag) cudaFreeHost(ctx->tc_diag);
  }
  delete ctx;
  return ONERF_OK;
}

extern "C" int64_t onerf_ctx_launch_count(const onerf_ctx* ctx) { return ctx ? ctx->launches : 0; }

// n_live: optional device-side count of the rays to evaluate (field_common.cuh: FieldParams::n_live)
static int field_fwd(onerf_ctx* ctx, const onerf_field_args* a, const int* n_live, void* stream_) {
  ONERF_CHECK_ARG(ctx && a, "null argument");
  ONERF_CHECK_ARG(a->rays && a->z && a->packed && a->ray_const, "null buffer");
  ONERF_CHECK_ARG(a->n_rays >= 0 && a->n_samples >= 1, "bad shape");
  ONERF_CHECK_ARG(a->want_scene || a->want_object, "nothing to compute");
  if (a->want_scene) ONERF_CHECK_ARG(a->scene_out && onerf_aligned16(a->scene_out), "scene_out null or misaligned");
  if (a->want_object) {
    ONERF_CHECK_ARG(a->obj_out && onerf_aligned16(a->obj_out), "obj_out null or misaligned");
    ONERF_CHECK_ARG(a->codes || a->code_row, "object branch needs codes or code_row");
  }
  ONERF_CHECK_ARG(a->n_boxes == 0 || a->boxes, "n_boxes > 0 with null boxes");
  ONERF_CHECK_ARG(a->z_stride >= a->n_samples && a->out_stride >= a->n_samples, "bad strides");
  int rc = onerf_check_grid(__func__, a->grid);
  if (rc != ONERF_OK || a->n_rays == 0) return rc;
  cudaStream_t stream = (cudaStream_t)stream_;
  FieldParams p = onerf_field_params(a->grid, a->packed);
  p.rays = a->rays; p.xyz = a->xyz; p.z = a->z; p.z_stride = a->z_stride;
  p.codes = a->codes; p.code_row = a->code_row;
  p.n_rays = a->n_rays; p.S = a->n_samples;
  p.want_scene = a->want_scene; p.want_object = a->want_object;
  p.mute_zero_rays = a->mute_zero_rays;
  p.boxes = a->boxes; p.n_boxes = a->n_boxes;
  p.scene_out = a->scene_out; p.obj_out = a->obj_out; p.out_stride = a->out_stride;
  p.ray_const = a->ray_const;
  p.n_live = n_live;
  if (a->activations) {
    ONERF_UNSUPPORTED(a->precision != ONERF_PREC_FP32, "activation dump is built for ONERF_PREC_FP32 only");
    ONERF_UNSUPPORTED(a->z_stride != a->n_samples || a->out_stride != a->n_samples, "activation dump needs dense z / outputs");
    for (int i = 0; i < 17; ++i) ONERF_CHECK_ARG(a->activations[i], "null activation matrix");
    p.dump_x = a->activations[0];
    for (int i = 0; i < 10; ++i) p.dump_s[i] = a->activations[1 + i];
    for (int i = 0; i < 6; ++i) p.dump_o[i] = a->activations[11 + i];
  }
  if (a->train_ws) {
    ONERF_UNSUPPORTED(a->precision != ONERF_PREC_BF16, "the training dump is written by the tensor-core (bf16) kernel");
    ONERF_UNSUPPORTED(!a->want_scene, "the training dump needs the scene branch");
    ONERF_UNSUPPORTED(a->z_stride != a->n_samples || a->out_stride != a->n_samples, "training dump needs dense z / outputs");
    ONERF_UNSUPPORTED(a->mute_zero_rays || a->n_boxes > 0, "editing extras have no backward");
    ONERF_CHECK_ARG((reinterpret_cast<uintptr_t>(a->train_ws) & 1023u) == 0, "train_ws must be 1024-byte aligned");
    p.train_ws = a->train_ws;
  }
  rc = onerf_launch_ray_const(ctx, p, stream);
  if (rc != ONERF_OK) return rc;
  if (a->precision == ONERF_PREC_FP32) return onerf_launch_field_fp32(ctx, p, stream);
  if (a->precision == ONERF_PREC_BF16) return onerf_launch_field_bf16(ctx, p, stream);
  onerf_set_error("onerf_field_fwd: unknown precision %d", a->precision);
  return ONERF_ERR_BAD_ARG;
}

extern "C" int onerf_field_fwd(onerf_ctx* ctx, const onerf_field_args* a, void* stream) {
  return field_fwd(ctx, a, nullptr, stream);
}

// ------------------------------------------------------------------------------------------------
// render_rays() forward as one call: composition of the stage entry points (same kernels, same order and seeds as
// object_nerf_b200/rendering.py::_render_forward, so both routes give bit-identical results).
// ------------------------------------------------------------------------------------------------
struct RenderWs {
  float *ray_const, *scene, *obj;   // per-ray hoisted terms, (rgb, sigma) of both branches
  size_t total;
};

static RenderWs render_ws_layout(char* base, int n_rays, int n_samples, int n_importance) {
  const size_t n = n_rays, sf = (size_t)n_samples + (size_t)n_importance;
  WsCarver c{base};
  RenderWs w;
  w.ray_const = c.floats(n * ONERF_RAY_CONST_FLOATS);
  w.scene = c.floats(n * sf * 4);
  w.obj = c.floats(n * sf * 4);
  w.total = c.off;
  return w;
}

extern "C" size_t onerf_render_rays_workspace_bytes(int n_rays, int n_samples, int n_importance) {
  if (n_rays < 0 || n_samples < 1 || n_importance < 0) return 0;
  return render_ws_layout(nullptr, n_rays, n_samples, n_importance).total;
}

static int render_pass(onerf_ctx* ctx, const onerf_render_args* a, const void* packed, const float* z, int S,
                       const onerf_render_maps& m, const float* noise_scene, const float* noise_obj, uint64_t seed,
                       float* ray_const, float* scene, float* obj, void* train_ws, const onerf_step_composite* step,
                       uint64_t* seed_dev, void* stream) {
  onerf_field_args f;
  memset(&f, 0, sizeof(f));
  f.train_ws = train_ws;
  f.rays = a->rays; f.z = z; f.z_stride = S;
  f.codes = a->forward_instance ? a->codes : nullptr;
  f.n_rays = a->n_rays; f.n_samples = S;
  f.grid = a->grid; f.packed = packed;
  f.want_scene = 1; f.want_object = a->forward_instance ? 1 : 0;
  f.precision = a->precision;
  f.scene_out = scene; f.obj_out = a->forward_instance ? obj : nullptr; f.out_stride = S;
  f.ray_const = ray_const;
  int rc = onerf_field_fwd(ctx, &f, stream);
  if (rc != ONERF_OK) return rc;
  onerf_composite_args c;
  memset(&c, 0, sizeof(c));
  c.z = z; c.scene = scene; c.obj = a->forward_instance ? obj : nullptr;
  c.n_rays = a->n_rays; c.n_samples = S;
  c.noise_std = a->noise_std; c.noise_scene = noise_scene; c.noise_obj = noise_obj; c.seed = seed;
  c.white_back = a->white_back; c.is_eval = a->is_eval; c.zero_last_delta = a->zero_last_delta;
  c.rays_in_bbox = a->rays_in_bbox; c.frustum_bound_th = a->frustum_bound_th;
  c.pass_through_mask = a->pass_through_mask;
  c.weights = m.weights; c.opacity = m.opacity; c.rgb = m.rgb; c.depth = m.depth;
  c.rgb_instance = m.rgb_instance; c.depth_instance = m.depth_instance; c.opacity_instance = m.opacity_instance;
  if (step && step->eval) return onerf_launch_composite_eval(ctx, &c, step, (cudaStream_t)stream);
  if (step) return onerf_launch_composite_step(ctx, &c, step, seed_dev, (cudaStream_t)stream);
  return onerf_launch_composite(ctx, &c, seed_dev, (cudaStream_t)stream);
}

static bool maps_ok(const onerf_render_maps& m, int forward_instance) {
  if (!(m.weights && m.opacity && m.z_vals && m.rgb && m.depth)) return false;
  return !forward_instance || (m.rgb_instance && m.depth_instance && m.opacity_instance);
}

extern "C" int onerf_render_rays_fwd(onerf_ctx* ctx, const onerf_render_args* a, void* stream) {
  return onerf_render_fwd_impl(ctx, a, nullptr, nullptr, stream);
}

extern "C" int onerf_render_rays_fwd_dseed(onerf_ctx* ctx, const onerf_render_args* a, uint64_t* seed_dev, void* stream) {
  ONERF_CHECK_ARG(ctx && a && seed_dev, "null argument");
  ONERF_CHECK_ARG((reinterpret_cast<uintptr_t>(seed_dev) & 7u) == 0, "seed_dev must be 8-byte aligned");
  ONERF_CHECK_ARG(!a->train_ws, "train_ws is refused: onerf_render_rays_bwd replays the noise from the host seed");
  const int rc = onerf_render_fwd_impl(ctx, a, nullptr, seed_dev, stream);
  if (rc != ONERF_OK) return rc;
  return onerf_launch_seed_advance(ctx, seed_dev, (cudaStream_t)stream);
}

int onerf_render_fwd_impl(onerf_ctx* ctx, const onerf_render_args* a, const onerf_step_composite* step, uint64_t* seed_dev,
                          void* stream) {
  ONERF_CHECK_ARG(ctx && a, "null argument");
  ONERF_CHECK_ARG(a->rays && a->packed_coarse, "null rays / packed_coarse");
  ONERF_CHECK_ARG(a->n_rays >= 0 && a->n_samples >= 2 && a->n_importance >= 0, "bad shape");
  // the importance sampler sorts S + K depths per ray in shared memory; refused here, before the coarse pass runs
  ONERF_UNSUPPORTED(a->n_importance > 0 && (int64_t)a->n_samples + a->n_importance > 2048, "S + K > 2048");
  ONERF_CHECK_ARG(!a->forward_instance || a->codes, "forward_instance needs codes");
  ONERF_CHECK_ARG(a->n_importance == 0 || a->packed_fine, "n_importance > 0 needs packed_fine");
  ONERF_CHECK_ARG(maps_ok(a->coarse, a->forward_instance), "null coarse output map");
  ONERF_CHECK_ARG(a->n_importance == 0 || maps_ok(a->fine, a->forward_instance), "null fine output map");
  const RenderWs w = render_ws_layout(reinterpret_cast<char*>(a->workspace), a->n_rays, a->n_samples, a->n_importance);
  int rc = onerf_check_workspace("onerf_render_rays_fwd", a->workspace, a->workspace_bytes, w.total, ONERF_ERR_WORKSPACE);
  if (rc != ONERF_OK || a->n_rays == 0) return rc;
  const int S = a->n_samples, SF = a->n_samples + a->n_importance;
  // training: both passes' fields are kept in the training workspace, and with bf16 the backward operands too (the fp32
  // backward re-runs the FFMA forward chunk by chunk instead)
  float *scene_c = w.scene, *obj_c = w.obj, *scene_f = w.scene, *obj_f = w.obj;
  void *tl_c = nullptr, *tl_f = nullptr;
  if (a->train_ws) {
    ONERF_CHECK_ARG((reinterpret_cast<uintptr_t>(a->train_ws) & 1023u) == 0, "train_ws must be 1024-byte aligned");
    const TrainWs W = onerf_make_train_ws(a->precision, onerf_train_use_voxel(a), a->n_rays, a->n_samples, a->n_importance);
    if (a->train_ws_bytes < (size_t)W.total) {
      onerf_set_error("onerf_render_rays_fwd: training workspace too small (%zu < %lld)", a->train_ws_bytes, (long long)W.total);
      return ONERF_ERR_WORKSPACE;
    }
    char* t = reinterpret_cast<char*>(a->train_ws);
    scene_c = reinterpret_cast<float*>(t + W.scene_c); obj_c = reinterpret_cast<float*>(t + W.obj_c);
    scene_f = reinterpret_cast<float*>(t + W.scene_f); obj_f = reinterpret_cast<float*>(t + W.obj_f);
    if (a->precision == ONERF_PREC_BF16) { tl_c = t + W.tl_coarse; tl_f = t + W.tl_fine; }
  }
  // training step: the coarse pass's field gradients go to the step's extension of the workspace, the fine pass's where
  // onerf_render_rays_bwd puts them; the fine pass (or the coarse one without importance samples) finalizes the loss
  onerf_step_composite step_c, step_f;
  if (step && step->eval) {
    // validation: both passes add their squared errors to the record; the last pass carries the PSNR
    step_c = step_f = *step;
    step_c.fine = 0; step_f.fine = 1;
    if (a->n_importance > 0) step_c.psnr = 0;
  } else if (step) {
    ONERF_CHECK_ARG(a->train_ws, "the training step needs a training workspace");
    const TrainWs W = onerf_make_train_ws(a->precision, onerf_train_use_voxel(a), a->n_rays, a->n_samples, a->n_importance);
    const TrainStepWs T = onerf_make_train_step_ws(W, a->n_rays, a->n_samples);
    char* t = reinterpret_cast<char*>(a->train_ws);
    step_c = step_f = *step;
    step_c.fine = 0; step_c.finalize = a->n_importance == 0;
    step_c.dscene = reinterpret_cast<float*>(t + T.dscene_c); step_c.dobj = reinterpret_cast<float*>(t + T.dobj_c);
    step_f.fine = 1; step_f.finalize = 1;
    step_f.dscene = reinterpret_cast<float*>(t + W.dscene); step_f.dobj = reinterpret_cast<float*>(t + W.dobj);
  }
  // seeds: coarse depths, coarse noise, importance u, fine noise (rendering.py::_render_forward); with seed_dev the kernels
  // add *seed_dev to these offsets
  const uint64_t seed = seed_dev ? 0 : a->seed;
  rc = onerf_launch_sample_coarse(ctx, a->rays, a->n_rays, S, a->use_disp, a->perturb, a->jitter, seed, seed_dev,
                                  a->coarse.z_vals, stream);
  if (rc != ONERF_OK) return rc;
  rc = render_pass(ctx, a, a->packed_coarse, a->coarse.z_vals, S, a->coarse, a->noise_scene_coarse, a->noise_obj_coarse,
                   seed + 1, w.ray_const, scene_c, obj_c, tl_c, step ? &step_c : nullptr, seed_dev, stream);
  if (rc != ONERF_OK || a->n_importance == 0) return rc;
  rc = onerf_launch_sample_pdf_merge(ctx, a->coarse.z_vals, a->coarse.weights, a->n_rays, S, a->n_importance,
                                     a->perturb == 0.0f ? 1 : 0, a->u, seed + 2, seed_dev, a->fine.z_vals, stream);
  if (rc != ONERF_OK) return rc;
  return render_pass(ctx, a, a->packed_fine, a->fine.z_vals, SF, a->fine, a->noise_scene_fine, a->noise_obj_fine, seed + 3,
                     w.ray_const, scene_f, obj_f, tl_f, step ? &step_f : nullptr, seed_dev, stream);
}

// ------------------------------------------------------------------------------------------------
// render_rays_multi() forward as one call (render_tools/multi_rendering.py:160-325): per ray set coarse depths and a
// one-branch field evaluation (scene branch + removed-object boxes for id 0, object branch with the id's code row
// otherwise, zero-length rays muted), joint stable depth sort + compositing, per-set importance resampling, fine pass.
// Same kernels, order and arguments as object_nerf_b200/multi_rendering.py::render_rays_multi (staged route), except that
// object sets evaluate only the rays that hit their box (multi_fields); the outputs are bit-identical.
// ------------------------------------------------------------------------------------------------
struct MultiWs {
  float *ray_const, *z_all, *z_fine, *field_all, *w_unsorted;
  int *live, *slot, *count;                // box culling of one object set (reused set after set)
  float *rays_c, *z_c, *field_c;
  void* sort;                              // onerf_composite_multi_ws scratch
  size_t sort_bytes;
  size_t total;
};

static MultiWs multi_ws_layout(char* base, int n_rays, int n_obj, int n_samples, int n_importance) {
  const size_t sf = (size_t)n_samples + (size_t)n_importance, no = (size_t)n_obj, n = (size_t)n_rays;
  MultiWs w;
  WsCarver c{base};
  w.ray_const = c.floats(n * ONERF_RAY_CONST_FLOATS);   // per-ray hoisted terms (one set at a time)
  w.z_all = c.floats(no * n * n_samples);               // coarse depths of every set
  w.z_fine = c.floats(no * n * sf);                     // fine depths
  w.field_all = c.floats(no * n * sf * 4);              // fields (rgb, sigma) of every set
  w.w_unsorted = c.floats(no * n * n_samples);          // per-set coarse weights in sample order
  w.live = static_cast<int*>(c.take(n * sizeof(int)));
  w.slot = static_cast<int*>(c.take(n * sizeof(int)));
  w.count = static_cast<int*>(c.take(sizeof(int)));
  w.rays_c = c.floats(n * 8);
  w.z_c = c.floats(n * sf);
  w.field_c = c.floats(n * sf * 4);
  w.sort_bytes = onerf_composite_multi_workspace_bytes(n_rays, n_obj, (int)sf);
  w.sort = c.take(w.sort_bytes);
  w.total = c.off;
  return w;
}

extern "C" size_t onerf_render_multi_workspace_bytes(int n_rays, int n_obj, int n_samples, int n_importance) {
  if (n_rays < 0 || n_obj < 1 || n_samples < 1 || n_importance < 0) return 0;
  return multi_ws_layout(nullptr, n_rays, n_obj, n_samples, n_importance).total;
}

// Where each set of an edited frame comes from (onerf_render_edit_frame_scenes): its scene's grid, weights and code table,
// and k = float(s_src / s_base), the factor that puts the set's depths on the frame's axis (1 for the base scene).
struct SetSource {
  const onerf_grid* grid;
  const void* packed_coarse;
  const void* packed_fine;
  const float* code_table;
  float k;
};

// The sets of one pass (pass 0 coarse, 1 fine); with `src`, set i reads its grid, weights and code row from src[i]
// instead of from `a` and `packed`.
static int multi_fields(onerf_ctx* ctx, const onerf_render_multi_args* a, const void* packed, const float* z_all, int S,
                        const MultiWs& w, void* stream, const SetSource* src = nullptr, int pass = 0) {
  const int N = a->n_rays;
  for (int i = 0; i < a->n_obj; ++i) {
    const int id = a->obj_ids_host[i];
    const float* z = z_all + (size_t)i * N * S;
    float* out = w.field_all + (size_t)i * N * S * 4;
    const float* code_table = src ? src[i].code_table : a->code_table;
    onerf_field_args f;
    memset(&f, 0, sizeof(f));
    f.rays = a->rays_list_host[i];
    f.z = z;
    f.z_stride = S;
    f.code_row = id > 0 ? code_table + (size_t)id * ONERF_NCODE : nullptr;
    f.n_rays = N; f.n_samples = S;
    f.grid = src ? src[i].grid : a->grid;
    f.packed = src ? (pass ? src[i].packed_fine : src[i].packed_coarse) : packed;
    f.want_scene = id > 0 ? 0 : 1; f.want_object = id > 0 ? 1 : 0;
    f.precision = a->precision;
    f.mute_zero_rays = 1;
    if (id == 0) { f.boxes = a->boxes; f.n_boxes = a->n_boxes; }
    f.scene_out = id > 0 ? nullptr : out;
    f.obj_out = id > 0 ? w.field_c : nullptr;
    f.out_stride = S;
    f.ray_const = w.ray_const;
    int rc;
    if (id == 0) {   // the scene set is evaluated on every ray
      f.scene_out = out;
      rc = field_fwd(ctx, &f, nullptr, stream);
      if (rc != ONERF_OK) return rc;
      continue;
    }
    // object set: only the rays that hit the box (the others would be muted), then scatter back with the muted value
    rc = onerf_cull_rays(ctx, f.rays, z, N, S, w.live, w.slot, w.count, w.rays_c, w.z_c, (cudaStream_t)stream);
    if (rc != ONERF_OK) return rc;
    f.rays = w.rays_c;
    f.z = w.z_c;
    rc = field_fwd(ctx, &f, w.count, stream);
    if (rc != ONERF_OK) return rc;
    rc = onerf_uncull_field(ctx, w.field_c, w.slot, N, S, out, (cudaStream_t)stream);
    if (rc != ONERF_OK) return rc;
  }
  return ONERF_OK;
}

// The argument checks of onerf_render_multi_fwd, reported under the entry `fn`.  with_rays_and_maps = 0 leaves out the ray
// sets and the outputs (onerf_render_edit_frame makes both itself).
// set_scene: NULL, or per set -1 (base scene) or the index of its source scene, whose ids the caller checks.
static int check_multi_args(const char* fn, const onerf_render_multi_args* a, bool with_rays_and_maps,
                            const int* set_scene = nullptr) {
  FN_CHECK_ARG((a->rays_list_host || !with_rays_and_maps) && a->obj_ids_host && a->packed_coarse && a->grid && a->code_table,
               "null input");
  FN_CHECK_ARG(a->n_rays >= 0 && a->n_obj >= 1 && a->n_samples >= 2 && a->n_importance >= 0, "bad shape");
  FN_UNSUPPORTED((int64_t)a->n_obj * (a->n_samples + a->n_importance) > INT32_MAX, "n_obj * samples >= 2^31");
  FN_UNSUPPORTED(a->n_samples + a->n_importance > 2048, "more than 2048 samples per ray set");
  FN_CHECK_ARG(a->n_importance == 0 || a->packed_fine, "n_importance > 0 needs packed_fine");
  FN_CHECK_ARG(a->n_boxes == 0 || a->boxes, "n_boxes > 0 with null boxes");
  for (int i = 0; i < a->n_obj; ++i) {
    if (with_rays_and_maps) FN_CHECK_ARG(a->rays_list_host[i], "null ray set");
    if (!set_scene || set_scene[i] < 0)
      FN_CHECK_ARG(a->obj_ids_host[i] >= 0 && a->obj_ids_host[i] < a->n_codes, "object id outside the code table");
  }
  if (!with_rays_and_maps) return ONERF_OK;
  const onerf_render_multi_maps& c = a->coarse;
  FN_CHECK_ARG(c.weights && c.opacity && c.z_vals && c.rgb && c.depth && c.obj_ids, "null coarse output");
  if (a->n_importance > 0)
    FN_CHECK_ARG(a->fine.weights && a->fine.opacity && a->fine.z_vals && a->fine.rgb && a->fine.depth, "null fine output");
  return ONERF_OK;
}

// The checks of onerf_render_multi_fwd_ext's extension block against the call's arguments.
static int check_multi_ext(const char* fn, const onerf_render_multi_args* a, const onerf_render_multi_ext* x) {
  FN_CHECK_ARG(x->noise_std >= 0.0f && x->noise_std <= FLT_MAX, "noise_std must be finite and >= 0");
  FN_CHECK_ARG(!(x->noise_coarse || x->noise_fine) || x->noise_std != 0.0f, "a noise buffer with noise_std = 0");
  FN_CHECK_ARG(!x->noise_fine || a->n_importance > 0, "noise_fine without a fine pass");
  FN_CHECK_ARG(onerf_aligned4(x->noise_coarse) && onerf_aligned4(x->noise_fine), "noise buffers must be 4-byte aligned");
  for (int i = 0; i < a->n_obj; ++i) {
    const float* u = x->u_list_host ? x->u_list_host[i] : nullptr;
    const float* clip = x->clip_list_host ? x->clip_list_host[i] : nullptr;
    FN_CHECK_ARG(!u || (a->n_importance > 0 && a->perturb != 0.0f), "a u buffer with perturb = 0 or without a fine pass");
    FN_CHECK_ARG(onerf_aligned4(u), "u buffers must be 4-byte aligned");
    FN_CHECK_ARG(onerf_aligned8(clip), "clip buffers must be 8-byte aligned");
  }
  return ONERF_OK;
}
// The per-set maps multi_forward writes (onerf_render_edit_frame_sets): the chunk's rows of each pass's outputs, and
// where the fine pass's weights go in set order ((n_obj, N, S + K), the edit workspace's extension).
struct SetMapsOut {
  onerf_set_maps coarse, fine;
  float* w_fine;
};

static bool any_set_map(const onerf_set_maps& m) { return m.opacity || m.depth || m.rgb; }

// The sets' sources of an edited frame with source scenes (multi_forward): per set its SetSource; with `rescale` (some
// set has k != 1) each pass composites a frame-axis copy of its depths, z_frame ((n_obj, N, S + K), the edit
// workspace's extension).
struct FrameScenes {
  const SetSource* set;
  bool rescale;
  float* z_frame;
};

static int multi_forward(onerf_ctx* ctx, const onerf_render_multi_args* a, const onerf_render_multi_ext& x, void* stream,
                         const SetMapsOut* sets = nullptr, const FrameScenes* scenes = nullptr);

static int render_multi_fwd(const char* fn, onerf_ctx* ctx, const onerf_render_multi_args* a,
                            const onerf_render_multi_ext* ext, void* stream) {
  int rc = check_multi_args(fn, a, true);
  if (rc != ONERF_OK) return rc;
  onerf_render_multi_ext none;
  memset(&none, 0, sizeof(none));
  const onerf_render_multi_ext& x = ext ? *ext : none;
  rc = check_multi_ext(fn, a, &x);
  if (rc != ONERF_OK) return rc;
  rc = onerf_check_workspace(fn, a->workspace, a->workspace_bytes,
                             onerf_render_multi_workspace_bytes(a->n_rays, a->n_obj, a->n_samples, a->n_importance),
                             ONERF_ERR_WORKSPACE);
  if (rc != ONERF_OK) return rc;
  return multi_forward(ctx, a, x, stream);
}

extern "C" int onerf_render_multi_fwd(onerf_ctx* ctx, const onerf_render_multi_args* a, void* stream) {
  ONERF_CHECK_ARG(ctx && a, "null argument");
  return render_multi_fwd(__func__, ctx, a, nullptr, stream);
}

extern "C" int onerf_render_multi_fwd_ext(onerf_ctx* ctx, const onerf_render_multi_args* a, const onerf_render_multi_ext* ext,
                                          void* stream) {
  ONERF_CHECK_ARG(ctx && a, "null argument");
  return render_multi_fwd(__func__, ctx, a, ext, stream);
}

// One pass's depths z_all (n_obj, N, S) on the frame's axis, in fs.z_frame: copied, then each set with k != 1 rewritten
// as z k, with its sigmas in field_all divided by k.  z_all keeps the sets' own units for their importance sampling.
static int to_frame_axis(onerf_ctx* ctx, const FrameScenes& fs, int n_obj, const float* z_all, float* field_all, int N,
                         int S, void* stream) {
  const size_t per_set = (size_t)N * S;
  ONERF_CUDA(cudaMemcpyAsync(fs.z_frame, z_all, n_obj * per_set * sizeof(float), cudaMemcpyDeviceToDevice,
                             (cudaStream_t)stream));
  for (int i = 0; i < n_obj; ++i) {
    if (fs.set[i].k == 1.0f) continue;
    const int rc = onerf_launch_rescale_set(ctx, z_all + i * per_set, fs.z_frame + i * per_set, field_all + i * per_set * 4,
                                            (int64_t)per_set, fs.set[i].k, (cudaStream_t)stream);
    if (rc != ONERF_OK) return rc;
  }
  return ONERF_OK;
}

// The forward of onerf_render_multi_fwd_ext on checked arguments: n_rays rays of every set in a->rays_list_host, maps
// written to a->coarse / a->fine, scratch in a->workspace; with `sets`, each pass's per-set maps too, from its weights
// in set order while the pass's depths and fields are still in the workspace; with `scenes`, each set's field from its
// own scene, composited on the frame's depth axis.
static int multi_forward(onerf_ctx* ctx, const onerf_render_multi_args* a, const onerf_render_multi_ext& x, void* stream,
                         const SetMapsOut* sets, const FrameScenes* scenes) {
  const onerf_render_multi_maps& c = a->coarse;
  if (a->n_rays == 0) return ONERF_OK;
  const bool sets_c = sets && any_set_map(sets->coarse), sets_f = sets && any_set_map(sets->fine);
  const int S = a->n_samples, SF = a->n_samples + a->n_importance, N = a->n_rays, NO = a->n_obj;
  const MultiWs w = multi_ws_layout(reinterpret_cast<char*>(a->workspace), N, NO, S, a->n_importance);
  int rc;
  for (int i = 0; i < NO; ++i) {   // multi_rendering.py:196-213: coarse depths are never jittered on this path
    rc = onerf_sample_coarse(ctx, a->rays_list_host[i], N, S, a->use_disp, 0.0f, nullptr, 0, w.z_all + (size_t)i * N * S, stream);
    if (rc != ONERF_OK) return rc;
  }
  const SetSource* src = scenes ? scenes->set : nullptr;
  rc = multi_fields(ctx, a, a->packed_coarse, w.z_all, S, w, stream, src, 0);
  if (rc != ONERF_OK) return rc;
  const float* z_c = w.z_all;   // the depths the compositing and the set maps see
  if (scenes && scenes->rescale) {
    rc = to_frame_axis(ctx, *scenes, NO, w.z_all, w.field_all, N, S, stream);
    if (rc != ONERF_OK) return rc;
    z_c = scenes->z_frame;
  }
  rc = onerf_composite_multi_noise_ws(ctx, z_c, w.field_all, N, NO, S, a->white_back, x.noise_std, x.noise_coarse, a->seed,
                                      0, c.z_vals, c.weights, c.obj_ids,
                                      (a->n_importance > 0 || sets_c) ? w.w_unsorted : nullptr, c.opacity, c.rgb, c.depth,
                                      w.sort, w.sort_bytes, stream);
  if (rc == ONERF_OK && sets_c)
    rc = onerf_launch_set_maps(ctx, z_c, w.field_all, w.w_unsorted, N, NO, S, sets->coarse.opacity, sets->coarse.depth,
                               sets->coarse.rgb, (cudaStream_t)stream);
  if (rc != ONERF_OK || a->n_importance == 0) return rc;
  const int det = a->perturb == 0.0f ? 1 : 0;
  for (int i = 0; i < NO; ++i) {
    const float* u = x.u_list_host ? x.u_list_host[i] : nullptr;
    const float* clip = x.clip_list_host ? x.clip_list_host[i] : nullptr;
    rc = onerf_launch_sample_pdf_merge(ctx, w.z_all + (size_t)i * N * S, w.w_unsorted + (size_t)i * N * S, N, S,
                                       a->n_importance, det, u, det ? 0 : a->seed + (uint64_t)i, nullptr,
                                       w.z_fine + (size_t)i * N * SF, stream, clip);
    if (rc != ONERF_OK) return rc;
  }
  rc = multi_fields(ctx, a, a->packed_fine, w.z_fine, SF, w, stream, src, 1);
  if (rc != ONERF_OK) return rc;
  const float* z_f = w.z_fine;
  if (scenes && scenes->rescale) {
    rc = to_frame_axis(ctx, *scenes, NO, w.z_fine, w.field_all, N, SF, stream);
    if (rc != ONERF_OK) return rc;
    z_f = scenes->z_frame;
  }
  rc = onerf_composite_multi_noise_ws(ctx, z_f, w.field_all, N, NO, SF, a->white_back, x.noise_std, x.noise_fine,
                                      a->seed, 1, a->fine.z_vals, a->fine.weights, nullptr, sets_f ? sets->w_fine : nullptr,
                                      a->fine.opacity, a->fine.rgb, a->fine.depth, w.sort, w.sort_bytes, stream);
  if (rc != ONERF_OK || !sets_f) return rc;
  return onerf_launch_set_maps(ctx, z_f, w.field_all, sets->w_fine, N, NO, SF, sets->fine.opacity, sets->fine.depth,
                               sets->fine.rgb, (cudaStream_t)stream);
}

// ------------------------------------------------------------------------------------------------
// An edited frame from a camera (EditableRenderer.render_edit, editable_renderer.py:203-294): per chunk of pixels, every
// set's camera rays (onerf_camera_rays' kernel on the chunk's pixels), then multi_forward with the chunk's rows of the
// caller's maps.  Chunks are independent: every stage works per ray.
// ------------------------------------------------------------------------------------------------
struct EditWs {
  float* rays;                            // (n_obj, chunk, 8): every set's rays of the current chunk
  onerf_render_multi_maps coarse, fine;   // one chunk of each map, for the maps the caller leaves NULL
  void* multi;                            // workspace of multi_forward for one chunk
  size_t multi_bytes;
  size_t total;
  float* w_fine;                          // onerf_render_edit_frame_sets: the fine pass's weights in set order (SetMapsOut)
  size_t total_sets;
  float* z_frame;                         // onerf_render_edit_frame_scenes: a pass's depths on the frame's axis (FrameScenes)
  size_t total_scenes;
};

static EditWs edit_ws_layout(char* base, int chunk, int n_obj, int n_samples, int n_importance) {
  const size_t n = chunk, nf = n_importance > 0 ? n : 0, no = n_obj;
  const size_t tc = no * n_samples, tf = no * (n_samples + n_importance);
  EditWs w;
  WsCarver c{base};
  w.rays = c.floats(no * n * 8);
  w.coarse.weights = c.floats(n * tc); w.coarse.opacity = c.floats(n); w.coarse.z_vals = c.floats(n * tc);
  w.coarse.rgb = c.floats(n * 3); w.coarse.depth = c.floats(n); w.coarse.obj_ids = c.floats(n * tc);
  w.fine.weights = c.floats(nf * tf); w.fine.opacity = c.floats(nf); w.fine.z_vals = c.floats(nf * tf);
  w.fine.rgb = c.floats(nf * 3); w.fine.depth = c.floats(nf); w.fine.obj_ids = nullptr;
  w.multi_bytes = onerf_render_multi_workspace_bytes(chunk, n_obj, n_samples, n_importance);
  w.multi = c.take(w.multi_bytes);
  w.total = c.off;
  w.w_fine = c.floats(no * nf * (n_samples + n_importance));   // past everything onerf_render_edit_frame uses; 0 bytes
  w.total_sets = c.off;                                         // without a fine pass
  w.z_frame = c.floats(no * n * (n_samples + n_importance));
  w.total_scenes = c.off;
  return w;
}

// rows [r0, ...) of a caller's map of `width` floats per row, or `scratch` where the caller leaves the map NULL
static float* rows_or(float* out, int64_t r0, int64_t width, float* scratch) { return out ? out + r0 * width : scratch; }

// rows [r0, r0 + chunk) of the tile's maps (T samples per row), or the chunk scratch where a map is NULL
static onerf_render_multi_maps chunk_maps(const onerf_render_multi_maps& out, const onerf_render_multi_maps& scratch,
                                          int64_t r0, int64_t T) {
  onerf_render_multi_maps m;
  m.weights = rows_or(out.weights, r0, T, scratch.weights);
  m.opacity = rows_or(out.opacity, r0, 1, scratch.opacity);
  m.z_vals = rows_or(out.z_vals, r0, T, scratch.z_vals);
  m.rgb = rows_or(out.rgb, r0, 3, scratch.rgb);
  m.depth = rows_or(out.depth, r0, 1, scratch.depth);
  m.obj_ids = rows_or(out.obj_ids, r0, T, scratch.obj_ids);
  return m;
}

extern "C" size_t onerf_render_edit_workspace_bytes(int chunk_rays, int n_obj, int n_samples, int n_importance) {
  if (chunk_rays < 1 || onerf_render_multi_workspace_bytes(chunk_rays, n_obj, n_samples, n_importance) == 0) return 0;
  return edit_ws_layout(nullptr, chunk_rays, n_obj, n_samples, n_importance).total;
}

extern "C" size_t onerf_render_edit_sets_workspace_bytes(int chunk_rays, int n_obj, int n_samples, int n_importance) {
  if (onerf_render_edit_workspace_bytes(chunk_rays, n_obj, n_samples, n_importance) == 0) return 0;
  return edit_ws_layout(nullptr, chunk_rays, n_obj, n_samples, n_importance).total_sets;
}

extern "C" size_t onerf_render_edit_scenes_workspace_bytes(int chunk_rays, int n_obj, int n_samples, int n_importance) {
  if (onerf_render_edit_workspace_bytes(chunk_rays, n_obj, n_samples, n_importance) == 0) return 0;
  return edit_ws_layout(nullptr, chunk_rays, n_obj, n_samples, n_importance).total_scenes;
}

// rows [r0, r0 + chunk) of tile-sized per-set maps (n_obj columns), NULL where the caller's array is NULL
static onerf_set_maps chunk_set_maps(const onerf_set_maps& out, int64_t r0, int64_t n_obj) {
  return onerf_set_maps{rows_or(out.opacity, r0, n_obj, nullptr), rows_or(out.depth, r0, n_obj, nullptr),
                        rows_or(out.rgb, r0, n_obj * 3, nullptr)};
}

// onerf_render_edit_frame(_sets, _scenes), refusals reported under the entry `fn`
static int render_edit_frame(const char* fn, onerf_ctx* ctx, const onerf_render_edit_args* a, const onerf_set_maps* sets_c,
                             const onerf_set_maps* sets_f, const onerf_edit_scene* scenes, int n_scenes,
                             const int* set_scene, void* stream) {
  FN_CHECK_ARG(ctx && a && a->sets_host, "null argument");
  FN_CHECK_ARG(a->n_obj >= 1, "bad shape");
  FN_CHECK_ARG(a->H > 0 && a->W > 0 && a->focal > 0, "bad camera");
  const int64_t n_tile = a->pixel_end - a->pixel_begin;
  FN_CHECK_ARG(a->pixel_begin >= 0 && n_tile >= 0 && a->pixel_end <= (int64_t)a->H * a->W, "tile outside the frame");
  FN_CHECK_ARG(a->chunk_rays >= 1, "chunk_rays < 1");
  FN_CHECK_ARG(a->scale_factor > 0, "scale_factor must be positive");
  FN_CHECK_ARG(n_scenes >= 0 && (n_scenes == 0 || scenes), "null or negative source scene list");
  for (int j = 0; j < n_scenes; ++j) {
    const onerf_edit_scene& sc = scenes[j];
    FN_CHECK_ARG(sc.grid && sc.packed_coarse && sc.code_table, "a source scene needs its grid, packed_coarse and code_table");
    const int rc = onerf_check_grid(fn, sc.grid, " in a source scene");
    if (rc != ONERF_OK) return rc;
    FN_CHECK_ARG(a->n_importance == 0 || sc.packed_fine, "n_importance > 0 needs a source scene's packed_fine");
    const double k = sc.scale_factor / a->scale_factor;
    FN_CHECK_ARG(sc.scale_factor > 0 && sc.scale_factor <= DBL_MAX && (float)k > 0 && (float)k <= FLT_MAX,
                 "a source scene's scale_factor must be positive and finite");
  }
  const int NO = a->n_obj;
  std::vector<int> ids(NO);
  bool any_source = false;
  for (int i = 0; i < NO; ++i) {
    const onerf_edit_set& s = a->sets_host[i];
    const int j = set_scene ? set_scene[i] : -1;
    FN_CHECK_ARG(j >= -1 && j < n_scenes, "set scene index outside [-1, n_scenes)");
    if (j >= 0) {
      FN_UNSUPPORTED(s.obj_id == 0, "a set of a source scene must be an object set (obj_id > 0)");
      FN_CHECK_ARG(s.obj_id > 0 && s.obj_id < scenes[j].n_codes, "object id outside its source scene's code table");
      any_source = true;
    }
    FN_CHECK_ARG(s.obj_id == 0 || s.box, "an object set needs its box");
    FN_CHECK_ARG(s.obj_id != 0 || !s.box, "the scene set takes no box");
    ids[i] = s.obj_id;
  }
  const int chunk = a->chunk_rays;
  onerf_render_multi_args m;
  memset(&m, 0, sizeof(m));
  onerf_render_multi_ext no_ext;
  memset(&no_ext, 0, sizeof(no_ext));
  m.obj_ids_host = ids.data();
  m.n_obj = NO; m.n_rays = (int)(n_tile < chunk ? n_tile : chunk);
  m.n_samples = a->n_samples; m.n_importance = a->n_importance;
  m.grid = a->grid; m.packed_coarse = a->packed_coarse; m.packed_fine = a->packed_fine;
  m.code_table = a->code_table; m.n_codes = a->n_codes;
  m.precision = a->precision; m.use_disp = a->use_disp; m.perturb = 0.0f; m.seed = 0; m.white_back = a->white_back;
  m.boxes = a->boxes; m.n_boxes = a->n_boxes;
  int rc = check_multi_args(fn, &m, false, set_scene);
  if (rc != ONERF_OK) return rc;
  const onerf_set_maps none = {nullptr, nullptr, nullptr};
  const onerf_set_maps& sc = sets_c ? *sets_c : none;
  const onerf_set_maps& sf = sets_f ? *sets_f : none;
  const bool with_sets = any_set_map(sc) || any_set_map(sf);
  FN_CHECK_ARG(!any_set_map(sf) || a->n_importance > 0, "fine set maps without a fine pass");
  for (const onerf_set_maps* p : {&sc, &sf})
    FN_CHECK_ARG(onerf_aligned4(p->opacity) && onerf_aligned4(p->depth) && onerf_aligned4(p->rgb),
                 "set maps must be 4-byte aligned");
  const size_t need = any_source ? onerf_render_edit_scenes_workspace_bytes(chunk, NO, a->n_samples, a->n_importance)
                     : with_sets  ? onerf_render_edit_sets_workspace_bytes(chunk, NO, a->n_samples, a->n_importance)
                                  : onerf_render_edit_workspace_bytes(chunk, NO, a->n_samples, a->n_importance);
  rc = onerf_check_workspace(fn, a->workspace, a->workspace_bytes, need, ONERF_ERR_WORKSPACE);
  if (rc != ONERF_OK) return rc;
  const EditWs w = edit_ws_layout(reinterpret_cast<char*>(a->workspace), chunk, NO, a->n_samples, a->n_importance);
  // sets of source scenes: every set's source (the base scene's for the others), k in float32 of the double ratio
  std::vector<SetSource> src;
  std::vector<double> set_scale(NO, a->scale_factor);
  FrameScenes fs = {nullptr, false, w.z_frame};
  if (any_source) {
    src.resize(NO);
    for (int i = 0; i < NO; ++i) {
      const int j = set_scene[i];
      src[i] = j < 0 ? SetSource{a->grid, a->packed_coarse, a->packed_fine, a->code_table, 1.0f}
                     : SetSource{scenes[j].grid, scenes[j].packed_coarse, scenes[j].packed_fine, scenes[j].code_table,
                                 (float)(scenes[j].scale_factor / a->scale_factor)};
      if (j >= 0) set_scale[i] = scenes[j].scale_factor;
      fs.rescale = fs.rescale || src[i].k != 1.0f;
    }
    fs.set = src.data();
  }
  std::vector<const float*> rays(NO);
  for (int i = 0; i < NO; ++i) rays[i] = w.rays + (size_t)i * chunk * 8;
  m.rays_list_host = rays.data();
  m.workspace = w.multi;
  m.workspace_bytes = w.multi_bytes;
  const int64_t TC = (int64_t)NO * a->n_samples, TF = (int64_t)NO * (a->n_samples + a->n_importance);
  for (int64_t r0 = 0; r0 < n_tile; r0 += chunk) {
    const int n = (int)(n_tile - r0 < chunk ? n_tile - r0 : chunk);
    for (int i = 0; i < NO; ++i) {
      const onerf_edit_set& s = a->sets_host[i];
      rc = onerf_launch_camera_rays(ctx, a->H, a->W, a->focal, s.Toc, s.box, set_scale[i], a->near, a->far,
                                    a->pixel_begin + r0, n, const_cast<float*>(rays[i]), nullptr, (cudaStream_t)stream);
      if (rc != ONERF_OK) return rc;
    }
    m.n_rays = n;
    m.coarse = chunk_maps(a->coarse, w.coarse, r0, TC);
    if (a->n_importance > 0) m.fine = chunk_maps(a->fine, w.fine, r0, TF);
    const SetMapsOut so = {chunk_set_maps(sc, r0, NO), chunk_set_maps(sf, r0, NO), w.w_fine};
    rc = multi_forward(ctx, &m, no_ext, stream, with_sets ? &so : nullptr, any_source ? &fs : nullptr);
    if (rc != ONERF_OK) return rc;
  }
  return ONERF_OK;
}

extern "C" int onerf_render_edit_frame(onerf_ctx* ctx, const onerf_render_edit_args* a, void* stream) {
  return render_edit_frame(__func__, ctx, a, nullptr, nullptr, nullptr, 0, nullptr, stream);
}

extern "C" int onerf_render_edit_frame_sets(onerf_ctx* ctx, const onerf_render_edit_args* a, const onerf_set_maps* coarse,
                                            const onerf_set_maps* fine, void* stream) {
  return render_edit_frame(__func__, ctx, a, coarse, fine, nullptr, 0, nullptr, stream);
}

extern "C" int onerf_render_edit_frame_scenes(onerf_ctx* ctx, const onerf_render_edit_args* a,
                                              const onerf_edit_scene* scenes_host, int n_scenes, const int* set_scene_host,
                                              const onerf_set_maps* coarse, const onerf_set_maps* fine, void* stream) {
  return render_edit_frame(__func__, ctx, a, coarse, fine, scenes_host, n_scenes, set_scene_host, stream);
}

// ------------------------------------------------------------------------------------------------
// A validation image (or a tile of it) in one call: the batch counts of the tile once, then per chunk a code gather and
// onerf_render_fwd_impl with the evaluation compositing, on the chunk's rows of the caller's maps.  Chunks are
// independent (every stage works per ray) and only add to the record.
// ------------------------------------------------------------------------------------------------
struct ValidateWs {
  float* codes;                     // (chunk,64)
  onerf_render_maps coarse, fine;   // one chunk of each map: the per-sample arrays, and the maps the caller leaves NULL
  void* render;                     // workspace of onerf_render_rays_fwd for one chunk
  size_t render_bytes;
  size_t total;
};

static ValidateWs validate_ws_layout(char* base, int chunk, int n_samples, int n_importance) {
  const size_t n = chunk, nf = n_importance > 0 ? n : 0;
  ValidateWs w;
  WsCarver c{base};
  auto maps = [&](size_t rows, size_t S) {
    onerf_render_maps m;
    m.weights = c.floats(rows * S); m.opacity = c.floats(rows); m.z_vals = c.floats(rows * S); m.rgb = c.floats(rows * 3);
    m.depth = c.floats(rows); m.rgb_instance = c.floats(rows * 3); m.depth_instance = c.floats(rows);
    m.opacity_instance = c.floats(rows);
    return m;
  };
  w.codes = c.floats(n * 64);
  w.coarse = maps(n, n_samples);
  w.fine = maps(nf, (size_t)n_samples + n_importance);
  w.render_bytes = onerf_render_rays_workspace_bytes(chunk, n_samples, n_importance);
  w.render = c.take(w.render_bytes);
  w.total = c.off;
  return w;
}

// rows [r0, ...) of the tile's maps, or the chunk scratch where a map is NULL; per-sample arrays always scratch
static onerf_render_maps validate_chunk_maps(const onerf_render_maps& out, const onerf_render_maps& scratch, int64_t r0) {
  onerf_render_maps m = scratch;
  m.opacity = rows_or(out.opacity, r0, 1, scratch.opacity);
  m.rgb = rows_or(out.rgb, r0, 3, scratch.rgb);
  m.depth = rows_or(out.depth, r0, 1, scratch.depth);
  m.rgb_instance = rows_or(out.rgb_instance, r0, 3, scratch.rgb_instance);
  m.depth_instance = rows_or(out.depth_instance, r0, 1, scratch.depth_instance);
  m.opacity_instance = rows_or(out.opacity_instance, r0, 1, scratch.opacity_instance);
  return m;
}

extern "C" size_t onerf_validate_workspace_bytes(int chunk_rays, int n_samples, int n_importance) {
  if (chunk_rays < 1 || n_samples < 2 || n_importance < 0) return 0;
  return validate_ws_layout(nullptr, chunk_rays, n_samples, n_importance).total;
}

extern "C" int onerf_validate_frame(onerf_ctx* ctx, const onerf_validate_args* v, void* stream) {
  ONERF_CHECK_ARG(ctx && v, "null argument");
  const onerf_render_args& ra = v->render;
  const onerf_loss_args& la = v->loss;
  const int64_t n_tile = v->ray_end - v->ray_begin;
  ONERF_CHECK_ARG(ra.n_rays >= 0 && ra.n_samples >= 2 && ra.n_importance >= 0, "bad shape");
  ONERF_CHECK_ARG(v->ray_begin >= 0 && n_tile >= 0 && v->ray_end <= ra.n_rays, "tile outside the image");
  ONERF_CHECK_ARG(v->chunk_rays >= 1, "chunk_rays < 1");
  ONERF_CHECK_ARG(ra.forward_instance, "TotalLoss needs the object branch's maps: forward_instance must be set");
  ONERF_CHECK_ARG(ra.is_eval, "validation renders with is_eval set");
  ONERF_CHECK_ARG(!ra.train_ws, "a training workspace is refused: validation keeps nothing for a backward");
  ONERF_CHECK_ARG(ra.perturb == 0.0f && ra.noise_std == 0.0f, "perturb and noise_std must be 0");
  ONERF_CHECK_ARG(v->record && (reinterpret_cast<uintptr_t>(v->record) & 7u) == 0, "record null or not 8-byte aligned");
  ONERF_CHECK_ARG(ra.rays && v->instance_ids && v->code_table, "null rays / instance_ids / code_table");
  ONERF_CHECK_ARG(la.rgbs && la.depths && la.valid_mask && la.instance_mask && la.instance_mask_weight, "null batch buffer");
  ONERF_CHECK_ARG(la.n_rays == ra.n_rays, "loss.n_rays differs from render.n_rays");
  ONERF_CHECK_ARG(v->psnr_mask == ONERF_PSNR_VALID_INSTANCE || v->psnr_mask == ONERF_PSNR_ALL_RAYS, "unknown psnr_mask");
  ONERF_CHECK_ARG(!v->finalize || (la.loss_sum_out && la.terms_out && la.present_out && v->psnr_out), "finalize with a null output");
  const int chunk = v->chunk_rays;
  int rc = onerf_check_workspace(__func__, ra.workspace, ra.workspace_bytes,
                                 onerf_validate_workspace_bytes(chunk, ra.n_samples, ra.n_importance), ONERF_ERR_BAD_ARG);
  if (rc != ONERF_OK) return rc;
  const ValidateWs w = validate_ws_layout(reinterpret_cast<char*>(ra.workspace), chunk, ra.n_samples, ra.n_importance);
  ONERF_CUDA(cudaMemsetAsync(v->record, 0, ONERF_VALIDATE_RECORD_DOUBLES * sizeof(double), (cudaStream_t)stream));
  // rows [first, first + n) of the image's batch
  auto batch_rows = [&](int64_t first, int64_t n) {
    onerf_loss_args l = la;
    l.n_rays = n;
    l.rgbs += first * 3; l.depths += first; l.valid_mask += first; l.instance_mask += first; l.instance_mask_weight += first;
    return l;
  };
  if (n_tile > 0) {
    const onerf_loss_args tile = batch_rows(v->ray_begin, n_tile);
    rc = onerf_launch_batch_stats(ctx, &tile, v->record, (cudaStream_t)stream);
    if (rc != ONERF_OK) return rc;
  }
  onerf_step_composite step;
  memset(&step, 0, sizeof(step));
  step.eval = 1;
  step.psnr = 1 + v->psnr_mask;
  step.acc = v->record;
  onerf_render_args c = ra;
  c.codes = w.codes;
  c.workspace = w.render; c.workspace_bytes = w.render_bytes;
  for (int64_t r0 = 0; r0 < n_tile; r0 += chunk) {
    const int n = (int)(n_tile - r0 < chunk ? n_tile - r0 : chunk);
    const int64_t first = v->ray_begin + r0;
    rc = onerf_code_gather(ctx, v->code_table, v->instance_ids + first, n, v->n_codes, w.codes, stream);
    if (rc != ONERF_OK) return rc;
    c.rays = ra.rays + first * 8;
    c.n_rays = n;
    c.coarse = validate_chunk_maps(ra.coarse, w.coarse, r0);
    if (ra.n_importance > 0) c.fine = validate_chunk_maps(ra.fine, w.fine, r0);
    step.loss = batch_rows(first, n);
    rc = onerf_render_fwd_impl(ctx, &c, &step, nullptr, stream);
    if (rc != ONERF_OK) return rc;
  }
  if (!v->finalize) return ONERF_OK;
  const float wt[5] = {la.color_weight, la.depth_weight, la.opacity_weight, la.instance_color_weight, la.instance_depth_weight};
  return onerf_validate_finalize(ctx, v->record, wt, ra.n_importance > 0, la.loss_sum_out, la.terms_out, la.present_out,
                                 v->psnr_out, stream);
}

// ------------------------------------------------------------------------------------------------
// Every object's maps of a tile of rays in one render (onerf_render_instances): per chunk the coarse depths, the K
// codes' per-ray constants, one field evaluation of the scene and every code, the scene compositing (whose weights
// feed the importance sampler) and one compositing launch of every object column, then the same for the fine pass.
// Same kernels, arguments and order of arithmetic as onerf_render_rays_fwd with is_eval and nothing random, so every
// column is bit-identical to that call with the column's code on every ray.
// ------------------------------------------------------------------------------------------------
struct InstancesWs {
  float *ray_const, *scene, *obj, *z_c, *w_c, *z_f, *w_f;
  onerf_instance_maps scratch;      // scene maps of one chunk, for those the caller leaves NULL
  int64_t rc_stride, obj_stride;    // floats between two codes' blocks of ray_const / obj
  size_t total;
};

static InstancesWs instances_ws_layout(char* base, int chunk, int n_codes, int n_samples, int n_importance) {
  const size_t n = chunk, K = n_codes, S = n_samples, SF = (size_t)n_samples + n_importance;
  const size_t nf = n_importance > 0 ? n : 0;
  InstancesWs w;
  WsCarver c{base};
  w.rc_stride = (int64_t)(n * ONERF_RAY_CONST_FLOATS);
  w.obj_stride = (int64_t)(n * SF * 4);
  w.ray_const = c.floats(K * n * ONERF_RAY_CONST_FLOATS);
  w.scene = c.floats(n * SF * 4);
  w.obj = c.floats(K * n * SF * 4);
  w.z_c = c.floats(n * S); w.w_c = c.floats(n * S);
  w.z_f = c.floats(nf * SF); w.w_f = c.floats(nf * SF);
  w.scratch = onerf_instance_maps{c.floats(n * 3), c.floats(n), c.floats(n), nullptr, nullptr, nullptr};
  w.total = c.off;
  return w;
}

extern "C" size_t onerf_render_instances_workspace_bytes(int chunk_rays, int n_codes, int n_samples, int n_importance) {
  if (chunk_rays < 1 || n_codes < 1 || n_codes > ONERF_INSTANCES_MAX_CODES || n_samples < 2 || n_importance < 0) return 0;
  return instances_ws_layout(nullptr, chunk_rays, n_codes, n_samples, n_importance).total;
}

static bool instance_maps_aligned(const onerf_instance_maps& m) {
  return onerf_aligned4(m.rgb) && onerf_aligned4(m.depth) && onerf_aligned4(m.opacity) &&
         onerf_aligned4(m.opacity_instance) && onerf_aligned4(m.depth_instance) && onerf_aligned4(m.rgb_instance);
}

static bool any_instance_map(const onerf_instance_maps& m) {
  return m.rgb || m.depth || m.opacity || m.opacity_instance || m.depth_instance || m.rgb_instance;
}

// One pass of one chunk of n rays (rows r0.. of the tile's maps) on depths z (n,S).  Only what the pass's maps need runs:
// the object branch (per-code ray constants, field, object compositing) when the pass has an object map, the scene
// branch (field and compositing, weights to w_out) when it has a scene map or its weights feed the fine samples
// (feeds_fine).  Neither changes the other's bits.
static int instances_pass(onerf_ctx* ctx, const onerf_instances_args* a, const InstancesWs& w, const float* rays, int n,
                          const void* packed, const float* z, int S, float* w_out, const onerf_instance_maps& m,
                          bool feeds_fine, int64_t r0, cudaStream_t stream) {
  const onerf_render_args& ra = a->render;
  const int K = a->n_ids;
  const bool want_obj = m.opacity_instance || m.depth_instance || m.rgb_instance;
  const bool want_scene = feeds_fine || m.rgb || m.depth || m.opacity;
  if (!want_obj && !want_scene) return ONERF_OK;
  FieldParams base = onerf_field_params(ra.grid, packed);
  base.rays = rays; base.z = z; base.z_stride = S;
  base.n_rays = n; base.S = S;
  base.out_stride = S;
  base.scene_out = w.scene;
  int rc;
  // code k's per-ray constants (the direction terms are the same in every block); the scene alone needs block 0's
  for (int k = 0; k < (want_obj ? K : 1); ++k) {
    FieldParams p = base;
    p.want_object = want_obj ? 1 : 0;
    p.code_row = a->code_table + (size_t)a->ids_host[k] * ONERF_NCODE;
    p.ray_const = w.ray_const + k * w.rc_stride;
    rc = onerf_launch_ray_const(ctx, p, stream);
    if (rc != ONERF_OK) return rc;
  }
  if (ra.precision == ONERF_PREC_BF16) {
    FieldParams p = base;
    p.want_scene = want_scene ? 1 : 0; p.want_object = want_obj ? 1 : 0;
    p.obj_out = want_obj ? w.obj : nullptr;
    p.ray_const = w.ray_const;
    rc = want_obj ? onerf_launch_field_bf16_codes(ctx, p, K, w.rc_stride, w.obj_stride, stream)
                  : onerf_launch_field_bf16(ctx, p, stream);
    if (rc != ONERF_OK) return rc;
  } else {   // ONERF_PREC_FP32: the FFMA field once for the scene, once per code for the object branch
    FieldParams p = base;
    if (want_scene) {
      p.want_scene = 1;
      p.ray_const = w.ray_const;
      rc = onerf_launch_field_fp32(ctx, p, stream);
      if (rc != ONERF_OK) return rc;
    }
    for (int k = 0; k < (want_obj ? K : 0); ++k) {
      p = base;
      p.want_object = 1;
      p.ray_const = w.ray_const + k * w.rc_stride;
      p.obj_out = w.obj + k * w.obj_stride;
      rc = onerf_launch_field_fp32(ctx, p, stream);
      if (rc != ONERF_OK) return rc;
    }
  }
  if (want_scene) {
    onerf_composite_args c;
    memset(&c, 0, sizeof(c));
    c.z = z; c.scene = w.scene; c.obj = nullptr;
    c.n_rays = n; c.n_samples = S;
    c.white_back = ra.white_back; c.is_eval = 1; c.zero_last_delta = ra.zero_last_delta;
    c.weights = w_out;
    c.opacity = rows_or(m.opacity, r0, 1, w.scratch.opacity);
    c.rgb = rows_or(m.rgb, r0, 3, w.scratch.rgb);
    c.depth = rows_or(m.depth, r0, 1, w.scratch.depth);
    rc = onerf_launch_composite(ctx, &c, nullptr, stream);
    if (rc != ONERF_OK) return rc;
  }
  return onerf_launch_composite_instances(ctx, z, w.obj, w.obj_stride, n, S, K,
                                          rows_or(m.opacity_instance, r0, K, nullptr),
                                          rows_or(m.depth_instance, r0, K, nullptr),
                                          rows_or(m.rgb_instance, r0, K * 3, nullptr), stream);
}

extern "C" int onerf_render_instances(onerf_ctx* ctx, const onerf_instances_args* a, void* stream_) {
  ONERF_CHECK_ARG(ctx && a, "null argument");
  const onerf_render_args& ra = a->render;
  const int64_t n_tile = a->ray_end - a->ray_begin;
  ONERF_CHECK_ARG(a->n_ids >= 1 && a->n_ids <= ONERF_INSTANCES_MAX_CODES, "n_ids outside [1, 64]");
  ONERF_CHECK_ARG(a->ids_host && a->code_table, "null ids_host / code_table");
  for (int k = 0; k < a->n_ids; ++k)
    ONERF_CHECK_ARG(a->ids_host[k] >= 0 && a->ids_host[k] < a->n_codes_table, "object id outside the code table");
  ONERF_CHECK_ARG(ra.is_eval, "the object maps are those of an evaluation render: is_eval must be set");
  ONERF_UNSUPPORTED(ra.rays_in_bbox, "rays_in_bbox (the fine depths would follow each object's weights)");
  ONERF_CHECK_ARG(ra.perturb == 0.0f && ra.noise_std == 0.0f, "perturb and noise_std must be 0");
  ONERF_CHECK_ARG(!ra.train_ws, "a training workspace is refused: nothing is kept for a backward");
  ONERF_CHECK_ARG(ra.n_rays >= 0 && ra.n_samples >= 2 && ra.n_importance >= 0, "bad shape");
  ONERF_UNSUPPORTED((int64_t)ra.n_samples + ra.n_importance > 2048, "S + K > 2048");
  ONERF_CHECK_ARG(a->ray_begin >= 0 && n_tile >= 0 && a->ray_end <= ra.n_rays, "tile outside the rays");
  ONERF_CHECK_ARG(a->chunk_rays >= 1, "chunk_rays < 1");
  ONERF_CHECK_ARG(ra.rays && ra.packed_coarse, "null rays / packed_coarse");
  ONERF_CHECK_ARG(ra.n_importance == 0 || ra.packed_fine, "n_importance > 0 needs packed_fine");
  int rc = onerf_check_grid(__func__, ra.grid);
  if (rc != ONERF_OK) return rc;
  ONERF_CHECK_ARG(ra.precision == ONERF_PREC_FP32 || ra.precision == ONERF_PREC_BF16, "unknown precision");
  ONERF_CHECK_ARG(ra.n_importance > 0 || !any_instance_map(a->fine), "fine maps without a fine pass");
  ONERF_CHECK_ARG(instance_maps_aligned(a->coarse) && instance_maps_aligned(a->fine), "maps must be 4-byte aligned");
  const int chunk = a->chunk_rays;
  rc = onerf_check_workspace(__func__, ra.workspace, ra.workspace_bytes,
                             onerf_render_instances_workspace_bytes(chunk, a->n_ids, ra.n_samples, ra.n_importance),
                             ONERF_ERR_BAD_ARG);
  if (rc != ONERF_OK) return rc;
  cudaStream_t stream = (cudaStream_t)stream_;
  const InstancesWs w = instances_ws_layout(reinterpret_cast<char*>(ra.workspace), chunk, a->n_ids, ra.n_samples,
                                            ra.n_importance);
  const int S = ra.n_samples, SF = ra.n_samples + ra.n_importance;
  for (int64_t r0 = 0; r0 < n_tile; r0 += chunk) {
    const int n = (int)(n_tile - r0 < chunk ? n_tile - r0 : chunk);
    const float* rays = ra.rays + (a->ray_begin + r0) * 8;
    rc = onerf_launch_sample_coarse(ctx, rays, n, S, ra.use_disp, 0.0f, nullptr, 0, nullptr, w.z_c, stream);
    if (rc != ONERF_OK) return rc;
    rc = instances_pass(ctx, a, w, rays, n, ra.packed_coarse, w.z_c, S, w.w_c, a->coarse, ra.n_importance > 0, r0,
                        stream);
    if (rc != ONERF_OK) return rc;
    if (ra.n_importance == 0) continue;
    rc = onerf_launch_sample_pdf_merge(ctx, w.z_c, w.w_c, n, S, ra.n_importance, 1, nullptr, 0, nullptr, w.z_f, stream);
    if (rc != ONERF_OK) return rc;
    rc = instances_pass(ctx, a, w, rays, n, ra.packed_fine, w.z_f, SF, w.w_f, a->fine, false, r0, stream);
    if (rc != ONERF_OK) return rc;
  }
  return ONERF_OK;
}
