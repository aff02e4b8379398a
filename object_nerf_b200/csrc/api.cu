// C-ABI plumbing: context, errors, and the field entry point's argument validation / dispatch.
#include <stdarg.h>
#include <string.h>

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
  if (a->grid)
    ONERF_CHECK_ARG(a->grid->table && a->grid->idx_map && a->grid->voxel_offset && a->grid->voxel_size &&
                        a->grid->voxel_shape && onerf_aligned16(a->grid->table),
                    "null / misaligned grid buffer");
  if (a->n_rays == 0) return ONERF_OK;
  cudaStream_t stream = (cudaStream_t)stream_;
  FieldParams p;
  memset(&p, 0, sizeof(p));
  p.rays = a->rays; p.xyz = a->xyz; p.z = a->z; p.z_stride = a->z_stride;
  p.codes = a->codes; p.code_row = a->code_row;
  p.n_rays = a->n_rays; p.S = a->n_samples;
  if (a->grid) p.grid = *a->grid;
  p.packed = a->packed;
  p.L = onerf_make_layout(a->grid ? 1 : 0);
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
    ONERF_UNSUPPORTED(a->z_stride != a->n_samples || a->out_stride != a->n_samples || a->xyz, "training dump needs dense z / outputs and no explicit xyz");
    ONERF_UNSUPPORTED(a->mute_zero_rays || a->n_boxes > 0, "editing extras have no backward");
    ONERF_CHECK_ARG((reinterpret_cast<uintptr_t>(a->train_ws) & 1023u) == 0, "train_ws must be 1024-byte aligned");
    p.train_ws = a->train_ws;
  }
  int rc = onerf_launch_ray_const(ctx, p, stream);
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
static size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

extern "C" size_t onerf_render_rays_workspace_bytes(int n_rays, int n_samples, int n_importance) {
  if (n_rays < 0 || n_samples < 1 || n_importance < 0) return 0;
  const size_t s_max = (size_t)n_samples + (size_t)n_importance;
  return align256((size_t)n_rays * ONERF_RAY_CONST_FLOATS * sizeof(float)) +   // per-ray hoisted terms
         2 * align256((size_t)n_rays * s_max * 4 * sizeof(float));             // (rgb, sigma) of both branches
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
  ONERF_CHECK_ARG(!a->forward_instance || a->codes, "forward_instance needs codes");
  ONERF_CHECK_ARG(a->n_importance == 0 || a->packed_fine, "n_importance > 0 needs packed_fine");
  ONERF_CHECK_ARG(maps_ok(a->coarse, a->forward_instance), "null coarse output map");
  ONERF_CHECK_ARG(a->n_importance == 0 || maps_ok(a->fine, a->forward_instance), "null fine output map");
  const size_t need = onerf_render_rays_workspace_bytes(a->n_rays, a->n_samples, a->n_importance);
  ONERF_CHECK_ARG(a->workspace && (reinterpret_cast<uintptr_t>(a->workspace) & 255u) == 0, "workspace null or not 256-byte aligned");
  if (a->workspace_bytes < need) {
    onerf_set_error("onerf_render_rays_fwd: workspace too small (%zu < %zu)", a->workspace_bytes, need);
    return ONERF_ERR_WORKSPACE;
  }
  if (a->n_rays == 0) return ONERF_OK;
  const int S = a->n_samples, SF = a->n_samples + a->n_importance;
  char* ws = reinterpret_cast<char*>(a->workspace);
  float* ray_const = reinterpret_cast<float*>(ws);
  ws += align256((size_t)a->n_rays * ONERF_RAY_CONST_FLOATS * sizeof(float));
  float* scene = reinterpret_cast<float*>(ws);
  ws += align256((size_t)a->n_rays * SF * 4 * sizeof(float));
  float* obj = reinterpret_cast<float*>(ws);
  // training: both passes' fields are kept in the training workspace, and with bf16 the backward operands too (the fp32
  // backward re-runs the FFMA forward chunk by chunk instead)
  float *scene_c = scene, *obj_c = obj, *scene_f = scene, *obj_f = obj;
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
  if (step) {
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
  int rc = onerf_launch_sample_coarse(ctx, a->rays, a->n_rays, S, a->use_disp, a->perturb, a->jitter, seed, seed_dev,
                                      a->coarse.z_vals, stream);
  if (rc != ONERF_OK) return rc;
  rc = render_pass(ctx, a, a->packed_coarse, a->coarse.z_vals, S, a->coarse, a->noise_scene_coarse, a->noise_obj_coarse,
                   seed + 1, ray_const, scene_c, obj_c, tl_c, step ? &step_c : nullptr, seed_dev, stream);
  if (rc != ONERF_OK || a->n_importance == 0) return rc;
  rc = onerf_launch_sample_pdf_merge(ctx, a->coarse.z_vals, a->coarse.weights, a->n_rays, S, a->n_importance,
                                     a->perturb == 0.0f ? 1 : 0, a->u, seed + 2, seed_dev, a->fine.z_vals, stream);
  if (rc != ONERF_OK) return rc;
  return render_pass(ctx, a, a->packed_fine, a->fine.z_vals, SF, a->fine, a->noise_scene_fine, a->noise_obj_fine, seed + 3,
                     ray_const, scene_f, obj_f, tl_f, step ? &step_f : nullptr, seed_dev, stream);
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
  size_t off = 0;
  auto take = [&](size_t bytes) { void* p = base + off; off += align256(bytes); return p; };
  w.ray_const = (float*)take(n * ONERF_RAY_CONST_FLOATS * sizeof(float));   // per-ray hoisted terms (one set at a time)
  w.z_all = (float*)take(no * n * n_samples * sizeof(float));               // coarse depths of every set
  w.z_fine = (float*)take(no * n * sf * sizeof(float));                     // fine depths
  w.field_all = (float*)take(no * n * sf * 4 * sizeof(float));              // fields (rgb, sigma) of every set
  w.w_unsorted = (float*)take(no * n * n_samples * sizeof(float));          // per-set coarse weights in sample order
  w.live = (int*)take(n * sizeof(int));
  w.slot = (int*)take(n * sizeof(int));
  w.count = (int*)take(sizeof(int));
  w.rays_c = (float*)take(n * 8 * sizeof(float));
  w.z_c = (float*)take(n * sf * sizeof(float));
  w.field_c = (float*)take(n * sf * 4 * sizeof(float));
  w.sort_bytes = onerf_composite_multi_workspace_bytes(n_rays, n_obj, (int)sf);
  w.sort = take(w.sort_bytes);
  w.total = off;
  return w;
}

extern "C" size_t onerf_render_multi_workspace_bytes(int n_rays, int n_obj, int n_samples, int n_importance) {
  if (n_rays < 0 || n_obj < 1 || n_samples < 1 || n_importance < 0) return 0;
  return multi_ws_layout(nullptr, n_rays, n_obj, n_samples, n_importance).total;
}

static int multi_fields(onerf_ctx* ctx, const onerf_render_multi_args* a, const void* packed, const float* z_all, int S,
                        const MultiWs& w, void* stream) {
  const int N = a->n_rays;
  for (int i = 0; i < a->n_obj; ++i) {
    const int id = a->obj_ids_host[i];
    const float* z = z_all + (size_t)i * N * S;
    float* out = w.field_all + (size_t)i * N * S * 4;
    onerf_field_args f;
    memset(&f, 0, sizeof(f));
    f.rays = a->rays_list_host[i];
    f.z = z;
    f.z_stride = S;
    f.code_row = id > 0 ? a->code_table + (size_t)id * ONERF_NCODE : nullptr;
    f.n_rays = N; f.n_samples = S;
    f.grid = a->grid; f.packed = packed;
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

extern "C" int onerf_render_multi_fwd(onerf_ctx* ctx, const onerf_render_multi_args* a, void* stream) {
  ONERF_CHECK_ARG(ctx && a, "null argument");
  ONERF_CHECK_ARG(a->rays_list_host && a->obj_ids_host && a->packed_coarse && a->grid && a->code_table, "null input");
  ONERF_CHECK_ARG(a->n_rays >= 0 && a->n_obj >= 1 && a->n_samples >= 2 && a->n_importance >= 0, "bad shape");
  ONERF_UNSUPPORTED((int64_t)a->n_obj * (a->n_samples + a->n_importance) > INT32_MAX, "n_obj * samples >= 2^31");
  ONERF_UNSUPPORTED(a->n_samples + a->n_importance > 2048, "more than 2048 samples per ray set");
  ONERF_CHECK_ARG(a->n_importance == 0 || a->packed_fine, "n_importance > 0 needs packed_fine");
  ONERF_CHECK_ARG(a->n_boxes == 0 || a->boxes, "n_boxes > 0 with null boxes");
  for (int i = 0; i < a->n_obj; ++i) {
    ONERF_CHECK_ARG(a->rays_list_host[i], "null ray set");
    ONERF_CHECK_ARG(a->obj_ids_host[i] >= 0 && a->obj_ids_host[i] < a->n_codes, "object id outside the code table");
  }
  const onerf_render_multi_maps& c = a->coarse;
  ONERF_CHECK_ARG(c.weights && c.opacity && c.z_vals && c.rgb && c.depth && c.obj_ids, "null coarse output");
  if (a->n_importance > 0)
    ONERF_CHECK_ARG(a->fine.weights && a->fine.opacity && a->fine.z_vals && a->fine.rgb && a->fine.depth, "null fine output");
  const size_t need = onerf_render_multi_workspace_bytes(a->n_rays, a->n_obj, a->n_samples, a->n_importance);
  ONERF_CHECK_ARG(a->workspace && (reinterpret_cast<uintptr_t>(a->workspace) & 255u) == 0, "workspace null or not 256-byte aligned");
  if (a->workspace_bytes < need) {
    onerf_set_error("onerf_render_multi_fwd: workspace too small (%zu < %zu)", a->workspace_bytes, need);
    return ONERF_ERR_WORKSPACE;
  }
  if (a->n_rays == 0) return ONERF_OK;
  const int S = a->n_samples, SF = a->n_samples + a->n_importance, N = a->n_rays, NO = a->n_obj;
  const MultiWs w = multi_ws_layout(reinterpret_cast<char*>(a->workspace), N, NO, S, a->n_importance);
  int rc;
  for (int i = 0; i < NO; ++i) {   // multi_rendering.py:196-213: coarse depths are never jittered on this path
    rc = onerf_sample_coarse(ctx, a->rays_list_host[i], N, S, a->use_disp, 0.0f, nullptr, 0, w.z_all + (size_t)i * N * S, stream);
    if (rc != ONERF_OK) return rc;
  }
  rc = multi_fields(ctx, a, a->packed_coarse, w.z_all, S, w, stream);
  if (rc != ONERF_OK) return rc;
  rc = onerf_composite_multi_ws(ctx, w.z_all, w.field_all, N, NO, S, a->white_back, c.z_vals, c.weights, c.obj_ids,
                                a->n_importance > 0 ? w.w_unsorted : nullptr, c.opacity, c.rgb, c.depth, w.sort, w.sort_bytes,
                                stream);
  if (rc != ONERF_OK || a->n_importance == 0) return rc;
  const int det = a->perturb == 0.0f ? 1 : 0;
  for (int i = 0; i < NO; ++i) {
    rc = onerf_sample_pdf_merge(ctx, w.z_all + (size_t)i * N * S, w.w_unsorted + (size_t)i * N * S, N, S, a->n_importance, det,
                                nullptr, det ? 0 : a->seed + (uint64_t)i, w.z_fine + (size_t)i * N * SF, stream);
    if (rc != ONERF_OK) return rc;
  }
  rc = multi_fields(ctx, a, a->packed_fine, w.z_fine, SF, w, stream);
  if (rc != ONERF_OK) return rc;
  return onerf_composite_multi_ws(ctx, w.z_fine, w.field_all, N, NO, SF, a->white_back, a->fine.z_vals, a->fine.weights, nullptr,
                                  nullptr, a->fine.opacity, a->fine.rgb, a->fine.depth, w.sort, w.sort_bytes, stream);
}
