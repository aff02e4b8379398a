/*
 * onerf.h — C ABI of libonerf_sm90.so: the H100-native (sm_90a) per-ray render path of
 * zju3dv/object_nerf (stratified + PDF sampling, positional / sparse-voxel encoding, the two-branch
 * scene+object MLP, sigma->alpha front-to-back compositing, single-scene and multi-object variants).
 *
 * The reference has no FFI layer: its boundary is three Python functions (SURVEY.md §8b).  This header
 * is what a binding for that boundary calls; `object_nerf_b200/_lib.py` is the ctypes binding and
 * INTEGRATION.md shows the reference-side stub.  Each entry point cites the reference code it replaces
 * (paths relative to the reference root).
 *
 * Conventions
 *  - every pointer is a DEVICE pointer on the ctx's device unless the parameter name ends in `_host`;
 *    the caller owns all buffers (inputs, outputs, workspace); fp32 row-major contiguous, 16-byte aligned;
 *  - `stream` is a cudaStream_t passed as void*; all work is enqueued on it, nothing synchronises;
 *  - every function returns 0 on success or a negative onerf_status; onerf_last_error() gives the
 *    thread-local message.  Unsupported configurations are hard errors: there is no CPU fallback.
 */
#ifndef ONERF_H_
#define ONERF_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ONERF_ABI_VERSION 2

typedef enum onerf_status {
  ONERF_OK = 0,
  ONERF_ERR_BAD_ARG = -1,      /* null pointer / bad shape / misaligned buffer */
  ONERF_ERR_UNSUPPORTED = -2,  /* configuration the kernels are not built for */
  ONERF_ERR_CUDA = -3,         /* a CUDA runtime call failed */
  ONERF_ERR_WORKSPACE = -4     /* caller-provided workspace too small */
} onerf_status;

/* arithmetic of the fused encode+MLP ("field") kernel */
typedef enum onerf_precision {
  ONERF_PREC_FP32 = 0, /* FFMA, fp32 throughout: verification / gradient-check mode */
  ONERF_PREC_BF16 = 1  /* wgmma tensor cores: bf16 operands, fp32 accumulate in registers (product default) */
} onerf_precision;

typedef struct onerf_ctx onerf_ctx;

int onerf_abi_version(void);
const char* onerf_last_error(void);
int onerf_ctx_create(int device, onerf_ctx** out);
int onerf_ctx_destroy(onerf_ctx* ctx);
/* number of kernels this ctx has launched since creation (bench.py's gpu_launches claim) */
int64_t onerf_ctx_launch_count(const onerf_ctx* ctx);

/* ---------------------------------------------------------------------------------------------
 * Model weights.  One ObjectNeRF (models/nerf_model.py:18-95) = 20 nn.Linear layers, passed in this
 * fixed order (W is [out,in] row-major fp32 exactly as nn.Linear stores it, b is [out]):
 *   0..7  scene  xyz_encoding_1..8     8 scene.sigma   9 scene xyz_encoding_final
 *   10    scene dir_encoding          11 scene rgb
 *   12..15 object instance_encoding_1..4  16 instance_sigma  17 instance_encoding_final
 *   18    inst_dir_encoding           19 inst_rgb
 * Only the default architecture is built: D=8, W=256, skips=[4], inst_D=4, inst_W=128, inst_skips=[2],
 * PE 10/4/6, 16+8 voxel channels, 64-long codes (config/default_conf.yml:7-36); use_voxel selects the
 * 271/439-wide (voxel) or 63/127-wide (plain PE) inputs.  Anything else -> ONERF_ERR_UNSUPPORTED.
 * ------------------------------------------------------------------------------------------- */
#define ONERF_N_LINEAR 20

size_t onerf_packed_weights_bytes(int use_voxel);
/* Re-lay the 20 (W,b) pairs into the kernels' formats (fp32 K-major for the FFMA path; bf16, K-major,
 * swizzled stage images in program order for the tensor-core path).  Re-run whenever parameters change. */
int onerf_pack_weights(onerf_ctx* ctx, int use_voxel, const float* const* W_host_ptrs,
                       const float* const* b_host_ptrs, void* packed, size_t packed_bytes, void* stream);

/* Sparse voxel grid: the buffers of EmbeddingVoxel the per-ray path reads
 * (models/embedding_helper.py:107-133,189-200).  Metadata stays in device memory (the reference mutates
 * it at epoch boundaries, :202-302) and is read by the kernels on every call. */
typedef struct onerf_grid {
  const float* table;         /* embedding_space_ftr.weight (n_rows, 24) */
  const int64_t* idx_map;     /* voxel_idx_map (X,Y,Z) int64, -1 = empty */
  const float* voxel_offset;  /* (3,) */
  const float* voxel_size;    /* scalar */
  const int64_t* voxel_shape; /* (3,) */
} onerf_grid;

/* ---------------------------------------------------------------------------------------------
 * Stage entry points (each is also a step of onerf_render_rays_fwd)
 * ------------------------------------------------------------------------------------------- */

/* Stratified depths, models/rendering.py:259-277.  rays (N,8) = [o, d, near, far]; z_out (N,S).
 * perturb > 0: jitter (N,S) U[0,1) is used if non-null, else drawn from Philox(seed). */
int onerf_sample_coarse(onerf_ctx* ctx, const float* rays, int n_rays, int n_samples, int use_disp,
                        float perturb, const float* jitter, uint64_t seed, float* z_out, void* stream);

/* Inverse-CDF importance sampling + sorted merge with the coarse depths,
 * models/rendering.py:11-61 and :301-313.  weights (N,S) are the full coarse weights (the [1:-1] slice
 * and the mid-point bins are formed inside).  det != 0: u = linspace(0,1,K); else u (N,K) if non-null,
 * else Philox(seed).  z_out (N, S+K) ascending. */
int onerf_sample_pdf_merge(onerf_ctx* ctx, const float* z_coarse, const float* weights, int n_rays,
                           int n_samples, int n_importance, int det, const float* u, uint64_t seed,
                           float* z_out, void* stream);

/* Stand-alone sample_pdf on explicit bins (N, n_bins) and weights (N, n_bins-1), the reference's exported
 * helper models/rendering.py:11-61; out (N, K) in draw order (no merge). */
int onerf_sample_pdf(onerf_ctx* ctx, const float* bins, const float* weights, int n_rays, int n_bins,
                     int n_importance, int det, const float* u, uint64_t seed, float* out, void* stream);

/* Encoding only (test / ncu entry): xyz (B,3) -> scene_in (B,271|63), obj_in (B,104) (null for plain
 * PE).  models/embedding_helper.py:57-74, :325-411.  grid == NULL selects plain PE(10); a grid's table
 * must be 16-byte aligned (rows are read as float4). */
int onerf_encode(onerf_ctx* ctx, const onerf_grid* grid, const float* xyz, int64_t n_points,
                 float* scene_in, float* obj_in, void* stream);

/* Raw trilinear voxel features (no positional encoding), models/embedding_helper.py:354-411 with
 * positional_embedding=False: xyz (B,3) -> out (B,24).  Used by the grid refinement (voxel_subdivision, :250-252). */
int onerf_voxel_features(onerf_ctx* ctx, const onerf_grid* grid, const float* xyz, int64_t n_points, float* out, void* stream);

/* Fused encode + two-branch MLP over all samples of a ray set,
 * models/rendering.py:85-137 (+ models/nerf_model.py:97-152, models/embedding_helper.py:325-411),
 * and render_tools/multi_rendering.py:16-93 for the one-branch-per-object editing variant. */
typedef struct onerf_field_args {
  const float* rays;       /* (N,8) */
  const float* xyz;        /* optional explicit sample positions (N,S,3) (the inference_model() call
                              surface, models/rendering.py:64-83); NULL -> o + d * z from rays */
  const float* z;          /* sample depths: sample i of ray r at z[r * z_stride + i] */
  int64_t z_stride;        /* >= S (S for a dense (N,S) array; n_obj*S inside a concatenated one) */
  const float* codes;      /* (N,64) per-ray object codes (code_library lookup done by the caller,
                              models/code_library.py:18-28), or NULL */
  const float* code_row;   /* (64,) one code for every ray (editing path), used when codes == NULL */
  int n_rays, n_samples;
  const onerf_grid* grid;  /* NULL -> plain PE model */
  const void* packed;      /* onerf_pack_weights output */
  int want_scene, want_object;
  int precision;           /* onerf_precision */
  /* editing extras (render_tools/multi_rendering.py:40,83,92 and :239-241) */
  int mute_zero_rays;      /* rays with z[:, -1] == 0 get sigma = -1e5 */
  const float* boxes;      /* (n_boxes, 18): A row-major (9), t (3), lo (3), hi (3); scene samples with
                              lo <= A p + t <= hi get sigma = -1e5 (utils/bbox_utils.py:119-130,158-207) */
  int n_boxes;
  float* scene_out;        /* float4 (rgb, sigma) of sample i of ray r at [r * out_stride + i]; iff want_scene */
  float* obj_out;          /* same for the object branch; iff want_object */
  int64_t out_stride;      /* >= S, in samples */
  float* ray_const;        /* workspace, n_rays * ONERF_RAY_CONST_FLOATS floats */
  /* backward support (ONERF_PREC_FP32 only): if non-NULL, 17 row-major [n_rays*S x width] matrices receiving the
   * activations of the forward: [0] X (384 voxel / 64 plain), [1..8] scene hidden 1..8 (256), [9] scene final (256),
   * [10] scene dir (128), [11..14] object hidden 1..4 (128), [15] object final (128), [16] object dir (64). */
  float* const* activations;
  /* training forward (ONERF_PREC_BF16, either model, dense z / outputs): if non-NULL, a workspace of
   * onerf_field_train_bytes(grid != NULL, n_rays * n_samples) bytes receiving what the tensor-core backward needs: every layer's
   * output activations and the encoded input as bf16 tiles in the tensor cores' operand layout, and 1-bit LeakyReLU
   * masks (object_nerf_b200/csrc/layout.h: TrainLayout). */
  void* train_ws;
} onerf_field_args;
size_t onerf_field_train_bytes(int use_voxel, int64_t n_samples);
#define ONERF_RAY_CONST_FLOATS 448

int onerf_field_fwd(onerf_ctx* ctx, const onerf_field_args* args, void* stream);

/* sigma->alpha->weights and front-to-back compositing of both branches, models/rendering.py:139-229. */
typedef struct onerf_composite_args {
  const float* z;          /* (N,S) */
  const float* scene;      /* (N,S,4) rgb,sigma */
  const float* obj;        /* (N,S,4) or NULL (forward_instance == False) */
  int n_rays, n_samples;
  float noise_std;
  const float* noise_scene; /* (N,S) N(0,1) or NULL -> Philox(seed) when noise_std > 0 */
  const float* noise_obj;
  uint64_t seed;
  int white_back, is_eval, zero_last_delta, rays_in_bbox;
  float frustum_bound_th;
  const uint8_t* pass_through_mask; /* (N,) or NULL */
  float* weights;          /* (N,S)  (object weights if rays_in_bbox) */
  float* opacity;          /* (N,) */
  float* rgb;              /* (N,3) */
  float* depth;            /* (N,) */
  float* rgb_instance;     /* (N,3)  } */
  float* depth_instance;   /* (N,)   } written iff obj != NULL */
  float* opacity_instance; /* (N,)   } */
} onerf_composite_args;

int onerf_composite(onerf_ctx* ctx, const onerf_composite_args* args, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Whole forward of render_rays() in ONE call, models/rendering.py:233-337 (inference / validation: no autograd):
 * stratified sampling -> coarse field + compositing -> importance resampling + merge -> fine field + compositing.
 * It only enqueues the stage kernels above on `stream` (no host reads of device data, no allocation): the call is
 * CUDA-graph capturable.  This is the function a non-Python host binds instead of models.rendering.render_rays.
 * ------------------------------------------------------------------------------------------- */
typedef struct onerf_render_maps {   /* the reference's result dict for one pass ("coarse" / "fine"); all required */
  float* weights;          /* (N,S) */
  float* opacity;          /* (N,) */
  float* z_vals;           /* (N,S): coarse = stratified depths, fine = merged sorted depths (S = n_samples + n_importance) */
  float* rgb;              /* (N,3) */
  float* depth;            /* (N,) */
  float* rgb_instance;     /* (N,3)  } */
  float* depth_instance;   /* (N,)   } required iff forward_instance */
  float* opacity_instance; /* (N,)   } */
} onerf_render_maps;

typedef struct onerf_render_args {
  const float* rays;            /* (N,8) = [o, d, near, far] */
  const float* codes;           /* (N,64) object codes (embedding_instance), required iff forward_instance */
  int n_rays, n_samples, n_importance;
  const onerf_grid* grid;       /* NULL -> plain PE model */
  const void* packed_coarse;    /* onerf_pack_weights of models["coarse"] */
  const void* packed_fine;      /* ... of models["fine"]; required iff n_importance > 0 */
  int precision;                /* onerf_precision */
  int use_disp;
  float perturb, noise_std;
  uint64_t seed;                /* Philox seed of whatever random input is not given explicitly below */
  const float* jitter;          /* (N, n_samples) U[0,1) or NULL */
  const float* u;               /* (N, n_importance) U[0,1) or NULL (perturb == 0 -> deterministic linspace) */
  const float* noise_scene_coarse, *noise_obj_coarse, *noise_scene_fine, *noise_obj_fine; /* (N,S) N(0,1) or NULL */
  int white_back, forward_instance, is_eval, zero_last_delta, rays_in_bbox;
  float frustum_bound_th;
  const uint8_t* pass_through_mask; /* (N,) or NULL */
  onerf_render_maps coarse;
  onerf_render_maps fine;       /* written iff n_importance > 0 */
  void* workspace;              /* >= onerf_render_rays_workspace_bytes(...) bytes, 256-byte aligned */
  size_t workspace_bytes;
  /* training: if non-NULL (either model, either precision), >= onerf_train_workspace_bytes_prec(precision, grid != NULL,
   * ...) bytes (include/onerf_ext.h; onerf_train_workspace_bytes for ONERF_PREC_BF16), 1024-byte aligned; the forward
   * then keeps both passes' per-sample fields there for onerf_render_rays_bwd, and with ONERF_PREC_BF16 also every
   * layer's operands (the fp32 backward re-runs the FFMA forward instead). */
  void* train_ws;
  size_t train_ws_bytes;
} onerf_render_args;

size_t onerf_render_rays_workspace_bytes(int n_rays, int n_samples, int n_importance);
int onerf_render_rays_fwd(onerf_ctx* ctx, const onerf_render_args* args, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Whole forward of render_rays_multi() in ONE call, render_tools/multi_rendering.py:160-325 (the editing path of
 * EditableRenderer.scene_inference / render_edit, editable_renderer.py:125-140, 272-287; inference only, as in the
 * reference).  Ray set k is rendered with the scene branch if obj_ids[k] == 0 (removed-object boxes applied on the device)
 * or with the object branch and code_table[obj_ids[k]] otherwise; the sets are composited jointly (stable depth sort).
 * `_host` arrays are read on the host at call time.  Only enqueues kernels on `stream`: CUDA-graph capturable.
 * ------------------------------------------------------------------------------------------- */
typedef struct onerf_render_multi_maps {   /* result dict of one pass, T = n_obj * samples of the pass */
  float* weights;          /* (N,T) in jointly sorted order */
  float* opacity;          /* (N,) */
  float* z_vals;           /* (N,T) sorted depths */
  float* rgb;              /* (N,3) */
  float* depth;            /* (N,) */
  float* obj_ids;          /* (N,T) list position of each sorted sample ("obj_ids_coarse"); coarse pass only */
} onerf_render_multi_maps;

typedef struct onerf_render_multi_args {
  const float* const* rays_list_host; /* n_obj DEVICE pointers to (N,8) ray sets, the array itself in host memory */
  const int* obj_ids_host;            /* n_obj instance ids (host) */
  int n_obj, n_rays, n_samples, n_importance;
  const onerf_grid* grid;             /* required (the reference's editing path assumes the voxel embedding) */
  const void* packed_coarse;
  const void* packed_fine;            /* required iff n_importance > 0 */
  const float* code_table;            /* (n_codes,64) CodeLibrary.embedding_instance.weight */
  int n_codes;
  int precision;                      /* onerf_precision */
  int use_disp;
  float perturb;                      /* 0: deterministic importance samples (what EditableRenderer passes) */
  uint64_t seed;
  int white_back;
  const float* boxes;                 /* (n_boxes,18) removed-object boxes (see onerf_field_args), or NULL */
  int n_boxes;
  onerf_render_multi_maps coarse;
  onerf_render_multi_maps fine;       /* written iff n_importance > 0 */
  void* workspace;                    /* >= onerf_render_multi_workspace_bytes(...) bytes, 256-byte aligned */
  size_t workspace_bytes;
} onerf_render_multi_args;

size_t onerf_render_multi_workspace_bytes(int n_rays, int n_obj, int n_samples, int n_importance);
int onerf_render_multi_fwd(onerf_ctx* ctx, const onerf_render_multi_args* args, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Rays: the two host steps directly in front of the path (SURVEY.md section 8f rows 1-2), on the device.
 * `_host` pointers are read on the host at call time (a 3x4 pose, one box), everything else is device memory.
 * ------------------------------------------------------------------------------------------- */

/* get_ray_directions, datasets/ray_utils.py:5-25: directions (H,W,3), pixel (row y, column x) ->
 * ((x - W/2) / focal, -(y - H/2) / focal, -1); no +0.5 pixel centring. */
int onerf_ray_directions(onerf_ctx* ctx, int H, int W, float focal, float* directions, void* stream);

/* get_rays, datasets/ray_utils.py:28-51: rays_d = normalise(directions @ c2w[:, :3]^T), rays_o = c2w[:, 3];
 * directions (n,3), c2w_host 12 floats row-major (3,4), outputs (n,3). */
int onerf_get_rays(onerf_ctx* ctx, const float* directions, int64_t n, const float* c2w_host, float* rays_o, float* rays_d,
                   void* stream);

/* One object's box as BBoxRayHelper holds it (utils/bbox_utils.py): pose_avg and axis_align_mat as row-major 4x4
 * (or 3x4: only the first 12 entries are read), bounds = [lo(3), hi(3)] with any bbox_enlarge already applied
 * (utils/bbox_utils.py:140-145). */
typedef struct onerf_box_host {
  double pose_avg[16];
  double axis_align[16];
  double bounds[6];
} onerf_box_host;

/* generate_rays, render_tools/editable_renderer.py:153-181: (n,8) rays = [o, d, near, far] of one object.
 * box == NULL (obj_id 0): near / far = the constants near / scale_factor, far / scale_factor.  Otherwise the ray is
 * taken to the box frame (utils/bbox_utils.py:102-117: fp32 unscale, float64 rigid transforms, direction rotated by the
 * axis-alignment matrix only) and slab-tested in float64 (datasets/geo_utils.py:126-162: zero direction components
 * -> 1e-14, origin inside the box -> miss); near / far = hit distances / scale_factor, 0 / 0 for a miss.
 * hit_out (n,) u8 or NULL = the bbox mask. */
int onerf_generate_rays(onerf_ctx* ctx, const float* rays_o, const float* rays_d, int64_t n, const onerf_box_host* box_host,
                        double scale_factor, double near, double far, float* rays_out, uint8_t* hit_out, void* stream);

/* The three steps fused: pixel grid + pose (+ box) -> (H*W,8) rays in one kernel; the renderer then needs only
 * (H, W, focal, pose) per object instead of host-built ray tensors. */
int onerf_camera_rays(onerf_ctx* ctx, int H, int W, float focal, const float* c2w_host, const onerf_box_host* box_host,
                      double scale_factor, double near, double far, float* rays_out, uint8_t* hit_out, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Training loss (SURVEY.md section 8f row 3): TotalLoss, models/losses.py:5-135, and d(loss_sum)/d(map) for the ten
 * rendered maps, without host synchronisation.  Five masked-MSE terms, each summed over the coarse (and fine) maps:
 *   color           mean over valid rays x 3 of (rgb - rgbs)^2
 *   depth           mean over valid & depths > 0 of (depth - depths)^2;  skipped if no depths > 0 at all
 *   opacity         mean over valid of (clamp(opacity_instance, 0, 1) - instance_mask)^2 * instance_mask_weight
 *   instance color  mean over valid & instance_mask (x 3) of (rgb_instance - rgbs)^2 * weight;  skipped if empty
 *   instance depth  mean over valid & depths > 0 & instance_mask of (depth_instance - depths)^2 * weight;  skipped if empty
 * loss_sum = sum of weight_t * term_t over the terms present.
 * ------------------------------------------------------------------------------------------- */
typedef struct onerf_loss_maps {      /* maps of one pass, or their gradients (same shapes) */
  const float* rgb;                   /* (N,3) */
  const float* depth;                 /* (N,) */
  const float* opacity_instance;      /* (N,) */
  const float* rgb_instance;          /* (N,3) */
  const float* depth_instance;        /* (N,) */
} onerf_loss_maps;

typedef struct onerf_loss_args {
  int64_t n_rays;
  int has_fine;
  onerf_loss_maps coarse, fine;            /* inputs */
  const float* rgbs;                       /* (N,3) batch["rgbs"] */
  const float* depths;                     /* (N,)  batch["depths"] */
  const uint8_t* valid_mask;               /* (N,)  batch["valid_mask"] */
  const uint8_t* instance_mask;            /* (N,)  batch["instance_mask"] */
  const float* instance_mask_weight;       /* (N,)  batch["instance_mask_weight"] */
  float color_weight, depth_weight, opacity_weight, instance_color_weight, instance_depth_weight; /* config loss.*_weight */
  onerf_loss_maps grad_coarse, grad_fine;  /* outputs (written): d(loss_sum)/d(map) */
  float* loss_sum_out;                     /* (1,) */
  float* terms_out;                        /* (5,) unweighted terms in the order above (0 where skipped) */
  int32_t* present_out;                    /* (5,) 1 = term present, 0 = skipped (the reference returns None) */
  void* workspace;                         /* onerf_total_loss_workspace_bytes() bytes, 8-byte aligned */
} onerf_loss_args;

size_t onerf_total_loss_workspace_bytes(void);
int onerf_total_loss(onerf_ctx* ctx, const onerf_loss_args* args, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Training (SURVEY.md §8 row a14: what loss.backward() does in the reference, train.py:147-180, through
 * models/rendering.py, models/nerf_model.py:97-152, models/embedding_helper.py:354-409, models/code_library.py).
 * onerf_render_rays_fwd with train_ws set runs the forward and keeps what the backward needs;
 * onerf_render_rays_bwd turns the upstream gradients of the rendered maps into gradients of the 2 x 20 nn.Linear
 * tensors, the per-ray object codes and (voxel model) the voxel feature table, for either model (fwd->grid NULL = plain
 * PE model, whose encoding has no trainable parameters) and in the forward's precision:
 *   ONERF_PREC_BF16: compositing backward -> head gradients -> input-gradient chain (wgmma, transposed weight images,
 *   operand resident in registers) -> weight gradients (wgmma, sample-axis reduction) -> encoding gradient (wgmma +
 *   scatter-add) -> per-ray-constant columns (direction encoding, object code) -> reference [out,in] layout.
 *   ONERF_PREC_FP32 (verification arithmetic): compositing backward, then per chunk of rays the FFMA forward re-run with
 *   its activation dump and the fp32 building blocks below, layer by layer.
 * No gradient flows to rays or depths (the importance samples are detached in the reference, models/rendering.py:307).
 * ------------------------------------------------------------------------------------------- */
size_t onerf_train_workspace_bytes(int use_voxel, int n_rays, int n_samples, int n_importance);

typedef struct onerf_map_grads {   /* upstream gradients of one pass's maps; NULL = zero */
  const float* rgb;              /* (N,3) */
  const float* depth;            /* (N,) */
  const float* opacity;          /* (N,) */
  const float* rgb_instance;     /* (N,3) */
  const float* depth_instance;   /* (N,) */
  const float* opacity_instance; /* (N,) */
} onerf_map_grads;

typedef struct onerf_render_bwd_args {
  onerf_map_grads coarse, fine;
  const float* const* W_coarse;  /* the 20 reference weight tensors of models["coarse"] (onerf_pack_weights order) */
  const float* const* W_fine;    /* ... of models["fine"]; required iff n_importance > 0 */
  /* outputs, ACCUMULATED into (the caller zero-fills or keeps earlier contributions) */
  float* const* dW_coarse;       /* 20 tensors shaped like W */
  float* const* db_coarse;       /* 20 tensors shaped like b */
  float* const* dW_fine;
  float* const* db_fine;
  float* d_codes;                /* (N,64); required iff forward_instance */
  float* table_grad;             /* (n_rows,24) gradient of grid->table, or NULL; must be NULL for the plain PE model
                                    (ONERF_ERR_BAD_ARG otherwise) */
} onerf_render_bwd_args;

int onerf_render_rays_bwd(onerf_ctx* ctx, const onerf_render_args* fwd, const onerf_render_bwd_args* bwd, void* stream);

/* stages of onerf_render_rays_bwd (tests / ncu).  ws = a field training workspace (onerf_field_train_bytes);
 * dA_* (n_samples,4) = d(rgb_pre, sigma) per sample (onerf_head_bwd); grad = kernel-layout gradient buffer of
 * onerf_grad_buffer_floats() floats, mapped to the reference layout by onerf_unpack_grads. */
size_t onerf_grad_buffer_floats(int use_voxel);
int onerf_unpack_grads(onerf_ctx* ctx, int use_voxel, const float* grad, float* const* dW, float* const* db, void* stream);
int onerf_bwd_chain(onerf_ctx* ctx, int use_voxel, int want_object, const void* packed, void* ws, int64_t n_samples,
                    const float* dA_scene, const float* dA_obj, void* stream);
int onerf_bwd_wgrad(onerf_ctx* ctx, int use_voxel, int want_object, const void* ws, int64_t n_samples, float* grad, void* stream);
int onerf_bwd_colsums(onerf_ctx* ctx, int use_voxel, int want_object, const void* ws, int64_t n_samples, const float* dA_scene,
                      const float* dA_obj, float* grad, void* stream);
int onerf_bwd_raysums(onerf_ctx* ctx, int use_voxel, int want_object, const void* ws, int n_rays, int n_samples, float* out,
                      void* stream);
int onerf_bwd_dx(onerf_ctx* ctx, int want_object, const void* packed, const void* ws, const float* rays, const float* z,
                 int n_rays, int n_samples, const onerf_grid* grid, float* table_grad, void* stream);

/* CodeLibrary.forward, models/code_library.py:18-28: out (n,64) = table[ids]; and its gradient (scatter-add by id). */
int onerf_code_gather(onerf_ctx* ctx, const float* table, const int64_t* ids, int n, int n_codes, float* out, void* stream);
int onerf_code_scatter_add(onerf_ctx* ctx, const float* d_codes, const int64_t* ids, int n, int n_codes, float* table_grad,
                           void* stream);

/* ---------------------------------------------------------------------------------------------
 * fp32 backward building blocks (verification arithmetic of the training path).
 * onerf_render_rays_bwd chains them into the gradient of render_rays for ONERF_PREC_FP32.
 * ------------------------------------------------------------------------------------------- */

/* Gradient of onerf_composite w.r.t. the per-sample fields: fwd = the forward's arguments (with noise_std > 0, NULL noise
 * buffers replay the forward's Philox(seed) draw), depth_scene = forward scene depth (occlusion mask), g_* = upstream
 * gradients of the maps (NULL = 0);
 * dscene / dobj (N,S,4) = d(r,g,b,sigma).  models/rendering.py:139-229 under autograd. */
int onerf_composite_bwd(onerf_ctx* ctx, const onerf_composite_args* fwd, const float* depth_scene, const float* g_rgb,
                        const float* g_depth, const float* g_opacity, const float* g_rgb_inst, const float* g_depth_inst,
                        const float* g_opacity_inst, float* dscene, float* dobj, void* stream);

/* C[M x N] (+)= op(A) . B in fp32; B [K x N] and C row-major; trans_a = 0: A [M x K]; 1: A [K x M] (reduction over
 * A's rows, split over CTAs, atomics).  Used for dgrad (dIn = dZ W) and wgrad (dW += dZ^T In) of every nn.Linear. */
int onerf_gemm(onerf_ctx* ctx, const float* A, int lda, int trans_a, const float* B, int ldb, float* C, int ldc, int M,
               int N, int K, int accumulate, void* stream);

/* d <- d * (h > 0 ? 1 : 0.01): LeakyReLU backward from the layer OUTPUT (nn.LeakyReLU(inplace=True), nerf_model.py:38). */
int onerf_leaky_bwd(onerf_ctx* ctx, float* d, int ld_d, const float* h, int ld_h, int64_t rows, int cols, void* stream);

/* dA (n,4) = (d_rgb * rgb * (1 - rgb), d_sigma) from dfield (n,4) and the forward field output (n,4): sigmoid head. */
int onerf_head_bwd(onerf_ctx* ctx, const float* dfield, const float* field, float* dA, int64_t n, void* stream);

/* out[r][c] = sum over the S consecutive rows of ray r of in (per-ray-constant terms: dir / code columns). */
int onerf_segment_sum(onerf_ctx* ctx, const float* in, int ld_in, float* out, int ld_out, int n_rays, int n_samples,
                      int cols, void* stream);

/* out[c] += sum over rows of in[r][c] (bias gradients). */
int onerf_colsum(onerf_ctx* ctx, const float* in, int ld, int64_t rows, int cols, float* out, void* stream);

/* PE4 of the ray directions, (N,8) -> (N,27) (models/embedding_helper.py:57-74 on rays_d). */
int onerf_dir_encode(onerf_ctx* ctx, const float* rays, int n_rays, float* out, void* stream);

/* Encoding backward: dX [n_chunk x ldx] (X layout) -> scatter-add into table_grad (n_rows,24); X holds the forward's
 * sin/cos values; rays/z (N,8)/(N,S) and sample0 locate the chunk's samples.  models/embedding_helper.py:354-409. */
int onerf_encode_bwd(onerf_ctx* ctx, const onerf_grid* grid, const float* rays, const float* z, int n_rays, int n_samples,
                     const float* X, const float* dX, int ldx, int64_t sample0, int64_t n_chunk, float* table_grad,
                     void* stream);

/* Joint depth sort over all objects' samples + compositing, render_tools/multi_rendering.py:96-157.
 * Inputs are object-major: z_all (n_obj, N, S), field_all (n_obj, N, S, 4); the reference's concatenated
 * sample index is c = obj * S + s, ties are kept in that order (stable sort).  Outputs in sorted order,
 * (N, n_obj*S): z_sorted, weights, obj_ids (float list positions, or NULL); weights_unsorted
 * (n_obj, N, S) = each object's weights back in its own sample order (what multi_rendering.py:269-271
 * recovers with a boolean mask), or NULL.  Last delta is 0 (:125-128). */
int onerf_composite_multi(onerf_ctx* ctx, const float* z_all, const float* field_all, int n_rays,
                          int n_obj, int n_samples, int white_back, float* z_sorted, float* weights,
                          float* obj_ids, float* weights_unsorted, float* opacity, float* rgb,
                          float* depth, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* ONERF_H_ */
