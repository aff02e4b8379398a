/* Entry points added to ABI version 2 after its base set (include/onerf.h).  Additive only: the structs and the functions
 * of onerf.h are unchanged, so code built against onerf.h alone keeps working.  Same conventions as onerf.h: device
 * pointers, status codes, onerf_last_error(), kernels only enqueued on `stream`. */
#ifndef ONERF_EXT_H_
#define ONERF_EXT_H_

#include "onerf.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---------------------------------------------------------------------------------------------
 * onerf_composite_multi without its n_obj * n_samples <= 4096 limit.  Same inputs, outputs and stable-sort contract
 * (ties in concatenated-index order c = obj * S + s).  T = n_obj * n_samples <= 4096 runs the same bitonic kernel as
 * onerf_composite_multi (bit-identical outputs, workspace unused).  Larger T sorts each set on its own (n_samples <= 2048),
 * ranks every sample by binary search in the other sets of its ray and composites in that order with the same arithmetic;
 * it needs T < 2^31 and a 256-byte aligned workspace of onerf_composite_multi_workspace_bytes(n_rays, n_obj, n_samples)
 * bytes.  z_sorted and weights double as scratch between the steps, so they must not alias the inputs.
 * ------------------------------------------------------------------------------------------- */
size_t onerf_composite_multi_workspace_bytes(int n_rays, int n_obj, int n_samples);
int onerf_composite_multi_ws(onerf_ctx* ctx, const float* z_all, const float* field_all, int n_rays, int n_obj,
                             int n_samples, int white_back, float* z_sorted, float* weights, float* obj_ids,
                             float* weights_unsorted, float* opacity, float* rgb, float* depth, void* workspace,
                             size_t workspace_bytes, void* stream);

/* The rank-merge path of onerf_composite_multi_ws for every T, small ones included (tests compare it with the bitonic
 * kernel bit for bit). */
int onerf_composite_multi_merge(onerf_ctx* ctx, const float* z_all, const float* field_all, int n_rays, int n_obj,
                                int n_samples, int white_back, float* z_sorted, float* weights, float* obj_ids,
                                float* weights_unsorted, float* opacity, float* rgb, float* depth, void* workspace,
                                size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Sigma noise and box-clipped ray sets on the editing path (render_tools/multi_rendering.py:131-132, 278-287).
 *
 * onerf_composite_multi_noise_ws / _merge: onerf_composite_multi_ws / _merge with alpha taken from
 * relu(sigma + noise * noise_std) (the multiply rounded first).  The noise is indexed by SORTED position: sample p of ray r
 * takes noise[r * T + p] ((N, T) row-major, T = n_obj * n_samples) if `noise` is given, else the Philox normal of stream
 * ONERF_STREAM_MULTI_NOISE_COARSE (pass 0) or ONERF_STREAM_MULTI_NOISE_FINE (pass 1) at element r * T + p keyed by
 * `seed` (the draw of onerf_composite's streams 2 / 3 with another stream id).  Both paths give the same bits for the same
 * order.  noise_std = 0 draws nothing and gives the bits of the entries without noise.  Refusals (ONERF_ERR_BAD_ARG):
 * noise_std negative or not finite, a noise buffer with noise_std = 0, a noise buffer not 4-byte aligned, pass not 0 / 1.
 *
 * onerf_sample_pdf_merge_clip: onerf_sample_pdf_merge whose merged row is stored through the box clip of a 10-column ray
 * set: with (near_box, far_box) = clip[r] ((N,2) row-major), every z with near_box < z < far_box (both strict) becomes
 * far_box.  Comparisons only: bit-exact, and the row stays ascending.  clip NULL is onerf_sample_pdf_merge.  Refusals: a
 * clip not 8-byte aligned or a u not 4-byte aligned, and those of onerf_sample_pdf_merge.
 * ------------------------------------------------------------------------------------------- */
#define ONERF_STREAM_MULTI_NOISE_COARSE 7
#define ONERF_STREAM_MULTI_NOISE_FINE 8
int onerf_composite_multi_noise_ws(onerf_ctx* ctx, const float* z_all, const float* field_all, int n_rays, int n_obj,
                                   int n_samples, int white_back, float noise_std, const float* noise, uint64_t seed,
                                   int pass, float* z_sorted, float* weights, float* obj_ids, float* weights_unsorted,
                                   float* opacity, float* rgb, float* depth, void* workspace, size_t workspace_bytes,
                                   void* stream);
int onerf_composite_multi_noise_merge(onerf_ctx* ctx, const float* z_all, const float* field_all, int n_rays, int n_obj,
                                      int n_samples, int white_back, float noise_std, const float* noise, uint64_t seed,
                                      int pass, float* z_sorted, float* weights, float* obj_ids, float* weights_unsorted,
                                      float* opacity, float* rgb, float* depth, void* workspace, size_t workspace_bytes,
                                      void* stream);
int onerf_sample_pdf_merge_clip(onerf_ctx* ctx, const float* z_coarse, const float* weights, int n_rays, int n_samples,
                                int n_importance, int det, const float* u, uint64_t seed, const float* clip, float* z_out,
                                void* stream);

/* onerf_render_multi_fwd with what render_rays_multi takes beyond it.  onerf_render_multi_fwd is this call with a zeroed
 * onerf_render_multi_ext (ext == NULL is the same).  The coarse pass composites with noise_coarse (or stream 7), the
 * fine pass with noise_fine (or stream 8), both keyed by args->seed; the coarse weights that feed each set's importance
 * sampling are the noised ones.  Set i draws its importance u from u_list_host[i] when given, else as
 * onerf_render_multi_fwd does (Philox stream 1 keyed by args->seed + i; linspace when perturb = 0).  A set with
 * clip_list_host[i] != NULL is a 10-column set: its fine depths go through onerf_sample_pdf_merge_clip's clip, which the
 * muting test (z[:, -1] == 0) and the box culling see; its coarse depths are not clipped, and without a fine pass the
 * clip is unused.  Sets with and without a clip may be mixed.
 * Refusals (ONERF_ERR_BAD_ARG), besides those of onerf_render_multi_fwd: noise_std negative or not finite; a noise buffer
 * with noise_std = 0, or noise_fine without a fine pass; a u with perturb = 0 or without a fine pass; a noise or u buffer
 * not 4-byte aligned, a clip not 8-byte aligned. */
typedef struct onerf_render_multi_ext {
  float noise_std;                    /* 0: no noise, nothing drawn */
  const float* noise_coarse;          /* (N, n_obj * n_samples) N(0,1) in sorted order, or NULL */
  const float* noise_fine;            /* (N, n_obj * (n_samples + n_importance)), or NULL */
  const float* const* clip_list_host; /* NULL, or n_obj DEVICE pointers (host array) to (N,2) (near_box, far_box), NULL
                                         for a set without a clip */
  const float* const* u_list_host;    /* NULL, or n_obj DEVICE pointers (host array) to (N, n_importance) U[0,1), NULL
                                         entries drawn */
} onerf_render_multi_ext;

int onerf_render_multi_fwd_ext(onerf_ctx* ctx, const onerf_render_multi_args* args, const onerf_render_multi_ext* ext,
                               void* stream);

/* ---------------------------------------------------------------------------------------------
 * Size of the training workspace of onerf_render_rays_fwd / onerf_render_rays_bwd for either arithmetic (precision =
 * onerf_precision); onerf_train_workspace_bytes is this with ONERF_PREC_BF16.  The fp32 workspace holds both passes'
 * fields and one chunk (at most 65 536 samples) of the backward's activation dump and gradient buffers.  0 for an
 * unknown precision or a bad shape.
 * ------------------------------------------------------------------------------------------- */
size_t onerf_train_workspace_bytes_prec(int precision, int use_voxel, int n_rays, int n_samples, int n_importance);

/* ---------------------------------------------------------------------------------------------
 * One training step in one call (train.py:147-180 up to loss.backward()): onerf_render_rays_fwd, TotalLoss and
 * onerf_render_rays_bwd with the loss and the compositing backward fused into the compositing kernels.  A batch kernel
 * first sums what TotalLoss normalises by and skips on (it depends on the batch only); each pass's compositing kernel then
 * composites a ray, forms its loss terms and map gradients and runs the compositing backward while the ray's alpha and
 * transmittance are on chip; the last one writes the loss outputs and the PSNR.  The field backward follows as in
 * onerf_render_rays_bwd.  Only enqueues work on `stream` (no host read, no allocation): CUDA-graph capturable.
 *   fwd    onerf_render_args as for onerf_render_rays_fwd; forward_instance must be set; train_ws of
 *          onerf_train_step_workspace_bytes(...) bytes, 1024-byte aligned.  Both passes' maps are written.
 *   loss   batch inputs, term weights and outputs of onerf_total_loss (loss_sum_out, terms_out, present_out);
 *          n_rays = fwd->n_rays, has_fine = (n_importance > 0); the map, grad_* and workspace fields are unused.
 *   bwd    as for onerf_render_rays_bwd (gradients accumulated); its map gradients are unused.
 *   psnr_out (1,) = -10 log10(mean over valid rays of (rgb - rgbs)^2) of the fine pass (coarse without one).
 * ------------------------------------------------------------------------------------------- */
size_t onerf_train_step_workspace_bytes(int precision, int use_voxel, int n_rays, int n_samples, int n_importance);
int onerf_train_step(onerf_ctx* ctx, const onerf_render_args* fwd, const onerf_loss_args* loss,
                     const onerf_render_bwd_args* bwd, float* psnr_out, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Device seed.  As onerf_render_rays_fwd / onerf_train_step, with args->seed ignored: every draw the call makes without
 * an injected buffer (jitter, u, noise_*) uses the seed *seed_dev holds when its kernel runs, exactly as the host-seed
 * call with args->seed = *seed_dev draws, and the call's last device work adds 4 to *seed_dev (also when nothing is
 * drawn).  seed_dev: one uint64 in device memory, 8-byte aligned.  Kernels only: CUDA-graph capturable, and each replay
 * draws with the next seed (replay k of a graph captured with *seed_dev = s0 draws as the host-seed call with s0 + 4k).
 * onerf_render_rays_fwd_dseed refuses train_ws != NULL (ONERF_ERR_BAD_ARG): onerf_render_rays_bwd replays the sigma noise
 * from the host seed.
 * ------------------------------------------------------------------------------------------- */
int onerf_render_rays_fwd_dseed(onerf_ctx* ctx, const onerf_render_args* args, uint64_t* seed_dev, void* stream);
int onerf_train_step_dseed(onerf_ctx* ctx, const onerf_render_args* fwd, const onerf_loss_args* loss,
                           const onerf_render_bwd_args* bwd, float* psnr_out, uint64_t* seed_dev, void* stream);

/* ---------------------------------------------------------------------------------------------
 * An edited frame from a camera (EditableRenderer.render_edit, editable_renderer.py:203-294), or a contiguous tile of it.
 * Pixels [pixel_begin, pixel_end) (row-major) of the H x W frame are rendered in chunks of chunk_rays pixels; for each
 * chunk every set's rays are generated on the device exactly as onerf_camera_rays generates them for those pixels, the
 * chunk runs through onerf_render_multi_fwd's path (perturb = 0 and no noise, so nothing is random; 8-column sets) and
 * its maps are written to rows
 * [chunk - pixel_begin, ...) of the tile-sized outputs.  Every result row depends on its pixel only, never on chunk_rays
 * or the tile bounds.
 *   sets_host  n_obj ray sets (host array).  obj_id 0 = scene branch (box NULL: near / far = near, far / scale_factor),
 *              otherwise the object branch with code_table[obj_id] (box required, bbox_enlarge applied: near / far from
 *              the slab test, 0 / 0 for a miss).  Toc: row-major (3,4) camera-to-set pose, translation at NeRF scale.
 *   maps       tile-sized (N = pixel_end - pixel_begin rows), shapes of onerf_render_multi_maps.  Any array may be NULL:
 *              it is not written (its values go to chunk scratch in the workspace).
 *   workspace  >= onerf_render_edit_workspace_bytes(chunk_rays, n_obj, n_samples, n_importance) bytes, 256-byte aligned
 *              (0 for a bad shape).
 * Limits and refusals of onerf_render_multi_fwd, plus: a tile outside [0, H*W], chunk_rays < 1, an object set without a
 * box or the scene set with one, a bad camera (H, W or focal not positive).  Kernels only, no host read.
 * ------------------------------------------------------------------------------------------- */
typedef struct onerf_edit_set {
  int obj_id;
  float Toc[12];
  const onerf_box_host* box;
} onerf_edit_set;

typedef struct onerf_render_edit_args {
  const onerf_edit_set* sets_host;
  int n_obj;
  int H, W;
  float focal;
  int64_t pixel_begin, pixel_end;
  double near, far, scale_factor;
  int n_samples, n_importance;
  const onerf_grid* grid;
  const void* packed_coarse;
  const void* packed_fine;            /* required iff n_importance > 0 */
  const float* code_table;            /* (n_codes,64) */
  int n_codes;
  int precision;                      /* onerf_precision */
  int use_disp, white_back;
  const float* boxes;                 /* (n_boxes,18) removed-object boxes of the scene set, or NULL */
  int n_boxes;
  int chunk_rays;
  onerf_render_multi_maps coarse;
  onerf_render_multi_maps fine;       /* written iff n_importance > 0 */
  void* workspace;
  size_t workspace_bytes;
} onerf_render_edit_args;

size_t onerf_render_edit_workspace_bytes(int chunk_rays, int n_obj, int n_samples, int n_importance);
int onerf_render_edit_frame(onerf_ctx* ctx, const onerf_render_edit_args* args, void* stream);

/* ---------------------------------------------------------------------------------------------
 * onerf_render_edit_frame plus, per pass, how much of each pixel each ray set shows.  For ray r, set position i (the
 * list position, as obj_ids numbers the sets: duplicates of one object are separate columns) and the pass's weights w
 * (those written to maps.weights: the joint compositing's, with the removed-object boxes and the box culling as there),
 * summed over set i's samples:
 *   opacity  (N, n_obj)     sum w
 *   depth    (N, n_obj)     sum w z
 *   rgb      (N, n_obj, 3)  sum w rgb, with no white background (white_back applies to maps.rgb only)
 * For the coarse pass this is weights summed by obj_ids; summed over i the maps give the pass's opacity, depth and rgb
 * (without the white background) up to float32 reassociation.  Each (ray, set) is a fixed-order sum over the set's
 * weights in sample order, so every value is bit-identical whatever chunk_rays, the tile bounds or the sort path.  A set
 * whose ray misses its box and a sample muted by a removed-object box add exactly 0.
 *   coarse, fine   NULL, or tile-sized outputs (rows as maps); any NULL array is not written.  A fine array needs
 *                  n_importance > 0.  Arrays 4-byte aligned.
 *   workspace      >= onerf_render_edit_sets_workspace_bytes(chunk_rays, n_obj, n_samples, n_importance) bytes when any
 *                  array is given (the fine pass's weights in set order need one more chunk-sized buffer; the same as
 *                  onerf_render_edit_workspace_bytes without a fine pass), else as onerf_render_edit_frame.
 * onerf_render_edit_frame is this call with coarse = fine = NULL, and the other outputs do not change with the set maps.
 * Refusals (ONERF_ERR_BAD_ARG), before any launch, besides those of onerf_render_edit_frame: a fine array without a fine
 * pass, an array not 4-byte aligned.  Kernels only, no host read: CUDA-graph capturable.
 * ------------------------------------------------------------------------------------------- */
typedef struct onerf_set_maps {
  float* opacity;                     /* (N, n_obj) or NULL */
  float* depth;                       /* (N, n_obj) or NULL */
  float* rgb;                         /* (N, n_obj, 3) or NULL */
} onerf_set_maps;

size_t onerf_render_edit_sets_workspace_bytes(int chunk_rays, int n_obj, int n_samples, int n_importance);
int onerf_render_edit_frame_sets(onerf_ctx* ctx, const onerf_render_edit_args* args, const onerf_set_maps* coarse,
                                 const onerf_set_maps* fine, void* stream);

/* ---------------------------------------------------------------------------------------------
 * onerf_render_edit_frame_sets with objects from other trained scenes.  The frame's BASE scene is the one args describes
 * (grid, packed weights, code_table, scale_factor s_base).  Set i with set_scene_host[i] = j >= 0 comes from SOURCE scene
 * scenes_host[j] instead, with its own voxel grid, packed weights (same architecture and precision as the frame), code
 * table and scale_factor s_src, and is evaluated exactly as a native object set of that scene:
 *   - its rays from its Toc, whose translation is at the source's NeRF scale (divided by s_src), and its box slab test
 *     un-scaled with s_src;
 *   - its coarse depths, fields (its grid, weights and code row), importance sampling and fine depths in the source's
 *     units, from its own weights.
 * The joint compositing of each pass then takes, with k = float32(s_src / s_base) computed in double, the set's depths
 * as z * k (on the base scene's axis) and its densities as sigma / k (each interval keeps its optical depth).  This is
 * render_rays_multi (multi_rendering.py:160-325) run per set in the set's own units, with volume_rendering_multi given
 * [z_i * k_i] and [sigma_i / k_i].  Every output is in base-scene units: z_vals, depth and the per-set depth maps.  A
 * frame whose sets all have k == 1 converts nothing: such a set's outputs are bit-identical to the same set rendered
 * natively from a base scene with its values.
 * Source scenes contribute object sets only (obj_id > 0); the removed-object boxes mute the base scene set only.
 *   scenes_host     n_scenes source scenes (host array; NULL when n_scenes = 0).
 *   set_scene_host  n_obj ints (host array): -1 = base scene, else an index into scenes_host.  NULL: every set is of
 *                   the base scene.
 *   coarse, fine    per-set maps as for onerf_render_edit_frame_sets (NULL: none).
 *   workspace       >= onerf_render_edit_scenes_workspace_bytes(chunk_rays, n_obj, n_samples, n_importance) bytes when
 *                   any set comes from a source scene (the sets entry's, plus one (n_obj, chunk, S + K) float buffer for
 *                   a pass's depths on the base axis), else as onerf_render_edit_frame_sets.
 * onerf_render_edit_frame_sets (and so onerf_render_edit_frame) is this call with no source scenes.  Refusals before any
 * launch, besides those of onerf_render_edit_frame_sets (ONERF_ERR_BAD_ARG unless noted): a negative n_scenes or a NULL
 * scenes_host with n_scenes > 0; in a scene a NULL grid, grid buffer, packed_coarse or code_table, a misaligned grid
 * table, a NULL packed_fine when n_importance > 0, a scale_factor that is not positive and finite (or whose ratio k is
 * not a positive finite float); a set scene index outside [-1, n_scenes); an object id outside its source scene's code
 * table; a source scene set with obj_id 0 (ONERF_ERR_UNSUPPORTED).  Kernels and device copies only, no host read:
 * CUDA-graph capturable.  Each pass with a set of k != 1 adds one device copy of its depths and one rescale launch per
 * such set.
 * ------------------------------------------------------------------------------------------- */
typedef struct onerf_edit_scene {
  const onerf_grid* grid;
  const void* packed_coarse;
  const void* packed_fine;            /* required iff n_importance > 0 */
  const float* code_table;            /* (n_codes,64) */
  int n_codes;
  double scale_factor;
} onerf_edit_scene;

size_t onerf_render_edit_scenes_workspace_bytes(int chunk_rays, int n_obj, int n_samples, int n_importance);
int onerf_render_edit_frame_scenes(onerf_ctx* ctx, const onerf_render_edit_args* args, const onerf_edit_scene* scenes_host,
                                   int n_scenes, const int* set_scene_host, const onerf_set_maps* coarse,
                                   const onerf_set_maps* fine, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Training batches drawn on the device (GenericDataset.__getitem__ through DataLoader(shuffle=True), and under DDP
 * DistributedSampler; datasets/generic_dataset.py:475-490, train.py:121-129).  The dataset's R rays stay in device
 * memory; one launch draws batch `step` of rank `rank` into B-row outputs:
 *   P = floor(R / (B * W)) full batches per epoch (the last R - P*B*W positions of each epoch's order are not drawn);
 *   epoch e = step / P, j = step mod P; element b takes position p = (j*B + b)*W + rank of epoch e's permutation
 *   pi_{seed,e} of [0, R) (a 6-round Feistel network on [0, 2^m), m the smallest even m >= 2 with 2^m >= R, round
 *   function philox4x32 keyed by seed with counter (right half, (uint32)e, 5, round), cycle-walked into [0, R));
 *   ray i = pi(p) gives rays, rgbs, depths, valid_mask and frame_idx; instance column c = (w * I) >> 32, with w word
 *   (n & 3) of philox4x32((n >> 2, n >> 34, 4, 0), seed) at n = (step*B + b)*W + rank, gives instance_mask,
 *   instance_mask_weight, instance_ids and pass_through_mask (row i, column c).
 * Every rank with the same seed shares the permutation and draws a disjoint stride of it.
 *   data       device buffers of the dataset.  frame_idx may be NULL (frame_idx_out is then filled with -1).
 *   outputs    B rows: rays (B,8), rgbs (B,3), depths, valid_mask, frame_idx (B,); instance_mask, instance_mask_weight,
 *              instance_ids, pass_through_mask (B,) (the layout of onerf_loss_args and onerf_train_step's batch).
 *              frame_idx and index_out may be NULL; index_out (B,2) = (ray i, column c) per row.
 * Refusals (ONERF_ERR_BAD_ARG): a null ctx, argument block or required buffer, B < 1, W < 1, rank outside [0, W),
 * I < 1, R < B*W (P = 0), R >= 2^40.  Kernels only, no host read: CUDA-graph capturable.
 * onerf_draw_batch_dstep ignores args->step: its kernel reads the step from *step_dev (one uint64, 8-byte aligned) and a
 * one-thread follow-up launch adds 1 to it, so each replay of a captured call draws the next batch.
 * ------------------------------------------------------------------------------------------- */
typedef struct onerf_ray_dataset {
  int64_t n_rays;                       /* R */
  int n_instances;                      /* I: instance columns per ray */
  const float* rays;                    /* (R,8) */
  const float* rgbs;                    /* (R,3) */
  const float* depths;                  /* (R,) */
  const uint8_t* valid_mask;            /* (R,) 0 / 1 */
  const int64_t* frame_idx;             /* (R,) or NULL */
  const uint8_t* instance_mask;         /* (R,I) 0 / 1 */
  const float* instance_mask_weight;    /* (R,I) */
  const int64_t* instance_ids;          /* (R,I) */
  const uint8_t* pass_through_mask;     /* (R,I) 0 / 1 */
} onerf_ray_dataset;

typedef struct onerf_batch_args {
  onerf_ray_dataset data;
  int batch;                            /* B */
  int rank, world;                      /* W = world */
  uint64_t seed;
  uint64_t step;                        /* onerf_draw_batch only */
  float* rays;
  float* rgbs;
  float* depths;
  uint8_t* valid_mask;
  int64_t* frame_idx;                   /* or NULL */
  uint8_t* instance_mask;
  float* instance_mask_weight;
  int64_t* instance_ids;
  uint8_t* pass_through_mask;
  int64_t* index_out;                   /* (B,2) or NULL */
} onerf_batch_args;

int onerf_draw_batch(onerf_ctx* ctx, const onerf_batch_args* args, void* stream);
int onerf_draw_batch_dstep(onerf_ctx* ctx, const onerf_batch_args* args, uint64_t* step_dev, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Training batches drawn from a frame store: onerf_draw_batch over the R = F*H*W rays GenericDataset would expand the
 * frames into, each drawn row rebuilt from its pixel instead of read from per-ray buffers.  Ray i = f*H*W + p (frame f,
 * pixel p = y*W + x row-major) and column c are drawn exactly as onerf_draw_batch draws them (same seed, step, rank and
 * world give the same (i, c)); the row's fields are
 *   rays           (o, d, near_s, far_s): o = poses[f] translation, d = directions[p] rotated by poses[f] and normalised
 *                  with onerf_get_rays' arithmetic;
 *   rgbs           rgb[f,p,k] / 255 (IEEE division, as torchvision's ToTensor);
 *   depths         depths[f,p];
 *   valid_mask     1 iff border <= x < W - border and border <= y < H - border;
 *   frame_idx      frame_idx[f];
 *   instance_ids   ids[c];
 *   instance_mask, instance_mask_weight, pass_through_mask
 *                  mask_all_ones[c]: 1, weights[f,c,1], 1; otherwise with l = labels[f,p]: m = (l == ids[c]),
 *                  weights[f,c,m], and 1 iff l is one of pass_ids[c, 0..n_pass) (-1 pads a row: it matches no label).
 * Outputs, seed, step, rank, world and index_out are those of onerf_batch_args; args->data is not read.
 * Refusals (ONERF_ERR_BAD_ARG): those of onerf_draw_batch with R = F*H*W, and a null frame store, a null table, a null
 * labels buffer with a column whose mask is not all ones, F, H or W < 1, border < 0, n_pass outside [1,
 * ONERF_FRAME_MAX_PASS].  Kernels only, no host read: CUDA-graph capturable; onerf_draw_frames_dstep steps as
 * onerf_draw_batch_dstep does.
 * ------------------------------------------------------------------------------------------- */
#define ONERF_FRAME_MAX_PASS 16

typedef struct onerf_frame_dataset {
  int n_frames, H, W;                   /* F, H, W */
  int n_instances;                      /* I */
  const float* poses;                   /* (F,12) row-major (3,4) c2w */
  const float* directions;              /* (H*W,3) from onerf_ray_directions */
  const uint8_t* rgb;                   /* (F,H*W,3) */
  const float* depths;                  /* (F,H*W) */
  const uint16_t* labels;               /* (F,H*W), or NULL when every column's mask is all ones */
  const int64_t* frame_idx;             /* (F,) */
  float near_s, far_s;                  /* near / scale_factor, far / scale_factor */
  int border;
  const int64_t* ids;                   /* (I,) */
  const uint8_t* mask_all_ones;         /* (I,) 0 / 1 */
  const float* weights;                 /* (F,I,2): [background, foreground] */
  const int32_t* pass_ids;              /* (I,n_pass) */
  int n_pass;
} onerf_frame_dataset;

int onerf_draw_frames(onerf_ctx* ctx, const onerf_frame_dataset* frames, const onerf_batch_args* args, void* stream);
int onerf_draw_frames_dstep(onerf_ctx* ctx, const onerf_frame_dataset* frames, const onerf_batch_args* args,
                            uint64_t* step_dev, void* stream);

/* ---------------------------------------------------------------------------------------------
 * One validation image, or a contiguous tile of it, in one call (train.py:73-105, 182-223: ObjectNeRFSystem.forward over
 * the image, TotalLoss, psnr).  Rays [ray_begin, ray_end) of the image's batch are rendered in chunks of chunk_rays rays
 * through onerf_render_rays_fwd's passes (is_eval, nothing random); the compositing kernel of each pass also adds the
 * ray's squared errors of the five TotalLoss terms and of the validation PSNR to `record`.  Per-sample arrays (weights,
 * z_vals) exist only for one chunk, in the workspace.
 *   record   ONERF_VALIDATE_RECORD_DOUBLES doubles, 8-byte aligned, zeroed by the call before it adds to it:
 *            [0..5) element counts of the five masked means, [5] number of depths > 0 (both from the tile's batch rows),
 *            [6..16) squared-error sums, term * 2 + (0 coarse / 1 fine), [16] PSNR squared-error sum, [17] PSNR element
 *            count.  All sums over rays: the record of a frame is the sum of the records of its tiles, which is what a
 *            process group all-reduces before onerf_validate_finalize.
 *   render   as for onerf_render_rays_fwd, for the whole image: rays (n_rays,8), n_rays, models, grid, precision, sample
 *            counts, use_disp, white_back, rays_in_bbox.  forward_instance and is_eval must be set, perturb and noise_std 0,
 *            train_ws NULL.  codes is ignored: each chunk's codes are gathered from code_table by instance_ids.
 *            coarse / fine: tile-sized maps (ray_end - ray_begin rows); any may be NULL: it is not written (its values
 *            go to chunk scratch).  weights and z_vals are ignored (never tile-sized).  workspace: >=
 *            onerf_validate_workspace_bytes(chunk_rays, n_samples, n_importance) bytes (0 for a bad shape), 256-byte
 *            aligned; its size does not depend on the image.
 *   loss     the image's batch rows (n_rays = render.n_rays), the term weights and, with `finalize`, the outputs
 *            loss_sum_out, terms_out, present_out as for onerf_total_loss; maps, grad_* and workspace are unused.
 *   psnr_mask  which rays the PSNR of the last pass's rgb averages over (train.py:185-190): ONERF_PSNR_VALID_INSTANCE =
 *            valid_mask * instance_mask, ONERF_PSNR_ALL_RAYS = every ray, valid or not (a batch without instance_mask).
 *   finalize 1: onerf_validate_finalize runs on the record as the call's last launch (the single-process frame);
 *            psnr_out (1,) is then required.
 * Every map row depends on its ray only, never on chunk_rays or the tile bounds, and is bit-identical to
 * onerf_render_rays_fwd (is_eval = 1) over the same rays.  Refusals (ONERF_ERR_BAD_ARG): a tile outside [0, n_rays],
 * chunk_rays < 1, forward_instance or is_eval off, a training workspace, perturb or noise_std non-zero, a NULL or
 * misaligned record, a NULL batch buffer, a misaligned or undersized workspace.  Kernels and one memset only, no host
 * read, no allocation: CUDA-graph capturable.
 *
 * onerf_validate_finalize: one single-block launch that turns a record into loss_sum (1,), the five unweighted terms
 * (5,), the present flags (5,) (skip rules of onerf_total_loss; an empty color mask gives NaN as the reference's mean of
 * an empty set does) and psnr (1,) = -10 log10(record[16] / record[17]) (NaN for an empty mask).  weights: host array of
 * the five loss.*_weight.  A launch of its own, so that the record can be reduced across ranks in between.
 * ------------------------------------------------------------------------------------------- */
#define ONERF_VALIDATE_RECORD_DOUBLES 18
typedef enum onerf_psnr_mask { ONERF_PSNR_VALID_INSTANCE = 0, ONERF_PSNR_ALL_RAYS = 1 } onerf_psnr_mask;

typedef struct onerf_validate_args {
  onerf_render_args render;
  onerf_loss_args loss;
  const int64_t* instance_ids;          /* (n_rays,) */
  const float* code_table;              /* (n_codes,64) */
  int n_codes;
  int64_t ray_begin, ray_end;
  int chunk_rays;
  int psnr_mask;                        /* onerf_psnr_mask */
  double* record;
  int finalize;
  float* psnr_out;                      /* (1,), with finalize */
} onerf_validate_args;

size_t onerf_validate_workspace_bytes(int chunk_rays, int n_samples, int n_importance);
int onerf_validate_frame(onerf_ctx* ctx, const onerf_validate_args* args, void* stream);
int onerf_validate_finalize(onerf_ctx* ctx, const double* record, const float weights[5], int has_fine,
                            float* loss_sum_out, float* terms_out, int* present_out, float* psnr_out, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Voxel pruning (EmbeddingVoxel.self_pruning_empty_voxels, models/embedding_helper.py:202-245), in two launches so that a
 * process group can all-gather the per-voxel maxima in between.
 *
 * onerf_prune_measure: for every voxel k of the shard [cell_begin, cell_end) of cells (K = n_cells rows (i, j, l), the
 * order of torch.nonzero(voxel_occupancy)), max_alpha_out[k - cell_begin] = the largest alpha = 1 - exp(-relu(sigma))
 * of the scene branch's density over the voxel's 4096 samples.  Sample s of voxel k sits at
 *   centre + (r * voxel_size - voxel_size / 2),   centre = float(cell) * voxel_size - voxel_offset
 * (fp32, each operation rounded on its own, the reference's order), r = jitter row k * 4096 + s, or without jitter
 * component c of r = philox4x32 uniform of stream 6 at element (k * 4096 + s) * 3 + c, keyed by seed (the draw of
 * onerf_sample_coarse's stream 0 with another stream id).  Rows of a voxel depend on k, never on the shard.
 *   grid       required: the voxel model only.  packed: its onerf_pack_weights blob.
 *   precision  ONERF_PREC_BF16: one fused tensor-core pass (sigma bit-identical to onerf_field_fwd's scene branch on the
 *              same points); ONERF_PREC_FP32: per chunk of 32 voxels, the points, onerf_field_fwd's FFMA field (scene
 *              only) and a per-voxel maximum.
 *   jitter     (n_cells * 4096, 3) U[0,1), indexed by the global k, or NULL.
 *   max_alpha_out  (cell_end - cell_begin,) floats, 4-byte aligned; zeroed by the call first.
 *   workspace  >= onerf_prune_workspace_bytes(precision) bytes, 256-byte aligned (0 bytes for bf16: may be NULL).
 * Refusals (ONERF_ERR_BAD_ARG): null ctx / args / grid / packed, null cells with K > 0, null max_alpha_out with a
 * non-empty shard, a shard outside [0, K], misaligned cells / jitter / max_alpha_out / workspace, an unknown precision;
 * ONERF_ERR_WORKSPACE: a workspace that is too small.
 *
 * onerf_prune_apply: every voxel k in [0, n_cells) with max_alpha[k] < max_alpha_th gets occupancy[cell] = 0 and
 * idx_map[cell] = -1 (dense (X, dim_y, dim_z) arrays, uint8 and int64); *n_pruned (int64, device) = their count.
 * Table rows are not renumbered.  Refusals (ONERF_ERR_BAD_ARG): null pointers, K < 0, dim_y or dim_z < 1, misaligned
 * buffers.
 * Both calls enqueue kernels and memsets only, with no host read.
 * ------------------------------------------------------------------------------------------- */
#define ONERF_PRUNE_SAMPLES 4096

typedef struct onerf_prune_args {
  const onerf_grid* grid;
  const void* packed;
  int precision;                        /* onerf_precision */
  const int64_t* cells;                 /* (n_cells,3) */
  int64_t n_cells;
  int64_t cell_begin, cell_end;
  const float* jitter;                  /* (n_cells * 4096,3) or NULL */
  uint64_t seed;
  float* max_alpha_out;                 /* (cell_end - cell_begin,) */
  void* workspace;
  size_t workspace_bytes;
} onerf_prune_args;

size_t onerf_prune_workspace_bytes(int precision);
int onerf_prune_measure(onerf_ctx* ctx, const onerf_prune_args* args, void* stream);
int onerf_prune_apply(onerf_ctx* ctx, const int64_t* cells, int64_t n_cells, const float* max_alpha, float max_alpha_th,
                      int64_t dim_y, int64_t dim_z, uint8_t* occupancy, int64_t* idx_map, int64_t* n_pruned, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Backward of one field evaluation: ObjectNeRF.forward / forward_instance and inference_model under autograd
 * (models/nerf_model.py:97-152, models/rendering.py:85-137).  A point query is a ray of one sample: rays[:, 3:6] = its
 * direction, z = 0, xyz (B,1,3) = the points, codes (B,64) one row per point.
 *   fwd      the onerf_field_fwd arguments of the forward: want_scene set, dense z and outputs (z_stride = out_stride =
 *            n_samples), no editing extras, per-ray `codes` (not code_row) with want_object, xyz optional.
 *            ONERF_PREC_BF16: the forward ran with train_ws (its dump) and its scene_out / obj_out still hold the fields;
 *            ONERF_PREC_FP32: the backward re-runs the FFMA forward chunk by chunk with its activation dump.
 *   d_scene, d_obj  (n_rays * n_samples, 4) d(r, g, b, sigma) of scene_out / obj_out (the float4 field layout); NULL = 0.
 *            d_obj needs want_object.
 *   grads    W: the 20 reference weight tensors (onerf_pack_weights order); dW / db: their gradients, ACCUMULATED (as
 *            in onerf_render_bwd_args), all 20 pairs required, also without want_object; d_codes (n_rays,64)
 *            accumulated, or NULL; table_grad (n_rows,24) accumulated, or
 *            NULL (must be NULL for the plain-PE model); workspace >= onerf_field_bwd_workspace_bytes(precision,
 *            grid != NULL, n_rays, n_samples) bytes, 1024-byte aligned.
 * The stages are those of onerf_render_rays_bwd after its compositing backward: head -> input-gradient chain -> weight
 * gradients -> per-ray-constant columns and d(code) -> encoding gradient, with each sample's position read from xyz when
 * it is given.  Without want_object the object layers' dW / db keep their values (bf16 adds zeros to them, fp32 does not
 * touch them).  No gradient flows to rays, z or xyz.
 * Refusals: ONERF_ERR_BAD_ARG for the conditions above, ONERF_ERR_WORKSPACE for a small workspace.
 *
 * onerf_bwd_dx_xyz / onerf_encode_bwd_xyz: onerf_bwd_dx / onerf_encode_bwd with sample e at xyz[3 e .. 3 e + 2] instead
 * of o + d z (stage entries).
 * ------------------------------------------------------------------------------------------- */
typedef struct onerf_field_bwd_args {
  const float* const* W;
  float* const* dW;
  float* const* db;
  float* d_codes;
  float* table_grad;
  void* workspace;
  size_t workspace_bytes;
} onerf_field_bwd_args;

size_t onerf_field_bwd_workspace_bytes(int precision, int use_voxel, int n_rays, int n_samples);
int onerf_field_bwd(onerf_ctx* ctx, const onerf_field_args* fwd, const float* d_scene, const float* d_obj,
                    const onerf_field_bwd_args* grads, void* stream);
int onerf_bwd_dx_xyz(onerf_ctx* ctx, int want_object, const void* packed, const void* ws, const float* xyz, int64_t n_samples,
                     const onerf_grid* grid, float* table_grad, void* stream);
int onerf_encode_bwd_xyz(onerf_ctx* ctx, const onerf_grid* grid, const float* xyz, const float* X, const float* dX, int ldx,
                         int64_t sample0, int64_t n_chunk, float* table_grad, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Masked PSNR and SSIM of a held-out frame, for the scene and for each of K objects (utils/metrics.py:14-23 with a mask).
 * Column 0 is the scene: mask m = valid, prediction pred_scene.  Column k >= 1 is object ids_host[k-1]: m = valid &
 * (labels == ids_host[k-1]), prediction pred_object.  Per column, with both images set to 0 outside m:
 *   - each channel filtered with g = outer(g1, g1), g1[i] = exp(-(i - w/2)^2 / (2 * 1.5^2)) normalised to sum 1
 *     (w = window), reflect padding of w/2 (F.pad(mode="reflect"): mirror without repeating the edge), H x W output;
 *   - mu_p, mu_g, s_pp = E[p^2] - mu_p^2, s_gg, s_pg from those window sums, and
 *     ssim_map = ((2 mu_p mu_g + C1)(2 s_pg + C2)) / ((mu_p^2 + mu_g^2 + C1)(s_pp + s_gg + C2)), C1 = 0.01^2, C2 = 0.03^2;
 *   - SSIM = mean of clamp(ssim_map, 0, 1) over the 3 channels of the pixels in m;
 *   - PSNR = -10 log10(mean squared error over the 3 channels of the pixels in m).
 * An empty mask gives NaN for both.  With m all ones, SSIM is kornia 0.4.1's losses.ssim(pred, gt, w) read as
 * 1 - 2 * dssim.  Window sums, ssim_map and the error sums are fp64.
 *
 * onerf_image_metrics: adds one frame's sums to `record` ((K+1) x 3 doubles: squared-error sum, clamped ssim_map sum,
 * pixel count of m, per column), which must hold zeros (or an earlier part of the same frame) before the call.
 * onerf_image_metrics_finalize: one launch that writes psnr_out[slot, :] and ssim_out[slot, :] ((F, K+1) row-major
 * float32; either may be NULL: not written) from the record and zeroes it.  Only window, n_ids, record, psnr_out and
 * ssim_out are read.
 *   pred_scene, gt  (H*W, 3) float32, row-major pixels; pred_object (H*W, 3), NULL when K = 0
 *   valid           (H*W) uint8 0 / 1, or NULL: every pixel
 *   labels          (H*W) uint16, NULL when K = 0
 *   ids_host        K ints in [0, 65535] (host array), 0 <= K <= ONERF_METRICS_MAX_IDS
 * Refusals (ONERF_ERR_BAD_ARG): an even window or one outside [1, ONERF_METRICS_MAX_WINDOW], H or W <= window / 2 (reflect
 * padding is undefined there), H > 1048560, K outside [0, ONERF_METRICS_MAX_IDS], an id outside [0, 65535], a NULL image, record or
 * (with K > 0) pred_object, labels or ids_host, misaligned buffers.  Kernels only, no allocation and no host read:
 * CUDA-graph capturable.  The record's fp64 sums are added with atomics, so their last bits may depend on the CTA order.
 * ------------------------------------------------------------------------------------------- */
#define ONERF_METRICS_MAX_WINDOW 11
#define ONERF_METRICS_MAX_IDS 64

typedef struct onerf_metrics_args {
  int H, W;
  const float* pred_scene;              /* (H*W,3) */
  const float* pred_object;             /* (H*W,3), or NULL when n_ids = 0 */
  const float* gt;                      /* (H*W,3) */
  const uint8_t* valid;                 /* (H*W) or NULL */
  const uint16_t* labels;               /* (H*W), or NULL when n_ids = 0 */
  const int* ids_host;                  /* (n_ids,) host array */
  int n_ids;                            /* K */
  int window;                           /* odd, 1 .. ONERF_METRICS_MAX_WINDOW */
  double* record;                       /* ((K+1),3) */
  float* psnr_out;                      /* (F,K+1), finalize only */
  float* ssim_out;                      /* (F,K+1), finalize only */
} onerf_metrics_args;

int onerf_image_metrics(onerf_ctx* ctx, const onerf_metrics_args* args, void* stream);
int onerf_image_metrics_finalize(onerf_ctx* ctx, const onerf_metrics_args* args, int slot, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Depth errors of a held-out frame, for the scene and for each of K objects.  Inputs are float32, every sum is fp64.
 * s = scale.  A pixel is in column 0 when valid and gt > 0; it is also in column k >= 1 when labelled ids_host[k-1].
 * Column 0 reads pred_scene, column k reads pred_object (depth_instance).  Per pixel of a column:
 *   g = gt * s, d = clamp(pred * s, d_min, d_max) (a NaN pred stays NaN),
 * and the column's record row holds the eight sums
 *   n, sum |d - g| / g, sum (d - g)^2 / g, sum (d - g)^2, sum (ln d - ln g)^2,
 *   and the counts of max(d / g, g / d) < 1.25, < 1.25^2, < 1.25^3 (a NaN ratio adds NaN to each count).
 * The seven outputs (ONERF_DEPTH_METRICS order) are
 *   abs_rel = sum |d - g| / g / n, sq_rel = sum (d - g)^2 / g / n, rmse = sqrt(sum (d - g)^2 / n),
 *   rmse_log = sqrt(sum (ln d - ln g)^2 / n), delta_i = count_i / n.
 * An empty column gives NaN for all seven; a NaN prediction in a column makes all seven NaN.
 *
 * onerf_depth_metrics: adds one frame's sums to `record` ((K+1) x 8 doubles in the order above), which must hold zeros
 * (or an earlier part of the same frame) before the call.
 * onerf_depth_metrics_finalize: one launch that writes out[slot, :, :] ((F, K+1, 7) row-major float32; NULL: not
 * written) from the record and zeroes it.  Only n_ids, record and out are read.
 *   pred_scene, gt  (H*W) float32; pred_object (H*W) float32, NULL when K = 0
 *   valid           (H*W) uint8 0 / 1, or NULL: every pixel
 *   labels          (H*W) uint16, NULL when K = 0
 *   ids_host        K distinct ints in [0, 65535] (host array), 0 <= K <= ONERF_METRICS_MAX_IDS
 *   scale           finite and > 0; d_min, d_max finite with 0 < d_min < d_max
 * Refusals (ONERF_ERR_BAD_ARG): a NULL ctx or args, H or W < 1, H * W >= 2^40, K outside [0, ONERF_METRICS_MAX_IDS], an
 * id outside [0, 65535] or repeated, d_min <= 0 or d_min >= d_max, a non-finite or non-positive scale or depth bound, a
 * NULL pred_scene, gt or record or (with K > 0) pred_object, labels or ids_host, misaligned buffers.
 *
 * Instance-mask agreement of one object's opacity map (the object branch's OpacityLoss target), over the valid pixels:
 *   G = (labels == id), P = (opacity >= threshold) (float32 comparison),
 *   iou = |P & G| / |P | G| (NaN when P | G is empty), opacity_l1 = sum |opacity - [G]| / n_valid (NaN when no pixel
 *   is valid).
 * onerf_mask_metrics: adds the four sums |P & G|, |P | G|, sum |opacity - [G]| and n_valid (fp64) to row `column` of
 * `record` (K x 4 doubles, K = n_ids), which must hold zeros (or an earlier part of the same frame) there.
 * onerf_mask_metrics_finalize: one launch that writes iou_out[slot, :] and opacity_l1_out[slot, :] ((F, K) row-major
 * float32; either may be NULL: not written) from the record and zeroes it.  Only n_ids, record and the outputs are
 * read.
 *   opacity         (H*W) float32 (opacity_instance rendered with object id's code)
 *   valid           (H*W) uint8 0 / 1, or NULL: every pixel
 *   labels          (H*W) uint16
 *   id              in [0, 65535]; column in [0, K), 1 <= K <= ONERF_METRICS_MAX_IDS; threshold finite
 * Refusals (ONERF_ERR_BAD_ARG): a NULL ctx or args, H or W < 1, H * W >= 2^40, K outside [1, ONERF_METRICS_MAX_IDS],
 * column outside [0, K), an id outside [0, 65535], a non-finite threshold, a NULL opacity, labels or record, misaligned
 * buffers.
 *
 * All four are kernels only, with no allocation and no host read: CUDA-graph capturable.  Counts are exact (integers
 * below 2^53); the other fp64 sums are added with atomics, so their last bits may depend on the CTA order.
 * ------------------------------------------------------------------------------------------- */
#define ONERF_DEPTH_METRICS 7
#define ONERF_DEPTH_RECORD 8
#define ONERF_MASK_RECORD 4

typedef struct onerf_depth_metrics_args {
  int H, W;
  const float* pred_scene;              /* (H*W) */
  const float* pred_object;             /* (H*W), or NULL when n_ids = 0 */
  const float* gt;                      /* (H*W) */
  const uint8_t* valid;                 /* (H*W) or NULL */
  const uint16_t* labels;               /* (H*W), or NULL when n_ids = 0 */
  const int* ids_host;                  /* (n_ids,) host array */
  int n_ids;                            /* K */
  double scale;                         /* s: metres per stored depth unit */
  double d_min, d_max;                  /* clamp of the prediction, metres */
  double* record;                       /* ((K+1),8) */
  float* out;                           /* (F,K+1,7), finalize only */
} onerf_depth_metrics_args;

typedef struct onerf_mask_metrics_args {
  int H, W;
  const float* opacity;                 /* (H*W) */
  const uint8_t* valid;                 /* (H*W) or NULL */
  const uint16_t* labels;               /* (H*W) */
  int id;                               /* the object's label */
  int column;                           /* its row of the record, 0 .. n_ids-1 */
  int n_ids;                            /* K */
  float threshold;                      /* tau */
  double* record;                       /* (K,4) */
  float* iou_out;                       /* (F,K), finalize only */
  float* opacity_l1_out;                /* (F,K), finalize only */
} onerf_mask_metrics_args;

int onerf_depth_metrics(onerf_ctx* ctx, const onerf_depth_metrics_args* args, void* stream);
int onerf_depth_metrics_finalize(onerf_ctx* ctx, const onerf_depth_metrics_args* args, int slot, void* stream);
int onerf_mask_metrics(onerf_ctx* ctx, const onerf_mask_metrics_args* args, void* stream);
int onerf_mask_metrics_finalize(onerf_ctx* ctx, const onerf_mask_metrics_args* args, int slot, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Every object's own maps of a set of rays in one render: the object branch's decomposition (opacity, depth and colour of
 * each object, what OpacityLoss trains) for K object codes at once.  For K codes code_table[ids_host[k]], column k of
 * each object map is bit for bit the opacity_instance / depth_instance / rgb_instance that onerf_render_rays_fwd writes
 * when every ray carries that code (is_eval, perturb = 0, noise_std = 0, rays_in_bbox = 0: models/rendering.py's
 * render_rays(..., forward_instance=True, is_eval=True, perturb=0, noise_std=0, rays_in_bbox=False)), at the same
 * precision, and the scene maps are that render's scene maps.  In such a render the coarse depths, the scene branch,
 * its weights, the importance samples and each sample's encoding do not depend on the code, so per chunk and pass they
 * are computed once: ONERF_PREC_BF16 runs one tensor-core field launch that encodes each sample once and runs the
 * object branch once per code, then the scene branch; ONERF_PREC_FP32 runs the FFMA field once for the scene and once
 * per code for the object branch.  One compositing launch gives the scene maps, one more every object map.  A pass
 * runs the object branch only when one of its object maps is given, and the scene branch only when one of its scene
 * maps is given or its weights feed the fine samples (the coarse pass of a render with n_importance > 0); what runs
 * gives the same bits either way.
 *   render     rays (n_rays,8), n_rays, grid, packed_coarse / packed_fine, precision, n_samples, n_importance, use_disp,
 *              white_back, zero_last_delta; is_eval must be set, perturb and noise_std 0, rays_in_bbox 0, train_ws NULL.
 *              codes, forward_instance, the random buffers and the maps of onerf_render_args are not read.  workspace:
 *              >= onerf_render_instances_workspace_bytes(chunk_rays, n_ids, n_samples, n_importance) bytes, 256-byte
 *              aligned (0 for a bad shape): per chunk the field rows of the K codes and the scene, K per-ray-constant
 *              blocks, depths and weights.  Its size does not depend on the image.
 *   code_table (n_codes_table,64); ids_host: n_ids ints (host array), 1 <= n_ids <= ONERF_INSTANCES_MAX_CODES, each a
 *              row of the table; repeats are allowed (each is its own column).
 *   ray_begin, ray_end  the tile [ray_begin, ray_end) of the rays rendered, in chunks of chunk_rays rays.
 *   coarse, fine  tile-sized maps (N = ray_end - ray_begin rows): scene rgb (N,3), depth (N,), opacity (N,); object
 *              opacity and depth (N,K), rgb (N,K,3), K = n_ids.  Any may be NULL: it is not written.  fine maps need
 *              n_importance > 0.  4-byte aligned.
 * Every row depends on its ray only, never on chunk_rays or the tile bounds.  Refusals before any launch: a NULL ctx or
 * args, n_ids outside [1, 64], a NULL ids_host or code_table, an id outside the code table, is_eval off, perturb or
 * noise_std non-zero, a training workspace, a bad shape, a tile outside [0, n_rays], chunk_rays < 1, NULL rays or packed
 * weights, a NULL or misaligned grid buffer, an unknown precision, fine maps without a fine pass, a misaligned map, a
 * misaligned or undersized workspace (ONERF_ERR_BAD_ARG); rays_in_bbox set (the fine depths would then follow the
 * object's weights) and n_samples + n_importance > 2048 (ONERF_ERR_UNSUPPORTED).  Kernels only, no allocation and no
 * host read: CUDA-graph capturable.
 * ------------------------------------------------------------------------------------------- */
#define ONERF_INSTANCES_MAX_CODES 64

typedef struct onerf_instance_maps {
  float* rgb;                           /* (N,3) scene */
  float* depth;                         /* (N,) scene */
  float* opacity;                       /* (N,) scene */
  float* opacity_instance;              /* (N,K) */
  float* depth_instance;                /* (N,K) */
  float* rgb_instance;                  /* (N,K,3) */
} onerf_instance_maps;

typedef struct onerf_instances_args {
  onerf_render_args render;
  const float* code_table;              /* (n_codes_table,64) */
  int n_codes_table;
  const int* ids_host;                  /* (n_ids,) host array */
  int n_ids;                            /* K */
  int64_t ray_begin, ray_end;
  int chunk_rays;
  onerf_instance_maps coarse;
  onerf_instance_maps fine;             /* n_importance > 0 only */
} onerf_instances_args;

size_t onerf_render_instances_workspace_bytes(int chunk_rays, int n_codes, int n_samples, int n_importance);
int onerf_render_instances(onerf_ctx* ctx, const onerf_instances_args* args, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Every object rendered inside its own box, from a camera, in one call: the object evaluation of a dataset with
 * use_bbox (GenericDataset's test split clips each ray to the object's box and scores instance_mask * bbox_mask; the
 * validation render runs with rays_in_bbox, so the object's weights drive the importance samples).
 * For K boxes boxes_host[k] with code rows ids_host[k] (1 <= K <= 64, repeats allowed), object k's rays are
 * onerf_camera_rays(H, W, focal, c2w_host, &boxes_host[k], scale_factor, near, far) and hit_k that call's hit_out:
 *   hit pixel of object k: its opacity, depth and rgb (on white) of each pass are bit for bit the opacity_instance /
 *     depth_instance / rgb_instance of onerf_render_rays_fwd over those rays with code_table[ids_host[k]] on every ray,
 *     forward_instance, is_eval, rays_in_bbox = 1, perturb = 0, noise_std = 0, at the same precision;
 *   missed pixel of object k: opacity +0, depth +0, rgb 1, what the editing path's muted field gives.  (The reference's
 *     render evaluates such rays at z = 0 instead; its metrics exclude them through instance_mask * bbox_mask.)
 * Every map given is first set to the missed values.  The rows are the (object, pixel) pairs of the tile, object-major (row k * T + p is pixel p_begin + p of object k,
 * T = p_end - p_begin), processed chunk_rays rows at a time.  Per chunk: the rows' box-clipped rays and hit bits (the
 * camera-ray kernel's pixel ray and float64 slab test); the hit rows listed in row order and their rays gathered; then,
 * on the listed rows only and stopping at the device-side count, the coarse depths,
 * the object branch and its compositing with rays_in_bbox semantics, whose weights feed the importance sampler, and
 * the fine pass.  No scene branch runs.
 *   grid (NULL: plain PE model), packed_coarse / packed_fine (the latter iff n_importance > 0), precision, n_samples,
 *   n_importance, use_disp: as onerf_render_args.  H, W, focal, c2w_host (12 floats, host, row-major 3x4): the camera.
 *   boxes_host: n_boxes boxes (host array).  scale_factor: as onerf_camera_rays.  near, far: not read (every ray takes
 *   its near / far from its box, as onerf_camera_rays' rays with a box do); kept for the camera call's argument set.
 *   ids_host: n_boxes ints
 *   (host), each a row of code_table (n_codes_table,64), 16-byte aligned.
 *   pixel_begin, pixel_end: the tile [pixel_begin, pixel_end) of the H*W pixels (row-major).
 *   coarse, fine: tile-sized maps, T rows: opacity and depth (T,K), rgb (T,K,3); column k is object k.  Any may be NULL
 *   (not written); fine maps need n_importance > 0.  hit: (T,K) u8 or NULL.  4-byte aligned (any alignment for hit).
 *   workspace: >= onerf_render_boxes_workspace_bytes(chunk_rays, n_samples, n_importance) bytes, 256-byte aligned (0
 *   for a bad shape).  Its size depends on neither K nor the image.
 * Every row depends on its pixel and box only, never on chunk_rays or the tile.  Refusals before any launch: a NULL ctx
 * or args; n_boxes outside [1, 64]; a NULL boxes_host, ids_host or code_table, an id outside the code table; a
 * non-finite box entry, camera entry or scale_factor, H or W < 1, focal <= 0 or scale_factor <= 0; a tile
 * outside [0, H*W]; chunk_rays < 1; a bad shape; NULL packed weights; a NULL or misaligned grid buffer; an unknown
 * precision; fine maps without a fine pass; a misaligned code table or map; a misaligned or undersized workspace
 * (ONERF_ERR_BAD_ARG); n_importance > 0 with n_samples + n_importance > 2048, as onerf_render_rays_fwd
 * (ONERF_ERR_UNSUPPORTED).  Kernels only, no allocation and no
 * host read: CUDA-graph capturable.
 * ------------------------------------------------------------------------------------------- */
#define ONERF_BOXES_MAX 64

typedef struct onerf_box_maps {
  float* opacity;                       /* (T,K) */
  float* depth;                         /* (T,K) */
  float* rgb;                           /* (T,K,3) */
} onerf_box_maps;

typedef struct onerf_render_boxes_args {
  const onerf_grid* grid;               /* NULL -> plain PE model */
  const void* packed_coarse;
  const void* packed_fine;              /* required iff n_importance > 0 */
  int precision;                        /* onerf_precision */
  int n_samples, n_importance;
  int use_disp;
  int H, W;
  float focal;
  const float* c2w_host;                /* 12 floats (host) */
  const onerf_box_host* boxes_host;     /* (n_boxes,) host array */
  int n_boxes;                          /* K */
  double scale_factor, near, far;
  const int* ids_host;                  /* (n_boxes,) host array */
  const float* code_table;              /* (n_codes_table,64) */
  int n_codes_table;
  int64_t pixel_begin, pixel_end;
  int chunk_rays;
  onerf_box_maps coarse;
  onerf_box_maps fine;                  /* n_importance > 0 only */
  uint8_t* hit;                         /* (T,K) or NULL */
  void* workspace;
  size_t workspace_bytes;
} onerf_render_boxes_args;

size_t onerf_render_boxes_workspace_bytes(int chunk_rays, int n_samples, int n_importance);
int onerf_render_boxes(onerf_ctx* ctx, const onerf_render_boxes_args* args, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* ONERF_EXT_H_ */
