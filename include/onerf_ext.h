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

#ifdef __cplusplus
}
#endif
#endif /* ONERF_EXT_H_ */
