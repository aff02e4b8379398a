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

#ifdef __cplusplus
}
#endif
#endif /* ONERF_EXT_H_ */
