// Layout of the training workspace of onerf_render_rays_fwd / onerf_render_rays_bwd (one caller-owned blob).
#pragma once
#include "../../include/onerf.h"
#include "layout.h"

// The model a training call trains: voxel when it carries a grid, plain PE otherwise.  The forward and the backward
// both derive the workspace layout from it.
static inline int onerf_train_use_voxel(const onerf_render_args* a) { return a->grid ? 1 : 0; }

struct TrainWs {
  int64_t tl_coarse, tl_fine;                   // field training workspaces (layout.h: TrainLayout) of the two passes
  int64_t scene_c, obj_c, scene_f, obj_f;       // per-sample fields (rgb, sigma) of both passes, kept for the backward
  int64_t dscene, dobj, dA_s, dA_o;             // per-sample gradients (one pass at a time)
  int64_t rs, pe;                               // per-ray sums (N,448), PE4 of the directions (N,27)
  int64_t gk;                                   // kernel-layout gradient buffer (one pass at a time)
  int64_t total;
};

static inline TrainWs onerf_make_train_ws(int use_voxel, int n_rays, int n_samples, int n_importance) {
  TrainWs W;
  int64_t o = 0;
  auto take = [&](int64_t bytes) { int64_t r = o; o += (bytes + 1023) & ~1023ll; return r; };
  const int64_t Bc = (int64_t)n_rays * n_samples, Bf = (int64_t)n_rays * (n_samples + n_importance);
  W.tl_coarse = take(onerf_make_train_layout(use_voxel, Bc).total_bytes);
  W.tl_fine = take(n_importance > 0 ? onerf_make_train_layout(use_voxel, Bf).total_bytes : 0);
  W.scene_c = take(Bc * 16); W.obj_c = take(Bc * 16);
  W.scene_f = take(Bf * 16); W.obj_f = take(Bf * 16);
  W.dscene = take(Bf * 16); W.dobj = take(Bf * 16); W.dA_s = take(Bf * 16); W.dA_o = take(Bf * 16);
  W.rs = take((int64_t)n_rays * ONERF_RAY_CONST_FLOATS * 4);
  W.pe = take((int64_t)n_rays * 27 * 4);
  W.gk = take(onerf_make_grad_layout(use_voxel).total_floats * 4);
  W.total = o;
  return W;
}
