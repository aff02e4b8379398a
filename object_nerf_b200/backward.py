"""Training path: render_rays() as a torch.autograd.Function whose backward runs on the library's CUDA kernels
(reference: loss.backward() through models/rendering.py, models/nerf_model.py, models/embedding_helper.py and
models/code_library.py; SURVEY.md §8 row a14).

Two arithmetics, selected by `precision`:
  bf16 (default)  RenderRaysTcFn: ONE C call forward (onerf_render_rays_fwd with a training workspace: the tensor-core forward
                  keeps every layer's activations as bf16 operand tiles) and ONE C call backward (onerf_render_rays_bwd:
                  wgmma input-gradient chain, weight-gradient and encoding-gradient GEMMs).  Voxel and plain-PE model;
                  the plain model has no voxel table and so no encoding gradient.
  fp32            RenderRaysFn below: the verification path (FFMA forward re-run with fp32 activation dump, fp32 GEMMs).

Gradients are produced for exactly what the reference trains: the 2 x 40 nn.Linear tensors of the coarse and fine
ObjectNeRF, the per-ray object codes (-> CodeLibrary's embedding table through autograd of the lookup) and the
voxel feature table.  No gradient flows to rays or depths (the importance samples are detached in the reference,
models/rendering.py:307).

Layout of the computation (all fp32, chunked over rays so that a chunk holds <= CHUNK_SAMPLES samples):
  forward (saved):   depths, per-sample fields (rgb, sigma) of both branches, noise buffers
  backward, per pass (fine then coarse):
    onerf_composite_bwd            d maps -> d(rgb, sigma) per sample and branch
    per chunk:  onerf_field_fwd (FFMA kernel, activations dumped as [samples x width] matrices)
                then per layer, last to first:  dZ = dH * act'(H)  (onerf_leaky_bwd / onerf_head_bwd)
                                                dW += dZ^T In, db += colsum(dZ), dIn = dZ W   (onerf_gemm, onerf_colsum)
                per-ray-constant columns (direction encoding, object code) use per-ray sums (onerf_segment_sum)
                onerf_encode_bwd   dX -> scatter-add into the voxel table gradient
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Optional

import torch

from . import _lib, engine

CHUNK_SAMPLES = 65536
ACT_WIDTHS_TAIL = [256] * 8 + [256, 128] + [128] * 4 + [128, 64]   # after X


def _p(t, col=0):
    return t.data_ptr() + 4 * col


class _Ops:
    """Thin wrappers over the backward C ABI on the current stream."""

    def __init__(self, dev):
        self.lib = _lib.load()
        self.ctx = _lib.ctx(dev)
        self.dev = dev

    def gemm(self, A, lda, trans_a, B, ldb, Cm, ldc, M, N, K, accumulate):
        _lib.check(self.lib.onerf_gemm(self.ctx, A, lda, int(trans_a), B, ldb, Cm, ldc, M, N, K, int(accumulate), _lib.stream()))

    def leaky_bwd(self, d, ld_d, h, ld_h, rows, cols):
        _lib.check(self.lib.onerf_leaky_bwd(self.ctx, d, ld_d, h, ld_h, rows, cols, _lib.stream()))

    def head_bwd(self, dfield, field, dA, n):
        _lib.check(self.lib.onerf_head_bwd(self.ctx, dfield, field, dA, n, _lib.stream()))

    def segment_sum(self, src, ld_in, out, ld_out, n_rays, S, cols):
        _lib.check(self.lib.onerf_segment_sum(self.ctx, src, ld_in, out, ld_out, n_rays, S, cols, _lib.stream()))

    def colsum(self, src, ld, rows, cols, out):
        _lib.check(self.lib.onerf_colsum(self.ctx, src, ld, rows, cols, out, _lib.stream()))

    def dir_encode(self, rays, n, out):
        _lib.check(self.lib.onerf_dir_encode(self.ctx, rays, n, out, _lib.stream()))


def composite_backward(z, scene, obj, depth_scene, grads, noise_std, white_back, is_eval, zero_last_delta,
                       frustum_bound_th, pass_through_mask, noise_scene, noise_obj, seed=0):
    """grads: dict with optional rgb, depth, opacity, rgb_instance, depth_instance, opacity_instance (N,..) tensors.
    With noise_std > 0 and no noise buffer the noise is re-drawn from `seed`, as the forward (engine.composite) drew it."""
    n, s = z.shape
    dev = z.device
    dscene = torch.empty(n, s, 4, dtype=torch.float32, device=dev)
    dobj = torch.empty(n, s, 4, dtype=torch.float32, device=dev) if obj is not None else None
    a = _lib.CompositeArgs()
    a.z, a.scene, a.obj = z.data_ptr(), scene.data_ptr(), _lib.ptr(obj)
    a.n_rays, a.n_samples = n, s
    a.noise_std = float(noise_std)
    a.noise_scene, a.noise_obj, a.seed = _lib.ptr(noise_scene), _lib.ptr(noise_obj), seed
    a.white_back, a.is_eval = int(bool(white_back)), int(bool(is_eval))
    a.zero_last_delta, a.rays_in_bbox = int(bool(zero_last_delta)), 0
    a.frustum_bound_th = float(frustum_bound_th)
    ptm = pass_through_mask.reshape(-1).to(torch.uint8).contiguous() if pass_through_mask is not None else None
    a.pass_through_mask = _lib.ptr(ptm)
    g = {k: (v.contiguous().float() if v is not None else None) for k, v in grads.items()}
    _lib.check(_lib.load().onerf_composite_bwd(
        _lib.ctx(dev), C.byref(a), _lib.ptr(depth_scene), _lib.ptr(g.get("rgb")), _lib.ptr(g.get("depth")),
        _lib.ptr(g.get("opacity")), _lib.ptr(g.get("rgb_instance")), _lib.ptr(g.get("depth_instance")),
        _lib.ptr(g.get("opacity_instance")), dscene.data_ptr(), _lib.ptr(dobj), _lib.stream()))
    return dscene, dobj


def field_backward(model, emb_xyz, rays, z, codes, dscene, dobj, want_object=True):
    """Gradient of the fused encode + MLP.  Returns (list of 20 (dW, db), d_codes (N,64) | None, table_grad | None)."""
    dev = rays.device
    ops = _Ops(dev)
    use_voxel = hasattr(emb_xyz, "voxel_idx_map")
    grid = engine.GridBuffers.from_module(emb_xyz) if use_voxel else None
    packed = engine.packed_for(model, use_voxel, fresh=True)
    lin = engine.model_linears(model)
    W = [engine._f32(w.detach()) for w, _ in lin]
    dWb = [(torch.zeros_like(w, dtype=torch.float32), torch.zeros_like(b, dtype=torch.float32)) for w, b in lin]
    n, s = z.shape
    xin, ovx = (271, 104) if use_voxel else (63, 0)
    KO = 384 if use_voxel else 64
    oin = xin + ovx + 64
    d_codes = torch.zeros(n, 64, dtype=torch.float32, device=dev) if want_object else None
    table_grad = torch.zeros_like(emb_xyz.embedding_space_ftr.weight, dtype=torch.float32) if use_voxel else None
    rays_per_chunk = max(1, CHUNK_SAMPLES // s)
    f = lambda *shape: torch.empty(*shape, dtype=torch.float32, device=dev)
    for r0 in range(0, n, rays_per_chunk):
        r1 = min(n, r0 + rays_per_chunk)
        R, B = r1 - r0, (r1 - r0) * s
        rays_c, z_c = rays[r0:r1].contiguous(), z[r0:r1].contiguous()
        codes_c = codes[r0:r1].contiguous() if want_object else None
        # ---- forward re-run with activation dump ----
        acts = [f(B, KO)] + [f(B, wd) for wd in ACT_WIDTHS_TAIL]
        act_ptrs = (C.c_void_p * 17)(*[t.data_ptr() for t in acts])
        scene_c, obj_c = engine.field(rays_c, z_c, packed, grid, codes=codes_c, want_scene=True, want_object=want_object,
                                      precision="fp32", activations=act_ptrs)
        X, Hs, Hfin, Hdir = acts[0], acts[1:9], acts[9], acts[10]
        Ho, Hofin, Hodir = acts[11:15], acts[15], acts[16]
        dX = torch.zeros(B, KO, dtype=torch.float32, device=dev)
        pe = f(R, 27)
        ops.dir_encode(rays_c.data_ptr(), R, pe.data_ptr())
        bufA, bufB = f(B, 256), f(B, 256)
        rs = f(R, 128)
        dA = f(B, 4)

        def linear_bwd(dZ, ldz, n_out, idx, inputs, d_inputs):
            """dZ [B x n_out] (ld ldz).  inputs: list of (In ptr, ld_in, width, col_off in W) for dW; d_inputs: list of
            (dst ptr, ld_dst, width, col_off in W, accumulate) for dIn."""
            dW, db = dWb[idx]
            ldw = W[idx].shape[1]
            ops.colsum(dZ, ldz, B, n_out, db.data_ptr())
            for (src, ld_in, width, col) in inputs:
                ops.gemm(dZ, ldz, 1, src, ld_in, _p(dW, col), ldw, n_out, width, B, True)
            for (dst, ld_dst, width, col, acc) in d_inputs:
                ops.gemm(dZ, ldz, 0, _p(W[idx], col), ldw, dst, ld_dst, B, width, n_out, acc)

        def ray_columns(dZ, ldz, n_out, idx, col, per_ray, width, d_per_ray=None):
            """Columns of W[idx] fed by a per-ray constant [R x width]: dW[:, col:col+width] += (sum_s dZ)^T per_ray."""
            dW, _ = dWb[idx]
            ldw = W[idx].shape[1]
            ops.segment_sum(dZ, ldz, rs.data_ptr(), 128, R, s, n_out)
            ops.gemm(rs.data_ptr(), 128, 1, per_ray.data_ptr(), width, _p(dW, col), ldw, n_out, width, R, True)
            if d_per_ray is not None:
                ops.gemm(rs.data_ptr(), 128, 0, _p(W[idx], col), ldw, d_per_ray, width, R, width, n_out, True)

        # ================= scene branch (models/nerf_model.py:97-121) =================
        ops.head_bwd(dscene[r0:r1].data_ptr(), scene_c.data_ptr(), dA.data_ptr(), B)
        # rgb head (idx 11), input = dir-layer output
        linear_bwd(dA.data_ptr(), 4, 3, 11, [(Hdir.data_ptr(), 128, 128, 0)], [(bufA.data_ptr(), 256, 128, 0, False)])
        ops.leaky_bwd(bufA.data_ptr(), 256, Hdir.data_ptr(), 128, B, 128)
        # dir layer (idx 10): [final 256 | dir 27]
        linear_bwd(bufA.data_ptr(), 256, 128, 10, [(Hfin.data_ptr(), 256, 256, 0)], [(bufB.data_ptr(), 256, 256, 0, False)])
        ray_columns(bufA.data_ptr(), 256, 128, 10, 256, pe, 27)
        # final layer (idx 9), no activation; input = h8
        linear_bwd(bufB.data_ptr(), 256, 256, 9, [(Hs[7].data_ptr(), 256, 256, 0)], [(bufA.data_ptr(), 256, 256, 0, False)])
        # sigma head (idx 8): adds to dH8
        linear_bwd(_p(dA, 3), 4, 1, 8, [(Hs[7].data_ptr(), 256, 256, 0)], [(bufA.data_ptr(), 256, 256, 0, True)])
        dH, other = bufA, bufB
        for l in range(7, -1, -1):
            ops.leaky_bwd(dH.data_ptr(), 256, Hs[l].data_ptr(), 256, B, 256)
            if l == 0:
                linear_bwd(dH.data_ptr(), 256, 256, 0, [(X.data_ptr(), KO, xin, 0)], [(dX.data_ptr(), KO, xin, 0, True)])
            elif l == 4:
                linear_bwd(dH.data_ptr(), 256, 256, 4, [(X.data_ptr(), KO, xin, 0), (Hs[3].data_ptr(), 256, 256, xin)],
                           [(dX.data_ptr(), KO, xin, 0, True), (other.data_ptr(), 256, 256, xin, False)])
            else:
                linear_bwd(dH.data_ptr(), 256, 256, l, [(Hs[l - 1].data_ptr(), 256, 256, 0)],
                           [(other.data_ptr(), 256, 256, 0, False)])
            dH, other = other, dH
        # ================= object branch (models/nerf_model.py:123-152) =================
        if want_object:
            ops.head_bwd(dobj[r0:r1].data_ptr(), obj_c.data_ptr(), dA.data_ptr(), B)
            linear_bwd(dA.data_ptr(), 4, 3, 19, [(Hodir.data_ptr(), 64, 64, 0)], [(bufA.data_ptr(), 256, 64, 0, False)])
            ops.leaky_bwd(bufA.data_ptr(), 256, Hodir.data_ptr(), 64, B, 64)
            linear_bwd(bufA.data_ptr(), 256, 64, 18, [(Hofin.data_ptr(), 128, 128, 0)], [(bufB.data_ptr(), 256, 128, 0, False)])
            ray_columns(bufA.data_ptr(), 256, 64, 18, 128, pe, 27)
            linear_bwd(bufB.data_ptr(), 256, 128, 17, [(Ho[3].data_ptr(), 128, 128, 0)], [(bufA.data_ptr(), 256, 128, 0, False)])
            linear_bwd(_p(dA, 3), 4, 1, 16, [(Ho[3].data_ptr(), 128, 128, 0)], [(bufA.data_ptr(), 256, 128, 0, True)])
            dH, other = bufA, bufB
            dcodes_c = d_codes[r0:r1]
            for l in range(3, -1, -1):
                ops.leaky_bwd(dH.data_ptr(), 256, Ho[l].data_ptr(), 128, B, 128)
                idx = 12 + l
                if l in (0, 2):
                    ins = [(X.data_ptr(), KO, xin, 0)]
                    outs = [(dX.data_ptr(), KO, xin, 0, True)]
                    if ovx:
                        ins.append((_p(X, 272), KO, ovx, xin))
                        outs.append((_p(dX, 272), KO, ovx, xin, True))
                    if l == 2:
                        ins.append((Ho[1].data_ptr(), 128, 128, oin))
                        outs.append((other.data_ptr(), 256, 128, oin, False))
                    linear_bwd(dH.data_ptr(), 256, 128, idx, ins, outs)
                    ray_columns(dH.data_ptr(), 256, 128, idx, xin + ovx, codes_c, 64, d_per_ray=dcodes_c.data_ptr())
                else:
                    linear_bwd(dH.data_ptr(), 256, 128, idx, [(Ho[l - 1].data_ptr(), 128, 128, 0)],
                               [(other.data_ptr(), 256, 128, 0, False)])
                dH, other = other, dH
        # ================= encoding (models/embedding_helper.py:354-409) =================
        if use_voxel:
            _lib.check(_lib.load().onerf_encode_bwd(_lib.ctx(dev), C.byref(grid.c), rays_c.data_ptr(), z_c.data_ptr(), R, s,
                                                    X.data_ptr(), dX.data_ptr(), KO, 0, B, table_grad.data_ptr(),
                                                    _lib.stream()))
    return dWb, d_codes, table_grad


class RenderRaysFn(torch.autograd.Function):
    """Differentiable render_rays.  Inputs after `cfg`: rays, codes, then the flat list of trainable tensors
    (voxel table, coarse 40, fine 40); see rendering.render_rays for how it is called."""

    @staticmethod
    def forward(ctx, cfg, rays, codes, *params):
        from . import rendering
        with torch.no_grad():
            out, saved = rendering._render_forward(cfg, rays, codes, keep=True)
        ctx.cfg, ctx.saved = cfg, saved
        ctx.n_params = len(params)
        ctx.save_for_backward(rays, codes if codes is not None else torch.empty(0, device=rays.device))
        keys = sorted(out)
        ctx.keys = keys
        tensors = tuple(out[k] for k in keys)
        ctx.mark_non_differentiable(*[t for k, t in zip(keys, tensors) if k.startswith(("weights_", "z_vals_"))])
        return tensors

    @staticmethod
    def backward(ctx, *gouts):
        cfg, saved = ctx.cfg, ctx.saved
        rays, codes = ctx.saved_tensors
        codes = codes if codes.numel() else None
        g = {k: v for k, v in zip(ctx.keys, gouts)}
        fi = cfg["forward_instance"]
        d_codes_total = torch.zeros_like(codes, dtype=torch.float32) if (codes is not None and fi) else None
        table_total = None
        model_grads: Dict[str, list] = {}
        for typ in ("fine", "coarse"):
            if typ not in saved:
                continue
            sv = saved[typ]
            grads = {name: g.get(f"{name}_{typ}") for name in ("rgb", "depth", "opacity", "rgb_instance", "depth_instance",
                                                               "opacity_instance")}
            if all(v is None for v in grads.values()):
                continue
            dscene, dobj = composite_backward(sv["z"], sv["scene"], sv["obj"], sv["depth"], grads, cfg["noise_std"],
                                              cfg["white_back"], cfg["is_eval"], cfg["zero_last_delta"],
                                              cfg["frustum_bound_th"], cfg["pass_through_mask"], sv["noise_scene"],
                                              sv["noise_obj"])
            dWb, d_codes, table_grad = field_backward(cfg["models"][typ], cfg["embeddings"]["xyz"], rays, sv["z"], codes,
                                                      dscene, dobj, want_object=fi)
            model_grads[typ] = dWb
            if d_codes is not None:
                d_codes_total += d_codes
            if table_grad is not None:
                table_total = table_grad if table_total is None else table_total + table_grad
        # order of `params` as assembled by rendering.render_rays: [table] + coarse 40 + fine 40
        flat: List[Optional[torch.Tensor]] = []
        if cfg["has_table"]:
            flat.append(table_total)
        for typ in cfg["model_order"]:
            gw = model_grads.get(typ)
            for i in range(20):
                flat += [gw[i][0], gw[i][1]] if gw is not None else [None, None]
        assert len(flat) == ctx.n_params
        return (None, None, d_codes_total) + tuple(flat)


# ------------------------------------------------------------------------------------------------
# tensor-core training path
# ------------------------------------------------------------------------------------------------
class _WsPool:
    """Training workspaces are large (2.6 MB per ray at 64 + 128 samples): keep them across steps.  A workspace is leased
    to one autograd graph (forward -> backward) and returns to the pool when that graph is released."""

    def __init__(self):
        self.free = {}

    def take(self, nbytes, dev):
        lst = self.free.setdefault((nbytes, dev), [])
        if lst:
            return lst.pop()
        t = torch.empty(nbytes + 1024, dtype=torch.uint8, device=dev)
        off = (-t.data_ptr()) % 1024
        return t[off:off + nbytes]

    def give(self, t):
        lst = self.free.setdefault((t.numel(), t.device), [])
        if len(lst) < 2:
            lst.append(t)


_pool = _WsPool()


class _Lease:
    def __init__(self, t):
        self.t = t

    def __del__(self):
        try:
            _pool.give(self.t)
        except Exception:
            pass


class RenderRaysTcFn(torch.autograd.Function):
    """Differentiable render_rays on the tensor cores.  Inputs after `cfg`: rays, codes, then the flat list of trainable
    tensors ([voxel table, voxel model only] + coarse 40 + fine 40), as assembled by rendering.render_rays."""

    @staticmethod
    def forward(ctx, cfg, rays, codes, *params):
        lib = _lib.load()
        dev = rays.device
        emb = cfg["embeddings"]["xyz"]
        n = rays.shape[0]
        ns, ni = cfg["N_samples"], cfg["N_importance"]
        fi = cfg["forward_instance"]
        rand = cfg["rand"]
        use_voxel = cfg["has_table"]
        f = lambda *shape: torch.empty(*shape, dtype=torch.float32, device=dev)
        grid = engine.GridBuffers.from_module(emb) if use_voxel else None
        keep = [rays, grid]
        a = _lib.RenderArgs()
        packed, lins = {}, {}
        for typ in cfg["model_order"]:
            lins[typ] = engine.model_linears(cfg["models"][typ])
            packed[typ] = engine.packed_for(cfg["models"][typ], use_voxel, fresh=True)
        maps = {}
        for typ, s in (("coarse", ns), ("fine", ns + ni)):
            if typ == "fine" and ni == 0:
                continue
            m = dict(weights=f(n, s), opacity=f(n), z_vals=f(n, s), rgb=f(n, 3), depth=f(n))
            if fi:
                m.update(rgb_instance=f(n, 3), depth_instance=f(n), opacity_instance=f(n))
            maps[typ] = m
            cm = getattr(a, typ)
            for k, v in m.items():
                setattr(cm, k, v.data_ptr())
        ws_bytes = lib.onerf_render_rays_workspace_bytes(n, ns, ni)
        workspace = torch.empty(max(ws_bytes, 256), dtype=torch.uint8, device=dev)
        tws_bytes = lib.onerf_train_workspace_bytes(int(use_voxel), n, ns, ni)
        lease = _Lease(_pool.take(tws_bytes, dev))
        codes_c = engine._f32(codes.detach()) if (codes is not None and fi) else None
        mask = cfg["pass_through_mask"]
        mask = mask.reshape(-1).to(torch.uint8).contiguous() if mask is not None else None
        opt = {k: (engine._f32(rand[k]) if rand.get(k) is not None else None)
               for k in ("jitter", "u", "noise_scene_coarse", "noise_obj_coarse", "noise_scene_fine", "noise_obj_fine")}
        keep += [codes_c, mask, opt, workspace, packed]
        a.rays, a.codes = rays.data_ptr(), _lib.ptr(codes_c)
        a.n_rays, a.n_samples, a.n_importance = n, ns, ni
        a.grid = C.pointer(grid.c) if use_voxel else None
        a.packed_coarse = packed["coarse"].data_ptr()
        a.packed_fine = packed["fine"].data_ptr() if ni > 0 else None
        a.precision = _lib.PREC_BF16
        seed = engine.new_seed() if (cfg["perturb"] > 0 or cfg["noise_std"] > 0) else 0
        a.use_disp, a.perturb, a.noise_std, a.seed = int(cfg["use_disp"]), cfg["perturb"], cfg["noise_std"], seed
        a.jitter, a.u = _lib.ptr(opt["jitter"]), _lib.ptr(opt["u"])
        a.noise_scene_coarse, a.noise_obj_coarse = _lib.ptr(opt["noise_scene_coarse"]), _lib.ptr(opt["noise_obj_coarse"])
        a.noise_scene_fine, a.noise_obj_fine = _lib.ptr(opt["noise_scene_fine"]), _lib.ptr(opt["noise_obj_fine"])
        a.white_back, a.forward_instance, a.is_eval = int(cfg["white_back"]), int(fi), int(cfg["is_eval"])
        a.zero_last_delta, a.rays_in_bbox = int(cfg["zero_last_delta"]), int(cfg["rays_in_bbox"])
        a.frustum_bound_th = cfg["frustum_bound_th"]
        a.pass_through_mask = _lib.ptr(mask)
        a.workspace, a.workspace_bytes = workspace.data_ptr(), workspace.numel()
        a.train_ws, a.train_ws_bytes = lease.t.data_ptr(), lease.t.numel()
        with torch.cuda.device(dev):
            _lib.check(lib.onerf_render_rays_fwd(_lib.ctx(dev), C.byref(a), _lib.stream()))
        out = {f"{k}_{typ}": v for typ, m in maps.items() for k, v in m.items()}
        ctx.args, ctx.keep, ctx.lease, ctx.lins, ctx.cfg = a, keep, lease, lins, cfg
        ctx.n_params = len(params)
        ctx.has_codes = codes_c is not None
        keys = sorted(out)
        ctx.keys = keys
        tensors = tuple(out[k] for k in keys)
        ctx.mark_non_differentiable(*[t for k, t in zip(keys, tensors) if k.startswith(("weights_", "z_vals_"))])
        # the backward reads the forward's maps (depths, scene depth) through the raw pointers in `a`: keep the tensors
        # alive (a caller may drop the result dict right after the loss; non-differentiable outputs have no other owner)
        ctx.save_for_backward(*tensors)
        return tensors

    @staticmethod
    def backward(ctx, *gouts):
        lib = _lib.load()
        a, cfg = ctx.args, ctx.cfg
        _alive = ctx.saved_tensors  # noqa: F841
        dev = ctx.keep[0].device
        g = {k: (v.contiguous().float() if v is not None else None) for k, v in zip(ctx.keys, gouts)}
        b = _lib.RenderBwdArgs()
        keep = [g]
        for typ in cfg["model_order"]:
            mg = getattr(b, typ)
            for name in ("rgb", "depth", "opacity", "rgb_instance", "depth_instance", "opacity_instance"):
                setattr(mg, name, _lib.ptr(g.get(f"{name}_{typ}")))
        grads = {}
        for typ in cfg["model_order"]:
            lin = ctx.lins[typ]
            ws = [engine._f32(w.detach()) for w, _ in lin]
            sizes = [t.numel() for pair in lin for t in pair]
            flat = torch.zeros(sum(sizes), dtype=torch.float32, device=dev)   # one fill for the 40 gradient tensors
            views, o = [], 0
            for (w, bb) in lin:
                views.append((flat[o:o + w.numel()].view_as(w), flat[o + w.numel():o + w.numel() + bb.numel()].view_as(bb)))
                o += w.numel() + bb.numel()
            grads[typ] = views
            Wp = (C.c_void_p * 20)(*[t.data_ptr() for t in ws])
            dWp = (C.c_void_p * 20)(*[v[0].data_ptr() for v in views])
            dbp = (C.c_void_p * 20)(*[v[1].data_ptr() for v in views])
            keep += [ws, Wp, dWp, dbp]
            setattr(b, "W_" + typ, Wp)
            setattr(b, "dW_" + typ, dWp)
            setattr(b, "db_" + typ, dbp)
        d_codes = torch.zeros(a.n_rays, 64, dtype=torch.float32, device=dev) if ctx.has_codes else None
        table_grad = None
        if cfg["has_table"]:
            table_grad = torch.zeros_like(cfg["embeddings"]["xyz"].embedding_space_ftr.weight, dtype=torch.float32)
        b.d_codes, b.table_grad = _lib.ptr(d_codes), _lib.ptr(table_grad)
        with torch.cuda.device(dev):
            _lib.check(lib.onerf_render_rays_bwd(_lib.ctx(dev), C.byref(a), C.byref(b), _lib.stream()))
        flat_out: List[Optional[torch.Tensor]] = []
        if cfg["has_table"]:
            flat_out.append(table_grad)
        for typ in cfg["model_order"]:
            for w, bb in grads[typ]:
                flat_out += [w, bb]
        assert len(flat_out) == ctx.n_params
        ctx.lease = None     # the workspace goes back to the pool
        return (None, None, d_codes) + tuple(flat_out)
