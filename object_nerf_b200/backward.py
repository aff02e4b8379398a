"""Training path: render_rays() as a torch.autograd.Function whose backward runs on the library's CUDA kernels
(reference: loss.backward() through models/rendering.py, models/nerf_model.py, models/embedding_helper.py and
models/code_library.py; SURVEY.md §8 row a14).

RenderRaysFn makes two C calls: the forward is onerf_render_rays_fwd with a training workspace (engine.RenderPlan), the
backward onerf_render_rays_bwd.  The precision only selects the kernels inside them:
  bf16 (default)  the tensor-core forward keeps every layer's activations as bf16 operand tiles; the backward runs the
                  wgmma input-gradient chain, weight-gradient and encoding-gradient GEMMs.
  fp32            the verification arithmetic: the same two calls with the FFMA kernels and fp32 GEMMs (the backward
                  re-runs the FFMA forward chunk by chunk with its activation dump, then goes layer by layer).
Voxel and plain-PE model alike; the plain model has no voxel table and so no encoding gradient.

Gradients are produced for exactly what the reference trains: the 2 x 40 nn.Linear tensors of the coarse and fine
ObjectNeRF, the per-ray object codes (-> CodeLibrary's embedding table through autograd of the lookup) and the
voxel feature table.  No gradient flows to rays or depths (the importance samples are detached in the reference,
models/rendering.py:307).
"""
from __future__ import annotations

import ctypes as C
from typing import List, Optional

import torch

from . import _lib, engine

# the compositing backward's stage wrapper lives in engine beside composite(); this name keeps existing callers working
composite_backward = engine.composite_bwd


class _WsPool:
    """Training workspaces are large (2.6 MB per ray at 64 + 128 samples): keep them across steps.  A workspace is leased
    to one autograd graph (forward -> backward) and returns to the pool when that graph is released."""

    def __init__(self):
        self.free = {}

    def take(self, nbytes, dev):
        lst = self.free.setdefault((nbytes, dev), [])
        return lst.pop() if lst else engine.aligned_bytes(nbytes, dev)

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


class RenderRaysFn(torch.autograd.Function):
    """Differentiable render_rays.  Inputs after `cfg`: rays, codes, then the flat list of trainable tensors
    ([voxel table, voxel model only] + coarse 40 + fine 40), as assembled by rendering.render_rays."""

    @staticmethod
    def forward(ctx, cfg, rays, codes, *params):
        lib = _lib.load()
        dev = rays.device
        n = rays.shape[0]
        ns, ni = cfg["N_samples"], cfg["N_importance"]
        use_voxel = cfg["has_table"]
        prec = engine.PRECISIONS[cfg["precision"]]
        grid = engine.GridBuffers.from_module(cfg["embeddings"]["xyz"]) if use_voxel else None
        lins = {typ: engine.model_linears(cfg["models"][typ]) for typ in cfg["model_order"]}
        packed = {typ: engine.packed_for(cfg["models"][typ], use_voxel, fresh=True) for typ in cfg["model_order"]}
        lease = _Lease(_pool.take(lib.onerf_train_workspace_bytes_prec(prec, int(use_voxel), n, ns, ni), dev))
        seed = engine.new_seed() if (cfg["perturb"] > 0 or cfg["noise_std"] > 0) else 0
        plan = engine.RenderPlan(
            rays, packed["coarse"], packed.get("fine"), grid, codes=codes.detach() if codes is not None else None,
            n_samples=ns, n_importance=ni,
            use_disp=cfg["use_disp"], perturb=cfg["perturb"], noise_std=cfg["noise_std"], white_back=cfg["white_back"],
            forward_instance=cfg["forward_instance"], is_eval=cfg["is_eval"], zero_last_delta=cfg["zero_last_delta"],
            rays_in_bbox=cfg["rays_in_bbox"], frustum_bound_th=cfg["frustum_bound_th"],
            pass_through_mask=cfg["pass_through_mask"], precision=cfg["precision"], seed=seed, rand=cfg["rand"],
            train_ws=lease.t)
        out = plan.run()
        # the argument block and what it points into, but not the plan's output maps: outputs held by ctx would form a
        # reference cycle through their grad_fn and keep every step's buffers alive until the garbage collector runs
        ctx.args, ctx.keep, ctx.lease, ctx.lins, ctx.cfg = plan.args, (plan._keep, plan.workspace), lease, lins, cfg
        ctx.n_params = len(params)
        ctx.has_codes = codes is not None and cfg["forward_instance"]
        keys = sorted(out)
        ctx.keys = keys
        tensors = tuple(out[k] for k in keys)
        ctx.mark_non_differentiable(*[t for k, t in zip(keys, tensors) if k.startswith(("weights_", "z_vals_"))])
        # the backward reads the forward's maps (depths, scene depth) through the raw pointers in the argument block:
        # keep the tensors alive (a caller may drop the result dict right after the loss; non-differentiable outputs
        # have no other owner)
        ctx.save_for_backward(*tensors)
        return tensors

    @staticmethod
    def backward(ctx, *gouts):
        a, cfg = ctx.args, ctx.cfg
        _alive = ctx.saved_tensors  # noqa: F841
        dev = ctx.keep[1].device
        g = {k: (v.contiguous().float() if v is not None else None) for k, v in zip(ctx.keys, gouts)}
        b = _lib.RenderBwdArgs()
        keep = [g]
        for typ in cfg["model_order"]:
            mg = getattr(b, typ)
            for name in ("rgb", "depth", "opacity", "rgb_instance", "depth_instance", "opacity_instance"):
                setattr(mg, name, _lib.ptr(g.get(f"{name}_{typ}")))
        grads = {}
        for typ in cfg["model_order"]:
            lin = [(engine._f32(w.detach()), bb) for w, bb in ctx.lins[typ]]
            views = engine.grad_buffer([t for pair in lin for t in pair], dev)[1]    # one fill for the 40 tensors
            grads[typ] = list(zip(views[0::2], views[1::2]))
            keep.append(lin)
            setattr(b, "W_" + typ, engine.pointer_tables(lin)[0])
            dW, db = engine.pointer_tables(grads[typ])
            setattr(b, "dW_" + typ, dW)
            setattr(b, "db_" + typ, db)
        d_codes = torch.zeros(a.n_rays, 64, dtype=torch.float32, device=dev) if ctx.has_codes else None
        table_grad = None
        if cfg["has_table"]:
            table_grad = torch.zeros_like(cfg["embeddings"]["xyz"].embedding_space_ftr.weight, dtype=torch.float32)
        b.d_codes, b.table_grad = _lib.ptr(d_codes), _lib.ptr(table_grad)
        _lib.call("onerf_render_rays_bwd", dev, C.byref(a), C.byref(b))
        flat_out: List[Optional[torch.Tensor]] = []
        if cfg["has_table"]:
            flat_out.append(table_grad)
        for typ in cfg["model_order"]:
            for w, bb in grads[typ]:
                flat_out += [w, bb]
        assert len(flat_out) == ctx.n_params
        ctx.lease = None     # the workspace goes back to the pool
        return (None, None, d_codes) + tuple(flat_out)
