"""Differentiable field evaluations at given positions: ObjectNeRF.forward / forward_instance on embedded points and
inference_model under autograd (reference models/nerf_model.py:97-152, models/rendering.py:64-230).

FieldEvalFn runs onerf_field_fwd over chunks of rays (bf16: with the tensor-core training dump; fp32: plain, the backward
re-runs it) and its backward onerf_field_bwd.  A point query is a ray of one sample: rays[:, 3:6] = the direction, z = 0,
the point as its explicit position.  CompositeFn is onerf_composite with onerf_composite_bwd as its backward.

Gradients go to what the reference's graph reaches: the Linear tensors of the evaluated branch (with sigma_only only the
trunk and the sigma head), the voxel table and the object codes.  Positions, directions and depths get none.
"""
from __future__ import annotations

import torch

from . import _lib, engine

# samples per field call: bounds the training dump (about 11.4 KB per sample, DESIGN §4.4) and the backward workspace
CHUNK_SAMPLES = 1 << 18

SCENE = tuple(range(0, 12))
SCENE_SIGMA = tuple(range(0, 9))          # xyz_encoding_1..8, sigma
OBJECT = tuple(range(12, 20))
OBJECT_SIGMA = tuple(range(12, 17))       # instance_encoding_1..4, instance_sigma


def table_of(grid_module):
    return grid_module.embedding_space_ftr.weight if grid_module is not None else None


class FieldEvalFn(torch.autograd.Function):
    """(codes, table, *40 Linear tensors) -> scene (N,S,4), obj (N,S,4) or None.  spec: model, grid_module (EmbeddingVoxel
    or None), rays (N,8), z (N,S), xyz (N,S,3) or None, want_object, precision ("bf16" / "fp32"), reached (ABI indices of
    the Linear pairs that receive gradients)."""

    @staticmethod
    def forward(ctx, spec, codes, table, *params):
        ctx.set_materialize_grads(False)
        rays, z, xyz = spec["rays"], spec["z"], spec["xyz"]
        n, s = z.shape
        dev = rays.device
        grid_module, fi, prec = spec["grid_module"], spec["want_object"], spec["precision"]
        use_voxel = grid_module is not None
        grid = engine.GridBuffers.from_module(grid_module) if use_voxel else None
        packed = engine.packed_for(spec["model"], use_voxel, fresh=True)
        codes_d = engine._f32(codes.detach()) if fi else None
        scene = torch.empty(n, s, 4, dtype=torch.float32, device=dev)
        obj = torch.empty(n, s, 4, dtype=torch.float32, device=dev) if fi else None
        lib = _lib.load()
        chunk = max(1, CHUNK_SAMPLES // s)
        ctx.chunks = []
        for r0 in range(0, n, chunk):
            r1 = min(n, r0 + chunk)
            tw = (engine.aligned_bytes(lib.onerf_field_train_bytes(int(use_voxel), (r1 - r0) * s), dev)
                  if prec == "bf16" else None)
            out = []
            engine.field(rays[r0:r1], z[r0:r1], packed, grid, codes=codes_d[r0:r1] if fi else None, want_scene=True,
                         want_object=fi, precision=prec, xyz=xyz[r0:r1] if xyz is not None else None,
                         scene_out=scene[r0:r1], obj_out=obj[r0:r1] if fi else None, train_ws=tw, _args_out=out)
            ctx.chunks.append((r0, r1, out[0], out[1]))
        # the argument blocks point at the fields (the bf16 head backward reads them): saved, not held by ctx, so that no
        # reference cycle output -> grad_fn -> ctx -> output keeps the dumps alive until the garbage collector runs
        ctx.save_for_backward(scene, obj)
        ctx.spec, ctx.n_params = spec, len(params)
        ctx.lins = engine.model_linears(spec["model"])
        ctx.dims = (n, s, use_voxel)
        return scene, obj

    @staticmethod
    def backward(ctx, g_scene, g_obj):
        spec = ctx.spec
        _alive = ctx.saved_tensors  # noqa: F841
        n, s, use_voxel = ctx.dims
        fi = spec["want_object"]
        dev = spec["rays"].device
        d_codes = (torch.zeros(n, 64, dtype=torch.float32, device=dev)
                   if fi and ctx.needs_input_grad[1] else None)
        table_grad = None
        if use_voxel and ctx.needs_input_grad[2]:
            table_grad = torch.zeros_like(table_of(spec["grid_module"]), dtype=torch.float32)
        g_obj = g_obj if fi else None
        prec = engine.PRECISIONS[spec["precision"]]
        chunk_rows = max((r1 - r0 for r0, r1, _, _ in ctx.chunks), default=0)
        grads = None
        if chunk_rows and (g_scene is not None or g_obj is not None):
            ws = engine.aligned_bytes(engine.field_bwd_workspace_bytes(prec, use_voxel, chunk_rows, s), dev)
            for r0, r1, args, _keep in ctx.chunks:
                grads = engine.field_bwd(args, g_scene[r0:r1].contiguous() if g_scene is not None else None,
                                         g_obj[r0:r1].contiguous() if g_obj is not None else None, ctx.lins, grads=grads,
                                         d_codes=d_codes[r0:r1] if d_codes is not None else None,
                                         table_grad=table_grad, workspace=ws)
        ctx.chunks = None
        out = []
        for i in range(len(ctx.lins)):
            for j in range(2):
                k = 3 + 2 * i + j
                ok = i in spec["reached"] and ctx.needs_input_grad[k]
                out.append((grads[i][j] if grads is not None else torch.zeros_like(ctx.lins[i][j])) if ok else None)
        return (None, d_codes, table_grad) + tuple(out)


def field_eval(model, grid_module, rays, z, xyz, codes, want_object, precision, reached):
    """FieldEvalFn over the model's tensors (ABI order): (scene, obj | None), each (N,S,4), differentiable."""
    params = [t for pair in engine.model_linears(model) for t in pair]
    spec = dict(model=model, grid_module=grid_module, rays=rays, z=z, xyz=xyz, want_object=want_object,
                precision=precision, reached=frozenset(reached))
    return FieldEvalFn.apply(spec, codes, table_of(grid_module), *params)


class CompositeFn(torch.autograd.Function):
    """onerf_composite (weights non-differentiable) with onerf_composite_bwd as its backward.  Outputs in KEYS order."""
    KEYS = ("weights", "opacity", "rgb", "depth", "rgb_instance", "depth_instance", "opacity_instance")

    @staticmethod
    def forward(ctx, cfg, z, scene, obj):
        ctx.set_materialize_grads(False)
        out = engine.composite(z, scene, obj, **cfg)
        ctx.cfg = cfg
        ctx.save_for_backward(z, scene, obj, out["depth"])
        ctx.mark_non_differentiable(out["weights"])
        return tuple(out.get(k) for k in CompositeFn.KEYS)

    @staticmethod
    def backward(ctx, *gouts):
        z, scene, obj, depth = ctx.saved_tensors
        cfg = {k: v for k, v in ctx.cfg.items() if k != "rays_in_bbox"}
        grads = {k: g for k, g in zip(CompositeFn.KEYS, gouts) if g is not None}
        dscene, dobj = engine.composite_bwd(z, scene, obj, depth, grads, **cfg)
        return None, None, dscene, dobj
