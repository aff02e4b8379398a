"""Generate tests/golden/field_query_*.npz by running the reference's own ObjectNeRF, Embedding, EmbeddingVoxel and
inference_model (/root/reference, CPU) on the cases of tests/field_query_cases.py.  Build container only:

    python tools/make_field_query_golden.py

Point fixtures: forward / forward_instance outputs and, for the loss sum(out * cotangent) over both branches, gradient
summaries of every Linear tensor, of obj_code and of the voxel table (with the rows touched).  inference_model fixtures:
the maps of one pass (sigma noise injected through torch.randn_like in the reference's draw order: scene, then object)
and the same gradient summaries for sum(map * cotangent)."""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import make_golden as G  # noqa: E402  (installs the reference modules)
from models.embedding_helper import Embedding  # noqa: E402
from models.rendering import inference_model as ref_inference_model  # noqa: E402

from tests import field_query_cases as FQ  # noqa: E402


def _table_rows(emb, fix):
    g = emb.embedding_space_ftr.weight.grad
    fix["voxel|nonzero_rows"] = torch.nonzero(g.abs().sum(1)).view(-1)


def gen_points():
    for name, c in FQ.POINT_CASES.items():
        inp = FQ.build_point_case(c)
        use_voxel = c["use_voxel"]
        m = G.ref_model(inp["weights"], use_voxel).train()
        codes = inp["codes"].clone().requires_grad_(True)
        if use_voxel:
            emb = G.ref_voxel_embedding(inp["grid"])
            emb_xyz, obj_voxel = emb(inp["pts"].clone())
        else:
            emb, emb_xyz, obj_voxel = None, Embedding(3, 10)(inp["pts"].clone()), None
        emb_dir = Embedding(3, 4)(inp["dirs"].clone())
        o = m.forward({"emb_xyz": emb_xyz, "emb_dir": emb_dir})
        oi = m.forward_instance({"emb_xyz": emb_xyz, "emb_dir": emb_dir, "obj_voxel": obj_voxel, "obj_code": codes})
        out = {"sigma": o["sigma"], "rgb": o["rgb"], "inst_sigma": oi["inst_sigma"], "inst_rgb": oi["inst_rgb"]}
        sum((out[k] * inp["cot"][k]).sum() for k in out).backward()
        named = [(k, p.grad) for k, p in m.named_parameters()] + [("obj_code", codes.grad)]
        if use_voxel:
            named.append(("voxel", emb.embedding_space_ftr.weight.grad))
        fix = {k: v.detach() for k, v in out.items()}
        fix.update(FQ.grad_summary(named))
        if use_voxel:
            _table_rows(emb, fix)
        G.save(f"field_query_{name}", **fix)


def gen_infer():
    for name, c in FQ.INFER_CASES.items():
        inp = FQ.build_infer_case(c)
        m = G.ref_model(inp["weights"], True).train()
        emb = G.ref_voxel_embedding(inp["grid"])
        codes = inp["codes"].clone().requires_grad_(True)
        res = {}
        seq = [inp["noise"]["noise_scene"]] + ([inp["noise"]["noise_obj"]] if c["forward_instance"] else [])
        with G.InjectRandom([], [], seq):   # drawn (and multiplied by noise_std) also when noise_std = 0
            ref_inference_model(res, m, {"xyz": emb, "dir": Embedding(3, 4)}, "coarse", inp["xyz"].clone(),
                                inp["rays"][:, None, 3:6].clone(), inp["z"].clone(), 1 << 20, c["noise_std"], False,
                                is_eval=c["is_eval"], use_zero_as_last_delta=c["zero_last_delta"],
                                forward_instance=c["forward_instance"], embedding_instance=codes,
                                frustum_bound_th=c["frustum_bound_th"], pass_through_mask=inp["pass_through_mask"])
        keys = [k for k in FQ.MAP_KEYS if f"{k}_coarse" in res]
        sum((res[f"{k}_coarse"] * inp["cot"][k]).sum() for k in keys).backward()
        named = [(k, p.grad) for k, p in m.named_parameters()] + [("obj_code", codes.grad),
                                                                  ("voxel", emb.embedding_space_ftr.weight.grad)]
        fix = {k: v.detach() for k, v in res.items() if torch.is_tensor(v)}
        fix.update(FQ.grad_summary(named))
        _table_rows(emb, fix)
        G.save(f"field_query_{name}", **fix)


if __name__ == "__main__":
    gen_points()
    gen_infer()
