"""The oracle (oracle/onerf_oracle.py, autograd on the CPU) against the field-query fixtures made from the reference's own
modules (tools/make_field_query_golden.py): point queries of both branches and inference_model passes with injected
noise, occlusion mask, eval mode and without the object branch - outputs and gradient summaries."""
import pytest
import torch

from oracle import onerf_oracle as O
from tests import field_query_cases as FQ, synth


def _params(w):
    """oracle weight dict whose tensors require grad, and their reference names"""
    p = {k: (a.clone().requires_grad_(True), b.clone().requires_grad_(True)) for k, (a, b) in w.items()}
    named = []
    for k, (a, b) in p.items():
        named += [(synth.REF_NAMES[k] + ".weight", a), (synth.REF_NAMES[k] + ".bias", b)]
    return p, named


def _grid(g, table):
    return O.VoxelGrid(g["offset"], g["voxel_size"], g["shape"].tolist(), g["idx_map"], table)


def _check_grads(fix, named):
    """Every gradient bit for bit, except the voxel table's: the reference stacks the 8 trilinear corner terms and sums
    them, the oracle adds them one by one, so the table rows' sums may differ in the last bits (1e-5 relative)."""
    for name, t in named:
        exact = name != "voxel"
        if name + "|norm" not in fix:
            assert t.grad is None or not t.grad.any(), name   # not reached by the reference's graph
            continue
        g = t.grad.reshape(-1)
        for key, got in (("norm", g.norm()), ("sum", g.sum())):
            want = fix[f"{name}|{key}"]
            if exact:
                assert torch.equal(got, want), (name, key)
            else:
                assert abs(got.item() - want.item()) <= 1e-5 * max(1.0, abs(want.item())) + 1e-6, (name, key)
        from tests import cases
        s = g[cases.sample_indices(name, g.numel())]
        if exact:
            assert torch.equal(s, fix[name + "|samples"]), name
        else:
            assert (s - fix[name + "|samples"]).abs().max().item() <= 1e-5 * max(1.0, fix[name + "|norm"].item()), name


@pytest.mark.parametrize("name", list(FQ.POINT_CASES))
def test_point_queries_match_reference(golden, name):
    c = FQ.POINT_CASES[name]
    inp = FQ.build_point_case(c)
    fix = golden(f"field_query_{name}")
    w, named = _params(inp["weights"])
    codes = inp["codes"].clone().requires_grad_(True)
    table = inp["grid"]["table"].clone().requires_grad_(True)
    grid = _grid(inp["grid"], table) if c["use_voxel"] else None
    out = O.field_eval(w, grid, inp["pts"], inp["dirs"], codes)
    out = {"sigma": out["sigma"][:, None], "rgb": out["rgb"], "inst_sigma": out["inst_sigma"][:, None],
           "inst_rgb": out["inst_rgb"]}
    for k, v in out.items():
        assert torch.equal(v, fix[k]), k
    sum((out[k] * inp["cot"][k]).sum() for k in out).backward()
    named += [("obj_code", codes)] + ([("voxel", table)] if c["use_voxel"] else [])
    _check_grads(fix, named)
    if c["use_voxel"]:
        assert torch.equal(torch.nonzero(table.grad.abs().sum(1)).view(-1), fix["voxel|nonzero_rows"])


@pytest.mark.parametrize("name", list(FQ.INFER_CASES))
def test_inference_passes_match_reference(golden, name):
    c = FQ.INFER_CASES[name]
    inp = FQ.build_infer_case(c)
    fix = golden(f"field_query_{name}")
    w, named = _params(inp["weights"])
    codes = inp["codes"].clone().requires_grad_(True)
    table = inp["grid"]["table"].clone().requires_grad_(True)
    n, s = inp["z"].shape
    fi = c["forward_instance"]
    f = O.field_eval(w, _grid(inp["grid"], table), inp["xyz"].reshape(-1, 3),
                     inp["rays"][:, None, 3:6].expand(n, s, 3).reshape(-1, 3),
                     codes[:, None].expand(n, s, 64).reshape(-1, 64), want_object=fi)
    out = {}
    O.composite_pass(out, "coarse", f["sigma"].view(n, s), f["rgb"].view(n, s, 3),
                     f["inst_sigma"].view(n, s) if fi else None, f["inst_rgb"].view(n, s, 3) if fi else None,
                     inp["z"], noise_std=c["noise_std"], is_eval=c["is_eval"], zero_last_delta=c["zero_last_delta"],
                     forward_instance=fi, frustum_bound_th=c["frustum_bound_th"],
                     pass_through_mask=inp["pass_through_mask"], noise_scene=inp["noise"]["noise_scene"],
                     noise_obj=inp["noise"]["noise_obj"])
    keys = [k for k in FQ.MAP_KEYS if f"{k}_coarse" in out]
    assert sorted(keys) == sorted(k for k in FQ.MAP_KEYS if f"{k}_coarse" in fix)
    for k in keys + ["weights"]:
        assert torch.equal(out[f"{k}_coarse"], fix[f"{k}_coarse"]), k
    sum((out[f"{k}_coarse"] * inp["cot"][k]).sum() for k in keys).backward()
    _check_grads(fix, named + [("obj_code", codes), ("voxel", table)])
