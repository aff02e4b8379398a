"""The editing path's joint sort and compositing stage by stage against the float64 references of
tests/test_multi_stages_cpu.py, where the references and their gates are checked (pytest -m gpu):
  - onerf_composite_multi_ws (the bitonic kernel, T = n_obj S <= 4096) and onerf_composite_multi_merge (the rank merge, any
    T) at every shape edge, on 1 ray, the planted 37 and 9 000, white background off and on: sorted depths and object ids
    bit for bit, weights and maps inside the gates, weights_unsorted exactly the weights scattered back to set order, NaN
    exactly where the reference is NaN; the two paths bit-identical to each other;
  - weights_unsorted against the reference's per-set selection weights[obj_ids == i] (multi_rendering.py:269-271);
  - the one-call chain (onerf_render_multi_fwd): coarse maps inside the gates on the staged route's fields, fine depths
    the sorted union of the per-set importance merges;
  - box culling of object ray sets around the 1024-thread list block: the culled one call bit-identical to the staged
    route.
Each gate check prints the largest share of its gate that a result used (RATIO label: x)."""
import numpy as np
import pytest
import torch

from tests.test_gpu_many_objects import _boxes, _case, _equal, _render, _setup
from tests.test_multi_stages_cpu import (BITONIC_MAX_T, MAP_KEYS, MULTI_SHAPES, N_PLANT, OUT_KEYS, ROW_DESC, ROW_NAN,
                                         ROW_NAN_NEG, ROW_ZEROS, composite_multi64, descending_sets, multi_inputs,
                                         multi_verdict, non_descending_sets, ray_counts)

pytestmark = pytest.mark.gpu
DEV = "cuda"
NAN_FILL = 0x7FA00001      # a NaN bit pattern no kernel writes: an output entry still holding it was never written


def _report(label, r):
    print(f"RATIO {label}: {r:.3e}")
    return r


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _filled(*shape):
    return torch.full(shape, NAN_FILL, dtype=torch.int32, device=DEV).view(torch.float32)


def _composite_multi(z_all, field_all, white_back, merge):
    """engine.composite_multi's two entries with every output prefilled with NAN_FILL: onerf_composite_multi_ws (merge =
    False; the bitonic kernel for T <= 4096) or onerf_composite_multi_merge.  -> numpy dict of OUT_KEYS."""
    from object_nerf_b200 import _lib
    lib = _lib.load()
    n_obj, n, S = z_all.shape
    T = n_obj * S
    out = dict(z_vals=_filled(n, T), weights=_filled(n, T), obj_ids=_filled(n, T), weights_unsorted=_filled(n_obj, n, S),
               opacity=_filled(n), rgb=_filled(n, 3), depth=_filled(n))
    ws = None
    if merge or T > BITONIC_MAX_T:
        ws = torch.empty(max(lib.onerf_composite_multi_workspace_bytes(n, n_obj, S), 256), dtype=torch.uint8, device=DEV)
    entry = lib.onerf_composite_multi_merge if merge else lib.onerf_composite_multi_ws
    _lib.check(entry(_lib.ctx(z_all.device), z_all.data_ptr(), field_all.data_ptr(), n, n_obj, S, int(bool(white_back)),
                     out["z_vals"].data_ptr(), out["weights"].data_ptr(), out["obj_ids"].data_ptr(),
                     out["weights_unsorted"].data_ptr(), out["opacity"].data_ptr(), out["rgb"].data_ptr(),
                     out["depth"].data_ptr(), _lib.ptr(ws), ws.numel() if ws is not None else 0, _lib.stream()))
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in out.items()}


def _per_set_selection(got, z):
    """weights_unsorted[i] against the reference's selection weights[obj_ids == i].view(n, S): bit for bit on every
    non-descending set; on a strictly descending set (near > far) it is the selection reversed, i.e. each weight stays
    with its own sample (DESIGN §4.3).  -> number of descending sets checked."""
    n_obj, n, S = z.shape
    w, ids, wu = got["weights"], got["obj_ids"], got["weights_unsorted"]
    asc, desc = non_descending_sets(z), descending_sets(z)
    for i in range(n_obj):
        sel = w[ids == i].reshape(n, S)
        assert np.array_equal(_bits(wu[i][asc[i]]), _bits(sel[asc[i]])), i
        assert np.array_equal(_bits(wu[i][desc[i]]), _bits(sel[desc[i]][:, ::-1])), i
    return int(desc.sum())


@pytest.mark.parametrize("white_back", [False, True])
@pytest.mark.parametrize("n_obj,S", MULTI_SHAPES)
def test_joint_sort_and_compositing_inside_the_float64_gates(n_obj, S, white_back):
    """Both paths (the bitonic kernel where T <= 4096, the rank merge everywhere) on multi_inputs: every output passes
    multi_verdict (NaN-prefilled buffers, so an entry left unwritten fails), the two paths agree bit for bit, and
    weights_unsorted is the reference's per-set selection on non-descending sets and its reverse on descending ones."""
    T = n_obj * S
    for n in ray_counts(n_obj, S):
        z, f = multi_inputs(n, n_obj, S, seed=n_obj * 10000 + S + n)
        want = composite_multi64(z, f, white_back)
        Z, F = _t(z), _t(f)
        got = {}
        for path in (("bitonic",) if T <= BITONIC_MAX_T else ()) + ("merge",):
            got[path] = _composite_multi(Z, F, white_back, merge=path == "merge")
            fails, shares = multi_verdict(got[path], want)
            label = f"composite_multi {path} n_obj={n_obj} S={S} n={n} white={int(white_back)}"
            _report(label + " weights", shares["weights"])
            _report(label + " maps", max(v for k, v in shares.items() if k != "weights"))
            assert not fails, (path, n, fails, shares)
            desc = _per_set_selection(got[path], z)
            assert desc > 0 or S == 1 or n < N_PLANT
        if len(got) == 2:
            for k in OUT_KEYS:
                assert np.array_equal(_bits(got["bitonic"][k]), _bits(got["merge"][k])), (n, k)


def test_planted_rows_reach_the_kernels_as_planted():
    """The rows the contract is about are in the device inputs: -0.0 after +0.0 in a set, NaN of both signs, a
    descending set; and the sorted output of the -0.0 row keeps +0.0 first (index order), the NaN rows end in NaN."""
    z, f = multi_inputs(N_PLANT, 3, 11, seed=3 * 10000 + 11 + N_PLANT)
    got = _composite_multi(_t(z), _t(f), False, merge=True)
    zs = got["z_vals"]
    zeros = zs[ROW_ZEROS][zs[ROW_ZEROS] == 0]
    assert len(zeros) == 3 and list(np.signbit(zeros)) == [False, True, True]
    for r in (ROW_NAN, ROW_NAN_NEG):
        assert np.isnan(zs[r, -1]) and not np.isnan(zs[r, :-1]).any()
    assert np.signbit(zs[ROW_NAN_NEG, -1])
    assert descending_sets(z)[1, ROW_DESC]


# ------------------------------------------------------------------------------------------------
# the one-call chain
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_one_call_chain_inside_the_gates(precision):
    """onerf_render_multi_fwd (render_rays_multi's default route) with a scene set under two removed-object boxes, a
    missed object set and a partly hit one: the coarse maps pass multi_verdict on the fields the staged route computes
    (engine.sample_coarse / engine.field as eval_pass does), and each ray's fine depths are the sorted union over sets
    of engine.sample_pdf_merge(z_coarse_i, W_i, K, det=True), W_i = weights_coarse[obj_ids_coarse == i] as the reference
    selects it."""
    from object_nerf_b200 import engine
    from object_nerf_b200.multi_rendering import boxes_to_tensor
    from object_nerf_b200.rendering import _grid_of
    ids, n, S, K = [0, 4, 6], 129, 64, 32
    c, inp = _case(n, ids, S, K, seed=710, hits=[None, "none", None])
    c["white_back"] = precision == "bf16"
    setup = _setup(inp)
    out = _render(c, inp, precision, setup=setup)
    models, emb, codes = setup
    grid = _grid_of(emb["xyz"])
    code_table = engine._f32(codes.embedding_instance.weight.detach())
    boxes = boxes_to_tensor(_boxes(inp), torch.device(DEV))
    rays = [r.to(DEV).contiguous().float() for r in inp["rays_list"]]
    packed = engine.packed_for(models["coarse"], True)
    with torch.no_grad():
        z_all = torch.empty(len(ids), n, S, device=DEV)
        field_all = torch.empty(len(ids), n, S, 4, device=DEV)
        for i, iid in enumerate(ids):
            engine.sample_coarse(rays[i], S, False, 0.0, out=z_all[i])
            is_obj = iid > 0
            engine.field(rays[i], z_all[i], packed, grid, code_row=code_table[iid] if is_obj else None,
                         want_scene=not is_obj, want_object=is_obj, precision=precision, mute_zero_rays=True,
                         boxes=None if is_obj else boxes, scene_out=None if is_obj else field_all[i],
                         obj_out=field_all[i] if is_obj else None)
    torch.cuda.synchronize()
    z, f = z_all.cpu().numpy(), field_all.cpu().numpy()
    assert (z[1] == 0).all() and (f[1, ..., 3] == -1e5).all()
    want = composite_multi64(z, f, c["white_back"])
    got = {k: out[k + "_coarse"].cpu().numpy() for k in ("z_vals", "obj_ids") + MAP_KEYS}
    fails, shares = multi_verdict(got, want)
    _report(f"one call {precision} coarse maps", max(shares.values()))
    assert not fails, (fails, shares)
    w, oid = out["weights_coarse"], out["obj_ids_coarse"]
    with torch.no_grad():
        zf = [engine.sample_pdf_merge(z_all[i], w[oid == i].view(n, S), K, True) for i in range(len(ids))]
        want_fine = torch.sort(torch.cat(zf, 1), dim=1, stable=True).values
    assert torch.equal(out["z_vals_fine"].view(torch.int32), want_fine.view(torch.int32))


# ------------------------------------------------------------------------------------------------
# box culling at the list block's edges
# ------------------------------------------------------------------------------------------------
CULL_SIZES = [1023, 1024, 1025, 2049, 70001]    # cull_list_kernel: 1024 threads, ceil(n / 1024) rays each


@pytest.mark.parametrize("n", CULL_SIZES)
def test_culled_one_call_at_the_list_block_edges(n):
    """Object sets with no hits, one hit, about half hits and all hits, at ray counts just under, at and over one ray per
    list thread, and many per thread: the culled one call is bit-identical to the staged (muted, unculled) route."""
    ids = [0, 4, 6, 4, 5]
    c, inp = _case(n, ids, 16, 16, seed=720 + n % 89, hits=[None, "none", "one", "all", "all"])
    half = inp["rays_list"][3]
    miss = torch.from_numpy(np.random.default_rng(n).random(n) < 0.5)
    half[miss, 6], half[miss, 7] = 0.0, 0.0
    live = [int((r[:, 7] != 0).sum()) for r in inp["rays_list"][1:]]
    assert live[0] == 0 and live[1] == 1 and 0 < live[2] < n and live[3] == n
    setup = _setup(inp)
    one = _render(c, inp, "bf16", setup=setup)
    staged = _render(c, inp, "bf16", staged=True, setup=setup)
    _equal(one, staged)
