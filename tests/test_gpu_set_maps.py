"""Per-set maps of edited frames on the GPU (editing.set_keys, onerf_render_edit_frame_sets), on the synthetic scene of
tests/test_gpu_edit_frame.py:
  * asking for them changes no other output bit, and summed over the sets they give the joint maps (white background on
    and off); one set gives the joint maps;
  * fp32 coarse maps against float64 sums of the same call's weights_coarse / z_vals_coarse by obj_ids_coarse, and both
    passes (rgb included, fp32 and bf16) inside the float64 gates of tests/set_maps_oracle.py on the fields the staged
    route computes;
  * bit-identical over chunk_rays, tiles, and with the fine pass on the rank-merge sort (n_obj * (S + K) > 4096);
  * exact zeros for a set whose box is missed; duplicates in separate columns, and moving one leaves the other columns
    alone where its rays miss;
  * refusals launch nothing; a captured render_tile replays; render_edit through install(keys=...); two gloo ranks.
Each gate check prints the largest share of its gate that a result used (RATIO label: x)."""
import os
import socket
import sys
import types

import numpy as np
import pytest
import torch

from tests import set_maps_oracle as SO
from tests.test_gpu_edit_frame import (CONFIGS, FAR, FOCAL, NEAR, SF, Box, H, W, _frame, _kw, _look_at,
                                       _make_scene, _moved)

pytestmark = pytest.mark.gpu
U24 = 2.0 ** -24


@pytest.fixture(scope="module")
def scene():
    return _make_scene(torch.device("cuda:0"))


def _set_keys(kw):
    from object_nerf_b200 import editing
    return editing.set_keys(kw["N_importance"])


def _all_keys(kw):
    from object_nerf_b200 import editing
    return editing.result_keys(kw["N_importance"]) + _set_keys(kw)


def _within(got, want, bound, label):
    err = (got.double() - want.double()).abs()
    print(f"RATIO {label}: {(err / bound).max().item():.3e}")
    assert (err <= bound).all(), (label, err.max().item())


def _sum_over_sets(out, kw, label):
    """Summed over the sets the maps are the pass's joint maps (rgb without the white background), within the rounding
    of sums of T products: (T + 8) u sum |.| (plus the white background's two roundings)."""
    n_obj = len(kw["sets"])
    for typ in ("coarse", "fine") if kw["N_importance"] > 0 else ("coarse",):
        T = n_obj * (kw["N_samples"] + (kw["N_importance"] if typ == "fine" else 0))
        op = out[f"opacity_{typ}"]
        rgb = out[f"rgb_{typ}"] - ((1 - op)[:, None] if kw["white_back"] else 0)
        for k, joint in (("opacity", op), ("depth", out[f"depth_{typ}"]), ("rgb", rgb)):
            sets = out[f"{k}_sets_{typ}"]
            assert sets.shape[:2] == (op.shape[0], n_obj) and not torch.isnan(sets).any(), k
            bound = (T + 8) * U24 * (sets.double().abs().sum(1) + (2.0 if k == "rgb" else 0.0)) + 1e-30
            _within(sets.sum(1), joint, bound, f"{label} sum over sets {k}_{typ}")


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_set_maps_change_nothing_else_and_sum_to_the_joint_maps(scene, name, precision):
    kw = _kw(scene, name, precision)
    base = _frame(scene, kw, chunk_rays=1000)
    out = _frame(scene, kw, chunk_rays=1000, keys=_all_keys(kw))
    assert list(out) == _all_keys(kw)
    for k in base:
        assert torch.equal(out[k].view(torch.int32), base[k].view(torch.int32)), k
    _sum_over_sets(out, kw, f"{name} {precision}")
    n_obj = len(kw["sets"])
    if n_obj == 1:
        for typ in ("coarse", "fine"):
            for k in ("opacity", "depth"):
                _within(out[f"{k}_sets_{typ}"][:, 0], out[f"{k}_{typ}"], 2 * U24 * out[f"{k}_{typ}"].abs() + 1e-30,
                        f"one set {k}_{typ}")
            print(f"one set {name} {precision}: bitwise joint maps:",
                  {k: torch.equal(out[f"{k}_sets_{typ}"][:, 0], out[f"{k}_{typ}"]) for k in ("opacity", "depth")})
    z, ids = out["z_vals_coarse"], out["obj_ids_coarse"]
    for i in range(n_obj):                        # a ray that misses set i's box gives exact zeros in every map
        missed = ((ids == i) & (z == 0)).any(1)
        for typ in ("coarse", "fine") if kw["N_importance"] > 0 else ("coarse",):
            for k in SO.SET_KEYS:
                assert (out[f"{k}_{typ}"][missed, i] == 0).all(), (k, typ, i)
    if name == "missed_box_coarse_only":
        for k in SO.SET_KEYS:
            assert (out[f"{k}_coarse"][:, 2] == 0).all()
    if precision == "fp32":                       # coarse maps: the call's own weights summed by set, in float64
        w, zz = out["weights_coarse"].double(), z.double()
        T = w.shape[1]
        for i in range(n_obj):
            wi = torch.where(ids == i, w, torch.zeros_like(w))
            for k, v in (("opacity", 1.0), ("depth", zz)):
                _within(out[f"{k}_sets_coarse"][:, i], (wi * v).sum(1),
                        (T + 8) * U24 * (wi * v).abs().sum(1) + 1e-30, f"{name} {k}_sets_coarse[{i}] by obj_ids")


def _many_sets(sc):
    """33 sets (the scene and 32 copies of object 4 at spread poses): coarse T = 33 * 64 on the bitonic sort, fine
    T = 33 * 128 > 4096 on the rank merge."""
    Twc = _look_at((-3.2, 0.2, 0.3))
    box = sc["sets"]["dup_moved"][1][2]
    sets = [sc["sets"]["scene"][0]]
    for j in range(32):
        a = 2 * np.pi * j / 32
        sets.append((4, _moved(Twc, [0.4 * np.cos(a), 0.5 * np.sin(a), 0.05 * (j % 3)], a), box, 0.02))
    return sets


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("name", ["dup_moved_removed", "many_sets"])
def test_bit_identical_over_chunks_tiles_and_sort_paths(scene, name, precision):
    from object_nerf_b200 import editing
    kw = _kw(scene, "dup_moved_removed", precision)
    if name == "many_sets":
        kw["sets"] = _many_sets(scene)
    keys = _set_keys(kw)
    want = _frame(scene, kw, chunk_rays=4096, keys=keys + ["rgb_fine", "opacity_fine", "depth_fine", "rgb_coarse",
                                                             "opacity_coarse", "depth_coarse"])
    _sum_over_sets(want, kw, f"{name} {precision}")
    want = {k: want[k] for k in keys}
    assert (want["opacity_sets_fine"][:, 1:] > 0).any()
    for chunk in (997, 65536):
        got = _frame(scene, kw, chunk_rays=chunk, keys=keys)
        for k in keys:
            assert torch.equal(got[k].view(torch.int32), want[k].view(torch.int32)), (chunk, k)
    sets = kw.pop("sets")
    for begin, end, chunk in ((17, 18, 1000), (123, 4567, 4096), (4096, H * W, 997)):
        got = editing.render_tile(scene["models"], scene["emb"], scene["lib"], H, W, FOCAL, sets, NEAR, FAR, SF, begin,
                                  end, chunk_rays=chunk, keys=keys, **kw)
        for k in keys:
            assert torch.equal(got[k].view(torch.int32), want[k][begin:end].view(torch.int32)), (begin, end, k)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_both_passes_inside_the_float64_gates(scene, precision):
    """Pixels [1000, 2500) of the duplicated, moved, removed-box frame: the staged route's depths and fields of each set
    (camera_rays, engine.sample_coarse / field, and for the fine pass engine.sample_pdf_merge on the frame's coarse
    weights selected by set) give set_maps64, and the frame's set maps pass set_maps_verdict."""
    from object_nerf_b200 import engine
    from object_nerf_b200.multi_rendering import boxes_to_tensor
    from object_nerf_b200.ray_utils import camera_rays
    from object_nerf_b200.rendering import _grid_of
    dev = scene["dev"]
    kw = _kw(scene, "dup_moved_removed", precision)
    b, e = 1000, 2500
    out = _frame(scene, kw, chunk_rays=1000, keys=_all_keys(kw))
    out = {k: v[b:e] for k, v in out.items()}
    sets, S, K = kw["sets"], kw["N_samples"], kw["N_importance"]
    n, n_obj = e - b, len(sets)
    rays = [camera_rays(H, W, FOCAL, Toc, NEAR, FAR, SF, box=box, bbox_enlarge=enl, device=dev)[b:e].contiguous()
            for _, Toc, box, enl in sets]
    grid = _grid_of(scene["emb"]["xyz"])
    code_table = engine._f32(scene["lib"].embedding_instance.weight.detach())
    boxes = boxes_to_tensor(kw["background_skip_bbox"], dev)

    def fields(typ, z_all):
        packed = engine.packed_for(scene["models"][typ], True)
        f = torch.empty(n_obj, n, z_all.shape[2], 4, device=dev)
        for i, (iid, _, _, _) in enumerate(sets):
            obj = iid > 0
            engine.field(rays[i], z_all[i], packed, grid, code_row=code_table[iid] if obj else None, want_scene=not obj,
                         want_object=obj, precision=precision, mute_zero_rays=True, boxes=None if obj else boxes,
                         scene_out=None if obj else f[i], obj_out=f[i] if obj else None)
        return f

    with torch.no_grad():
        z_c = torch.stack([engine.sample_coarse(r, S, False, 0.0) for r in rays])
        f_c = fields("coarse", z_c)
        w, oid = out["weights_coarse"], out["obj_ids_coarse"]
        z_f = torch.stack([engine.sample_pdf_merge(z_c[i], w[oid == i].view(n, S), K, True) for i in range(n_obj)])
        f_f = fields("fine", z_f)
    torch.cuda.synchronize()
    want_z = torch.sort(torch.cat(list(z_f), 1), dim=1, stable=True).values
    assert torch.equal(out["z_vals_fine"].view(torch.int32), want_z.view(torch.int32))
    for typ, z, f in (("coarse", z_c, f_c), ("fine", z_f, f_f)):
        want = SO.set_maps64(z.cpu().numpy(), f.cpu().numpy())
        got = {k: out[f"{k}_{typ}"].cpu().numpy() for k in SO.SET_KEYS}
        fails, shares = SO.set_maps_verdict(got, want)
        for k, v in shares.items():
            print(f"RATIO set maps {precision} {k}_{typ}: {v:.3e}")
        assert not fails, (typ, fails, shares)
        print(f"{typ}: {int((f[0, ..., 3] == -1e5).sum())} scene samples muted by the removed boxes")


def test_moving_one_duplicate_changes_only_its_own_column(scene):
    kw = _kw(scene, "dup_moved_removed", "bf16")
    keys = _set_keys(kw) + ["z_vals_coarse", "obj_ids_coarse"]
    a = _frame(scene, kw, chunk_rays=4096, keys=keys)
    Twc = _look_at((-3.2, 0.2, 0.3))
    s0, s1, s2 = kw["sets"]
    kw["sets"] = [s0, s1, (s2[0], _moved(Twc, [0.1, -0.6, 0.1], 0.3), s2[2], s2[3])]
    b = _frame(scene, kw, chunk_rays=4096, keys=keys)
    miss = lambda o: ((o["obj_ids_coarse"] == 2) & (o["z_vals_coarse"] == 0)).any(1)
    both_miss = miss(a) & miss(b)
    assert both_miss.any() and (~both_miss).any()
    for k in SO.SET_KEYS:
        for typ in ("coarse", "fine"):
            key = f"{k}_{typ}"
            assert torch.equal(a[key][both_miss][:, :2], b[key][both_miss][:, :2]), key
            assert (a[key][both_miss][:, 2] == 0).all() and (b[key][both_miss][:, 2] == 0).all(), key
            assert not torch.equal(a[key][:, 2], b[key][:, 2]), key
            assert not torch.equal(a[key][:, 1], a[key][:, 2]), key     # the duplicates are separate columns


def test_refusals_launch_nothing(scene):
    """Fine set keys without a fine pass raise KeyError before the library; the C entry refuses a fine map without a fine
    pass and a misaligned map with ONERF_ERR_BAD_ARG on a live context before it launches anything."""
    import ctypes
    from object_nerf_b200 import _lib
    from tests.test_edit_frame_cpu import _Args
    dev = scene["dev"]
    with pytest.raises(KeyError):
        _frame(scene, _kw(scene, "missed_box_coarse_only", "bf16"), keys=["opacity_sets_fine"])
    lib = _lib.load()
    torch.cuda.synchronize()
    before = _lib.launch_count(dev)
    good = 1 << 24
    for n_importance, coarse, fine, msg in ((0, _lib.SetMaps(good, None, None), _lib.SetMaps(None, None, good),
                                             b"fine set maps without a fine pass"),
                                            (64, _lib.SetMaps(None, good + 2, None), None, b"4-byte aligned")):
        t = _Args(lib)
        t.a.n_importance = n_importance
        t.a.workspace_bytes = 1 << 40
        rc = lib.onerf_render_edit_frame_sets(_lib.ctx(dev), ctypes.byref(t.a), ctypes.byref(coarse),
                                              ctypes.byref(fine) if fine else None, _lib.stream())
        assert rc == -1 and msg in lib.onerf_last_error(), (rc, lib.onerf_last_error())
    torch.cuda.synchronize()
    assert _lib.launch_count(dev) == before


def test_render_tile_with_set_maps_replays_in_a_cuda_graph(scene):
    from object_nerf_b200 import editing
    kw = _kw(scene, "dup_moved_white_back", "bf16")        # no removed boxes: nothing is copied from the host
    sets = kw.pop("sets")
    keys = ["rgb_fine"] + editing.set_keys(64)
    run = lambda: editing.render_tile(scene["models"], scene["emb"], scene["lib"], H, W, FOCAL, sets, NEAR, FAR, SF, 500,
                                      3700, chunk_rays=1000, keys=keys, **kw)
    eager = run()
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        run()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        captured = run()
    for k in keys:
        captured[k].fill_(float("nan"))
    g.replay()
    torch.cuda.synchronize()
    for k in keys:
        assert torch.equal(captured[k].view(torch.int32), eager[k].view(torch.int32)), k


def test_render_edit_through_install_returns_set_maps_on_the_cpu(scene):
    """editing.install on a stand-in for the reference's EditableRenderer (the attributes render_edit reads): keys= with
    set maps returns them on the CPU, and every other key equals the call without them bit for bit."""
    from object_nerf_b200 import editing
    mod = types.ModuleType("fake_editable_renderer")
    mod.center_pose_from_avg = lambda pose_avg, pose: np.asarray(pose, dtype=np.float64).copy()
    sys.modules[mod.__name__] = mod
    box = Box([0.25, 0.1, 0.05], 0.3, rot=0.2)
    box.get_world_to_object_transform = lambda: np.eye(4)

    class Renderer:
        pass
    Renderer.__module__ = mod.__name__
    Renderer.get_object_bbox_helper = lambda self, obj_id: box
    Renderer.get_skipping_bbox_helper = lambda self: {"4": box}

    def make():
        r = Renderer()
        r.pose_avg, r.scale_factor, r.bbox_enlarge, r.near, r.far = np.eye(4), SF, 0.02, NEAR, FAR
        r.active_object_ids = [0, 4, 4]
        r.object_pose_transform = {"4_0": np.eye(4), "4_1": np.eye(4)}
        r.object_pose_transform["4_1"][:3, 3] = [0.05, -0.4, 0.0]
        r.ckpt_config = types.SimpleNamespace(model=types.SimpleNamespace(N_samples=64, N_importance=64, use_disp=False))
        r.system = types.SimpleNamespace(models=scene["models"], embeddings=scene["emb"], code_library=scene["lib"])
        return r
    Twc = _look_at((-3.2, 0.2, 0.3))
    try:
        editing.install(Renderer)
        plain = make().render_edit(H, W, Twc.copy(), 60)
        keys = editing.result_keys(64) + ["opacity_sets_fine", "rgb_sets_coarse"]
        editing.install(Renderer, keys=keys)
        got = make().render_edit(H, W, Twc.copy(), 60)
    finally:
        del sys.modules[mod.__name__]
    assert list(got) == [k for k in editing.result_keys(64) + editing.set_keys(64) if k in keys]
    assert list(plain) == editing.result_keys(64)
    for k in plain:
        assert got[k].device.type == "cpu" and torch.equal(got[k].view(torch.int32), plain[k].view(torch.int32)), k
    assert got["opacity_sets_fine"].device.type == "cpu" and got["opacity_sets_fine"].shape == (H * W, 3)
    assert got["rgb_sets_coarse"].shape == (H * W, 3, 3)
    assert (got["opacity_sets_fine"] > 0).any(0).all()


def _shard_worker(rank, world, port, ret):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dev = torch.device("cuda", rank % torch.cuda.device_count())
    torch.cuda.set_device(dev)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        sc = _make_scene(dev)
        kw = _kw(sc, "dup_moved_removed", "bf16")
        keys = _all_keys(kw)
        single = _frame(sc, kw, chunk_rays=1000, keys=keys)
        gathered = _frame(sc, kw, chunk_rays=1000, keys=keys, group=dist.group.WORLD)
        bad = [k for k in single if not torch.equal(single[k], gathered[k])]
        ret[rank] = (list(gathered) == keys, bad)
    finally:
        dist.destroy_process_group()


def test_sharded_frame_equals_the_single_process_frame():
    import torch.multiprocessing as mp
    world = 2
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    ctx = mp.get_context("spawn")
    ret = ctx.Manager().dict()
    procs = [ctx.Process(target=_shard_worker, args=(r, world, port, ret)) for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=300)
        assert p.exitcode == 0
    assert len(ret) == world
    for rank, (same_keys, bad) in ret.items():
        assert same_keys and not bad, (rank, bad)
