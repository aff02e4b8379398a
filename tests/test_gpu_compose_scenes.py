"""Edited frames that compose objects from several trained scenes (editing.Scene, onerf_render_edit_frame_scenes) on the
GPU, on the synthetic scene of tests/test_gpu_edit_frame.py as the base and a second synthetic scene (other weights, grid
and codes) as the source:
  * a set whose scene is a Scene of the base's own modules and scale, or of deep copies of them (other buffers, the same
    values, built anew), is bit-identical on every key and set map to the native set, over chunk sizes and tiles, in fp32 and bf16;
  * a source scene that differs from the base only in its code table changes only the pixels its object's box covers;
  * two scenes at k = 1, 8 and 1/8 against the float64 reference of tests/compose_oracle.py (the tolerances of
    tests/test_gpu_edit_frame.py), and the joint order of the coarse pass bit for bit: every set's depths times its k,
    stably sorted, give z_vals_coarse and obj_ids_coarse;
  * a captured render_tile with a source set replays; two gloo ranks gather the frame one process renders."""
import os
import socket

import numpy as np
import pytest
import torch

from tests.test_gpu_edit_frame import (FAR, FOCAL, NEAR, SF, Box, H, W, _close, _frame, _kw, _look_at,
                                       _make_scene)

pytestmark = pytest.mark.gpu
TILE = (2400, 2720)                 # rows 30 .. 33 of the 64 x 80 frame: every object box is in view


@pytest.fixture(scope="module")
def base():
    return _make_scene(torch.device("cuda:0"))


def _keys(n_importance=64):
    from object_nerf_b200 import editing
    return editing.result_keys(n_importance) + editing.set_keys(n_importance)


def _toc(Twc, shift, rot, s):
    """Toc of an object set moved by `shift` (world units) and turned by `rot` about z, at the NeRF scale of a scene
    with scale_factor s."""
    c, si = np.cos(rot), np.sin(rot)
    transform = np.eye(4)
    transform[:2, :2] = [[c, -si], [si, c]]
    transform[:3, 3] = shift
    Toc = np.linalg.inv(transform) @ Twc
    Toc[:3, 3] /= s
    return torch.from_numpy(Toc).float()[:3, :4]


def _source_inputs(k):
    """Weights, grid and codes of the second scene; its grid covers the base grid's world region at scale SF * k."""
    from object_nerf_b200 import synthetic as S
    return dict(weights={"coarse": S.make_weights(20, True, sigma_gain=8.0, sigma_bias=1.0, rgb_gain=24.0),
                         "fine": S.make_weights(1020, True, sigma_gain=8.0, sigma_bias=1.0, rgb_gain=24.0)},
                grid=S.make_grid(seed=9, shape=(42, 42, 22), occupancy=0.5, voxel_size=0.05 / k), codes=S.make_codes(7))


def _base_inputs():
    """The inputs _make_scene builds the base scene from."""
    from object_nerf_b200 import synthetic as S
    return dict(weights={"coarse": S.make_weights(0, True, sigma_gain=8.0, sigma_bias=1.0, rgb_gain=24.0),
                         "fine": S.make_weights(1000, True, sigma_gain=8.0, sigma_bias=1.0, rgb_gain=24.0)},
                grid=S.make_grid(seed=5, shape=(42, 42, 22), occupancy=0.6, voxel_size=0.05), codes=S.make_codes(2))


def _copy_of_base(dev):
    """A Scene of new modules holding the base scene's values at its scale: other buffers, the same bits."""
    from object_nerf_b200 import Embedding, editing, synthetic as S
    inp = _base_inputs()
    models = {t: S.make_model(w, True, dev) for t, w in inp["weights"].items()}
    emb = {"xyz": S.GridModule(inp["grid"]).to(dev), "dir": Embedding(3, 4)}
    return editing.Scene(models, emb, S.make_code_library(inp["codes"]).to(dev), SF)


_SOURCES = {}


def _source(k, dev):
    if k not in _SOURCES:
        from object_nerf_b200 import Embedding, editing, synthetic as S
        inp = _source_inputs(k)
        models = {t: S.make_model(w, True, dev) for t, w in inp["weights"].items()}
        emb = {"xyz": S.GridModule(inp["grid"]).to(dev), "dir": Embedding(3, 4)}
        _SOURCES[k] = editing.Scene(models, emb, S.make_code_library(inp["codes"]).to(dev), SF * k)
    return _SOURCES[k]


def _two_scene_sets(base, k):
    """[scene, object 4 of the base, objects 4 and 6 of the source at scale SF * k]."""
    Twc = _look_at((-3.2, 0.2, 0.3))
    src = _source(k, base["dev"])
    s = src.scale_factor
    box4, box6 = Box([0.25, 0.1, 0.05], 0.3, rot=0.2), Box([-0.3, -0.2, 0.0], 0.25)
    return [base["sets"]["scene"][0], (4, _toc(Twc, [0.05, 0.3, 0], 0.1, SF), box4, 0.02),
            (4, _toc(Twc, [-0.05, -0.4, 0], -0.2, s), box4, 0.02, src), (6, _toc(Twc, [0.0, 0.1, 0.0], 0.4, s), box6, 0.0, src)]


def _bitwise(got, want, rows=slice(None)):
    assert list(got) == list(want)
    for k in want:
        assert torch.equal(got[k].view(torch.int32), want[k][rows].view(torch.int32)), k


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_self_composition_is_bit_identical_to_the_native_sets(base, precision):
    from object_nerf_b200 import editing
    kw = _kw(base, "dup_moved_removed", precision)
    want = _frame(base, kw, chunk_rays=4096, keys=_keys())
    own = editing.Scene(base["models"], base["emb"], base["lib"], SF)
    copied = _copy_of_base(base["dev"])
    assert copied.code_library.embedding_instance.weight.data_ptr() != base["lib"].embedding_instance.weight.data_ptr()
    for scene in (own, copied):
        sets = [s if s[0] == 0 else s + (scene,) for s in kw["sets"]]
        for chunk in (1000, 4096, 65536):
            _bitwise(_frame(base, dict(kw, sets=sets), chunk_rays=chunk, keys=_keys()), want)
        rest = {k: v for k, v in kw.items() if k != "sets"}
        for begin, end, chunk in ((17, 18, 1000), (123, 4567, 4096), (4096, H * W, 997)):
            got = editing.render_tile(base["models"], base["emb"], base["lib"], H, W, FOCAL, sets, NEAR, FAR, SF, begin,
                                      end, chunk_rays=chunk, keys=_keys(), **rest)
            _bitwise(got, want, slice(begin, end))
    assert (want["opacity_sets_fine"][:, 1:] > 0).any()


def test_a_different_code_table_changes_only_the_pixels_its_box_covers(base):
    from object_nerf_b200 import editing, synthetic as S
    kw = _kw(base, "dup_moved_removed", "bf16")
    native = _frame(base, kw, chunk_rays=4096, keys=_keys())
    other = editing.Scene(base["models"], base["emb"], S.make_code_library(S.make_codes(9)).to(base["dev"]), SF)
    sets = list(kw["sets"])
    sets[2] = sets[2] + (other,)
    got = _frame(base, dict(kw, sets=sets), chunk_rays=4096, keys=_keys())
    miss = ((native["obj_ids_coarse"] == 2) & (native["z_vals_coarse"] == 0)).any(1)
    assert miss.any() and (~miss).any()
    for k in native:
        assert torch.equal(got[k][miss], native[k][miss]), k
    assert not torch.equal(got["rgb_fine"][~miss], native["rgb_fine"][~miss])
    assert torch.equal(got["opacity_sets_fine"][:, :2][miss], native["opacity_sets_fine"][:, :2][miss])


# ------------------------------------------------------------------------------------------------
# two scenes against the float64 reference
# ------------------------------------------------------------------------------------------------
def _f64_scene(inp, k):
    from oracle import onerf_oracle as O
    g = inp["grid"]
    return dict(weights={t: {n: (Wt.double(), b.double()) for n, (Wt, b) in w.items()} for t, w in inp["weights"].items()},
                grid=O.VoxelGrid(g["offset"].double(), g["voxel_size"].double(), g["shape"].tolist(), g["idx_map"],
                                 g["table"].double()),
                code_table=inp["codes"].double(), k=k)


def _set_rays(base, sets, begin, end):
    from object_nerf_b200.ray_utils import camera_rays
    out = []
    for s in sets:
        scale = s[4].scale_factor if len(s) > 4 else SF
        out.append(camera_rays(H, W, FOCAL, s[1], NEAR, FAR, scale, box=s[2], bbox_enlarge=s[3],
                               device=base["dev"])[begin:end].contiguous())
    return out


_ORACLE = {}


def _oracle(base, k):
    """tests/compose_oracle.py in float64 on the tile's rays of _two_scene_sets(base, k)."""
    if k not in _ORACLE:
        from tests import cases
        from tests import compose_oracle as CO
        sets = _two_scene_sets(base, k)
        rays = [r.cpu().double() for r in _set_rays(base, sets, *TILE)]
        skip = []
        for b in base["removed"].values():
            A, t, lo, hi = cases.box_affine(dict(scale_factor=b.scale_factor, pose_avg=b.pose_avg,
                                                 axis_align_mat=b.axis_align_mat, bbox_bounds=b.bbox_bounds))
            skip.append((A.double(), t.double(), lo.double(), hi.double()))
        scenes = [_f64_scene(_base_inputs(), 1.0), _f64_scene(_source_inputs(k), CO.compose_k(SF * k, SF))]
        _ORACLE[k] = CO.render_rays_multi_scenes(scenes, [0, 0, 1, 1], rays, [s[0] for s in sets], n_samples=64,
                                                 n_importance=64, skip_boxes=skip)
    return _ORACLE[k]


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("k", [1.0, 8.0, 0.125])
def test_two_scenes_against_the_float64_reference(base, k, precision):
    from object_nerf_b200 import editing, engine
    sets = _two_scene_sets(base, k)
    kw = dict(background_skip_bbox=base["removed"], N_samples=64, N_importance=64, precision=precision)
    got = editing.render_tile(base["models"], base["emb"], base["lib"], H, W, FOCAL, sets, NEAR, FAR, SF, *TILE,
                              chunk_rays=1000, keys=_keys(), **kw)
    z, ids = got["z_vals_coarse"], got["obj_ids_coarse"]
    hit = [float((z[ids == i] > 0).float().mean()) for i in range(4)]
    print(f"k = {k} {precision}: hit fraction per set {hit}")
    assert min(hit[1:]) > 0
    # the joint order: each set's own coarse depths (its units) times its k, stably sorted
    rays = _set_rays(base, sets, *TILE)
    ks = [1.0, 1.0] + [float(np.float32(sets[2][4].scale_factor / SF))] * 2
    with torch.no_grad():
        zk = [engine.sample_coarse(r, 64, False, 0.0) for r in rays]
    zk = [zi if ki == 1.0 else zi * torch.tensor(ki, dtype=torch.float32, device=zi.device) for zi, ki in zip(zk, ks)]
    want_z, order = torch.sort(torch.cat(zk, 1), dim=1, stable=True)
    assert torch.equal(z.view(torch.int32), want_z.view(torch.int32))
    assert torch.equal(ids, (order // 64).float())
    want = _oracle(base, k)
    for typ in ("coarse", "fine"):
        for key in ("rgb", "depth", "opacity"):
            _close(f"k={k} {key}_{typ}", got[f"{key}_{typ}"].cpu(), want[f"{key}_{typ}"], precision)
        for key in ("opacity_sets", "depth_sets"):
            _close(f"k={k} {key}_{typ}", got[f"{key}_{typ}"].cpu(), want[f"{key}_{typ}"], precision)
        sets_sum = got[f"opacity_sets_{typ}"].double().sum(1).cpu()
        assert (sets_sum - got[f"opacity_{typ}"].double().cpu()).abs().max() < 1e-4


def test_equal_scale_source_of_copied_modules_is_the_native_frame(base):
    """A source scene of new modules with the base's values at the base's scale: every set of it reads its own scene's
    grid, weights and code rows, and the frame is bit for bit the native one."""
    from object_nerf_b200 import editing
    kw = _kw(base, "dup_moved_white_back", "fp32")
    copied = _copy_of_base(base["dev"])
    want = _frame(base, kw, chunk_rays=2048, keys=_keys())
    got = _frame(base, dict(kw, sets=[kw["sets"][0], kw["sets"][1] + (copied,), kw["sets"][2]]), chunk_rays=2048,
                 keys=_keys())
    _bitwise(got, want)


def test_render_tile_with_a_source_set_replays_in_a_cuda_graph(base):
    from object_nerf_b200 import editing
    sets = _two_scene_sets(base, 8.0)
    keys = ["rgb_fine", "depth_fine"] + editing.set_keys(64)
    run = lambda: editing.render_tile(base["models"], base["emb"], base["lib"], H, W, FOCAL, sets, NEAR, FAR, SF, 500,
                                      3700, chunk_rays=1000, keys=keys, N_samples=64, N_importance=64, precision="bf16")
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


def _shard_worker(rank, world, port, ret):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dev = torch.device("cuda", rank % torch.cuda.device_count())
    torch.cuda.set_device(dev)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        sc = _make_scene(dev)
        kw = dict(sets=_two_scene_sets(sc, 8.0), background_skip_bbox=sc["removed"], N_samples=64, N_importance=64,
                  precision="bf16")
        single = _frame(sc, kw, chunk_rays=1000, keys=_keys())
        gathered = _frame(sc, kw, chunk_rays=1000, keys=_keys(), group=dist.group.WORLD)
        bad = [k for k in single if not torch.equal(single[k], gathered[k])]
        ret[rank] = (list(gathered) == _keys(), bad)
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
