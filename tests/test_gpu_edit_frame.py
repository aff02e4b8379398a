"""Edited frames from a camera (object_nerf_b200.editing, onerf_render_edit_frame) on the GPU.

  * Chunk and tile independence: render_frame / render_tile equal, bit for bit on every key, what the existing entries
    give for the same frame: camera_rays per set, render_rays_multi over 4 096-ray chunks, concatenated.
  * A `keys` subset equals the same keys of the full call.
  * editing.render_edit / render_origin against the unmodified EditableRenderer over dropin.install() (oracle/_ref).
  * Two ranks (gloo on one GPU; NCCL when there are two GPUs) gather the frame one process renders.
  * The refusals of onerf_render_edit_frame through the Python entry."""
import os
import socket

import numpy as np
import pytest
import torch

from oracle import ref_loader as R

pytestmark = pytest.mark.gpu

H, W = 64, 80                     # 5 120 pixels: one to six chunks at chunk_rays 1 000 .. 65 536
FOCAL = 0.5 * W / np.tan(np.radians(30.0))
NEAR, FAR, SF = 0.3, 6.0, 2.0     # scene near / far in world units (rays: near / SF, far / SF)
CHUNK = 4096


class Box:
    """The BBoxRayHelper attributes the box test and the removed-object mask read: a box of half-size `half` around
    `center` in the axis-aligned frame (world units)."""

    def __init__(self, center, half, rot=0.0):
        self.scale_factor = SF
        self.pose_avg = np.eye(4)
        self.axis_align_mat = np.eye(4)
        c, s = np.cos(rot), np.sin(rot)
        self.axis_align_mat[:2, :2] = [[c, -s], [s, c]]
        self.axis_align_mat[:3, 3] = [0.02, -0.03, 0.01]
        self.bbox_bounds = np.array([np.asarray(center) - half, np.asarray(center) + half])


def _look_at(cam, target=(0.0, 0.0, 0.0)):
    cam = np.asarray(cam, dtype=np.float64)
    fwd = np.asarray(target) - cam
    fwd /= np.linalg.norm(fwd)
    right = np.cross(fwd, [0.0, 0.0, 1.0])
    right /= np.linalg.norm(right)
    up = np.cross(right, fwd)
    T = np.eye(4)
    T[:3, :3] = np.stack([right, up, -fwd], 1)
    T[:3, 3] = cam
    return T


def _moved(Twc, shift, rot=0.0):
    """Toc of an object set moved by `shift` (world units) and turned by `rot` about z, at NeRF scale."""
    c, s = np.cos(rot), np.sin(rot)
    transform = np.eye(4)
    transform[:2, :2] = [[c, -s], [s, c]]
    transform[:3, 3] = shift
    Toc = np.linalg.inv(transform) @ Twc
    Toc[:3, 3] /= SF
    return torch.from_numpy(Toc).float()[:3, :4]


def _make_scene(dev):
    from object_nerf_b200 import Embedding, synthetic as S
    wc = S.make_weights(0, True, sigma_gain=8.0, sigma_bias=1.0, rgb_gain=24.0)
    wf = S.make_weights(1000, True, sigma_gain=8.0, sigma_bias=1.0, rgb_gain=24.0)
    grid = S.make_grid(seed=5, shape=(42, 42, 22), occupancy=0.6, voxel_size=0.05)
    models = {"coarse": S.make_model(wc, True, dev), "fine": S.make_model(wf, True, dev)}
    emb = {"xyz": S.GridModule(grid).to(dev), "dir": Embedding(3, 4)}
    Twc = _look_at((-3.2, 0.2, 0.3))
    scene_toc = _moved(Twc, [0, 0, 0])
    boxes = {"4": Box([0.25, 0.1, 0.05], 0.3, rot=0.2), "6": Box([-0.3, -0.2, 0.0], 0.25),
             "9": Box([0.0, 0.0, 9.0], 0.2)}            # 9: above the camera's view, no ray hits it
    sets = {
        "scene": [(0, scene_toc, None, 0.0)],
        "dup_moved": [(0, scene_toc, None, 0.0), (4, _moved(Twc, [0.05, 0.3, 0], 0.1), boxes["4"], 0.02),
                      (4, _moved(Twc, [-0.05, -0.4, 0], -0.2), boxes["4"], 0.02)],
        "missed_box": [(0, scene_toc, None, 0.0), (6, _moved(Twc, [0, 0.2, 0]), boxes["6"], 0.0),
                       (9, scene_toc, boxes["9"], 0.0)],
    }
    removed = {"4": boxes["4"], "6": boxes["6"]}
    return dict(models=models, emb=emb, lib=S.make_code_library(S.make_codes(2)).to(dev), sets=sets, removed=removed,
                dev=dev)


@pytest.fixture(scope="module")
def scene():
    return _make_scene(torch.device("cuda:0"))


CONFIGS = {   # sets, removed boxes, N_importance, use_disp, white_back
    "scene_only_disp": ("scene", False, 64, True, False),
    "dup_moved_removed": ("dup_moved", True, 64, False, False),
    "missed_box_coarse_only": ("missed_box", True, 0, False, False),
    "dup_moved_white_back": ("dup_moved", False, 64, False, True),
}


def _kw(sc, name, precision):
    sets, removed, ni, use_disp, white_back = CONFIGS[name]
    return dict(sets=sc["sets"][sets], background_skip_bbox=sc["removed"] if removed else None, N_samples=64,
                N_importance=ni, use_disp=use_disp, white_back=white_back, precision=precision)


def _chunked_route(sc, kw):
    """camera_rays per set + render_rays_multi over 4 096-ray chunks, concatenated (render_edit over the drop-in)."""
    from object_nerf_b200.multi_rendering import render_rays_multi
    from object_nerf_b200.ray_utils import camera_rays
    rays = [camera_rays(H, W, FOCAL, Toc, NEAR, FAR, SF, box=box, bbox_enlarge=enl, device=sc["dev"])
            for _, Toc, box, enl in kw["sets"]]
    ids = [s[0] for s in kw["sets"]]
    parts = []
    with torch.no_grad():
        for i in range(0, H * W, CHUNK):
            parts.append(render_rays_multi(sc["models"], sc["emb"], sc["lib"], [r[i:i + CHUNK] for r in rays], ids,
                                           N_samples=kw["N_samples"], use_disp=kw["use_disp"], perturb=0, noise_std=0,
                                           N_importance=kw["N_importance"], white_back=kw["white_back"],
                                           background_skip_bbox=kw["background_skip_bbox"], precision=kw["precision"]))
    return {k: torch.cat([p[k] for p in parts], 0) for k in parts[0]}


def _frame(sc, kw, **extra):
    from object_nerf_b200 import editing
    kw = dict(kw)
    sets = kw.pop("sets")
    return editing.render_frame(sc["models"], sc["emb"], sc["lib"], H, W, FOCAL, sets, NEAR, FAR, SF, **kw, **extra)


def _assert_bitwise(got, want, rows=slice(None)):
    assert list(got) == list(want)
    for k in want:
        w = want[k][rows]
        assert got[k].shape == w.shape and got[k].dtype == w.dtype and got[k].device == w.device, k
        assert not torch.isnan(w).any(), k
        diff = got[k] != w
        assert not diff.any(), (k, int(diff.sum()), (got[k] - w).abs().max().item())


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_frame_equals_the_chunked_route_at_every_chunk_size(scene, name, precision):
    kw = _kw(scene, name, precision)
    want = _chunked_route(scene, kw)
    assert want["rgb_coarse"].std().item() > 1e-3                     # the frame has structure
    for chunk_rays in (1000, 4096, 65536):
        _assert_bitwise(_frame(scene, kw, chunk_rays=chunk_rays), want)
    if name == "missed_box_coarse_only":
        obj, z = want["obj_ids_coarse"], want["z_vals_coarse"]
        assert (z[obj == 2] == 0).all()                                # set 2 (id 9): no ray hits its box
        assert (z[obj == 1] > 0).any() and (z[obj == 1] == 0).any()    # set 1 (id 6): some rays do


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_tiles_are_rows_of_the_frame(scene, precision):
    from object_nerf_b200 import editing
    kw = _kw(scene, "dup_moved_removed", precision)
    want = _chunked_route(scene, kw)
    sets = kw.pop("sets")
    for begin, end, chunk in ((0, 0, 1000), (2000, 2000, 4096), (17, 18, 1000), (H * W - 1, H * W, 4096),
                              (1000, 3333, 1000), (123, 4567, 4096), (4096, H * W, 1000), (1, H * W, 65536)):
        got = editing.render_tile(scene["models"], scene["emb"], scene["lib"], H, W, FOCAL, sets, NEAR, FAR, SF, begin, end,
                                  chunk_rays=chunk, **kw)
        _assert_bitwise(got, want, slice(begin, end))


@pytest.mark.parametrize("keys", [["rgb_fine", "depth_fine"], ["weights_coarse", "obj_ids_coarse", "z_vals_fine"],
                                  ["opacity_coarse"]])
def test_keys_subset_equals_the_full_call(scene, keys):
    kw = _kw(scene, "dup_moved_removed", "bf16")
    full = _frame(scene, kw, chunk_rays=1000)
    got = _frame(scene, kw, chunk_rays=1000, keys=keys)
    assert list(got) == [k for k in full if k in keys]
    for k in keys:
        assert torch.equal(got[k], full[k]), k


def test_refusals(scene):
    from object_nerf_b200 import editing
    kw = _kw(scene, "dup_moved_removed", "bf16")
    sets = kw.pop("sets")
    ok = lambda **o: editing.render_tile(scene["models"], scene["emb"], scene["lib"], o.pop("H", H), o.pop("W", W),
                                         o.pop("focal", FOCAL), o.pop("sets", sets), NEAR, FAR, o.pop("sf", SF),
                                         o.pop("begin", 0), o.pop("end", 64), **{**kw, **o})
    assert ok()["rgb_fine"].shape == (64, 3)
    box = sets[1][2]
    bad = {
        "tile outside the frame": [dict(begin=-1), dict(begin=5, end=4), dict(end=H * W + 1)],
        "chunk_rays < 1": [dict(chunk_rays=0), dict(chunk_rays=-7)],
        "an object set needs its box": [dict(sets=[sets[0], (4, sets[1][1], None, 0.0)])],
        "the scene set takes no box": [dict(sets=[(0, sets[0][1], box, 0.0)] + sets[1:])],
        "bad camera": [dict(focal=0.0), dict(H=0, end=0), dict(W=-3, end=0)],
        "scale_factor": [dict(sf=0.0)],
        "bad shape": [dict(sets=[])],
        "object id outside the code table": [dict(sets=[sets[0], (64, sets[1][1], box, 0.0)])],
        "2048": [dict(N_samples=1024, N_importance=1025, chunk_rays=16)],
    }
    for msg, cases in bad.items():
        for o in cases:
            with pytest.raises(RuntimeError, match=msg):
                ok(**o)
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------
# against the unmodified EditableRenderer over dropin.install()
# ------------------------------------------------------------------------------------------------
def _ref_renderer(er, conf, paths, obj_ids):
    cfg = R.to_attr({"chunk": 256, "img_wh": [32, 24], "ckpt_path": paths["ckpt"], "ckpt_config_path": paths["snapshot"],
                     "obj_id_list": obj_ids, "edit_type": "duplication", "test_frame": 1, "ckpt_config": conf})
    r = er.EditableRenderer(config=cfg)
    r.load_frame_meta()
    for obj_id in obj_ids:
        r.initialize_object_bbox(obj_id)
    r.remove_scene_object_by_ids(obj_ids)
    return r, cfg


def _set_poses(r, obj_ids, progress):
    """test/demo_editable_render.py:60-78 with edit_type "duplication"."""
    processed = []
    for obj_id in obj_ids:
        dup = np.sum(np.array(processed) == obj_id)
        t = np.eye(4)
        a = np.sin(progress * np.pi * 2) * np.radians(10)
        t[:2, :2] = [[np.cos(a), -np.sin(a)], [np.sin(a), np.cos(a)]]
        sgn = -1 if dup > 0 else 1
        t[0, 3] += sgn * np.sin(progress * np.pi * 2) * 0.05
        t[1, 3] += -0.2 if dup > 0 else 0.55
        r.set_object_pose_transform(obj_id, t, dup)
        processed.append(obj_id)


def _hit_sets(res, n_sets):
    """(n_sets, N) bool: which sets' rays hit their box (a missed object set's samples all sit at depth 0)."""
    z, ids = res["z_vals_coarse"], res["obj_ids_coarse"]
    return torch.stack([((ids == k) & (z == 0)).sum(1) == 0 for k in range(n_sets)])


TOL = {"fp32": (2e-4, 5e-3, 5e-2), "bf16": (3e-2, 2e-2, 0.3)}   # per-value tolerance, outlier share, outlier bound


def _close(k, got, want, precision):
    tol, share, bound = TOL[precision]
    err = (got.float() - want.float()).abs()
    frac, worst = (err > tol).float().mean().item(), err.max().item()
    print(f"[{precision}] {k}: max |diff| {worst:.3g}, share above {tol:g}: {frac:.4f}")
    assert frac <= share and worst <= bound, (k, frac, worst)


@pytest.mark.skipif(not R.available(), reason="oracle/_ref not built (needs the reference checkout at build time)")
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_against_the_unmodified_renderer_over_dropin(tmp_path, precision, monkeypatch):
    import object_nerf_b200.dropin as dropin
    from object_nerf_b200 import editing
    from tests import dropin_fixture as F
    monkeypatch.setenv("ONERF_PRECISION", precision)
    try:
        F.purge_reference_modules()
        R.install(cuda_noop=True)
        conf, paths = F.write_scene(str(tmp_path))
        train, system = F.make_system(conf, "cpu")
        F.fill_synthetic_weights(system)
        torch.save({"state_dict": system.state_dict()}, paths["ckpt"])
        F.purge_reference_modules()
        R.cuda_noop(False)
        dropin.install()
        from render_tools import editable_renderer as er
        assert er.render_rays_multi.__module__ == "object_nerf_b200.multi_rendering"
        obj_ids = [4, 4]
        r, cfg = _ref_renderer(er, conf, paths, obj_ids)
        Wd, Hd = cfg.img_wh
        unmodified_edit, unmodified_origin = er.EditableRenderer.render_edit, er.EditableRenderer.render_origin
        _set_poses(r, obj_ids, 0.3)
        pose = r.get_camera_pose_by_frame_idx(cfg.test_frame)
        for kw in ({}, {"render_obj_only": True}, {"render_bg_only": True}):
            active = list(r.active_object_ids)
            want = unmodified_edit(r, h=Hd, w=Wd, camera_pose_Twc=pose.copy(), fovx_deg=r.fov_x_deg_dataset,
                                   show_progress=False, **kw)
            after_ref = list(r.active_object_ids)
            r.active_object_ids = active
            got = editing.render_edit(r, Hd, Wd, pose.copy(), r.fov_x_deg_dataset, show_progress=False, **kw)
            assert r.active_object_ids == after_ref
            assert list(got) == list(want)
            for k in want:
                assert (got[k].shape, got[k].dtype, got[k].device) == (want[k].shape, want[k].dtype, want[k].device), k
            n_sets = len(r.active_object_ids)
            assert torch.equal(_hit_sets(got, n_sets), _hit_sets(want, n_sets))
            for k in ("rgb_fine", "depth_fine", "opacity_fine", "rgb_coarse", "depth_coarse", "weights_fine"):
                _close(f"render_edit{kw} {k}", got[k], want[k], precision)
            r.active_object_ids = active
        r.reset_active_object_ids()
        want = unmodified_origin(r, h=Hd, w=Wd, camera_pose_Twc=pose.copy(), fovx_deg=r.fov_x_deg_dataset)
        got = editing.render_origin(r, Hd, Wd, pose.copy(), r.fov_x_deg_dataset)
        assert list(got) == list(want)
        for k in want:
            assert (got[k].shape, got[k].dtype, got[k].device) == (want[k].shape, want[k].dtype, want[k].device), k
        for k in ("rgb_fine", "depth_fine", "opacity_fine", "rgb_coarse"):
            _close(f"render_origin {k}", got[k], want[k], precision)
        # the demo's duplication loop (test/demo_editable_render.py:56-103) through editing.install
        editing.install(er.EditableRenderer)
        for idx in range(2):
            _set_poses(r, obj_ids, idx / 2)
            cam = r.get_camera_pose_by_frame_idx(cfg.test_frame)
            want = unmodified_edit(r, h=Hd, w=Wd, camera_pose_Twc=cam.copy(), fovx_deg=r.fov_x_deg_dataset,
                                   show_progress=False)
            results = r.render_edit(h=Hd, w=Wd, camera_pose_Twc=cam.copy(), fovx_deg=getattr(r, "fov_x_deg_dataset", 60))
            image = results["rgb_fine"].view(Hd, Wd, 3).detach().cpu().numpy()
            assert image.shape == (Hd, Wd, 3) and image.std() > 0.02
            _close(f"demo frame {idx} rgb_fine", results["rgb_fine"], want["rgb_fine"], precision)
            r.reset_active_object_ids()
    finally:
        F.purge_reference_modules()
        R.cuda_noop(not torch.cuda.is_available())


# ------------------------------------------------------------------------------------------------
# sharding
# ------------------------------------------------------------------------------------------------
def _shard_worker(rank, world, port, backend, ret):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dev = torch.device("cuda", rank % torch.cuda.device_count())
    torch.cuda.set_device(dev)
    dist.init_process_group(backend, rank=rank, world_size=world)
    try:
        sc = _make_scene(dev)
        kw = _kw(sc, "dup_moved_removed", "bf16")
        single = _frame(sc, kw, chunk_rays=1000)
        gathered = _frame(sc, kw, chunk_rays=1000, group=dist.group.WORLD)
        bad = [k for k in single if not torch.equal(single[k], gathered[k])]
        ret[rank] = (list(gathered) == list(single), bad, str(gathered["rgb_fine"].device))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("backend", ["gloo", "nccl"])
def test_sharded_frame_equals_the_single_process_frame(backend):
    import torch.multiprocessing as mp
    world = 2
    if backend == "nccl" and torch.cuda.device_count() < 2:
        pytest.skip("NCCL across devices needs two GPUs")
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    ctx = mp.get_context("spawn")
    ret = ctx.Manager().dict()
    procs = [ctx.Process(target=_shard_worker, args=(r, world, port, backend, ret)) for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=300)
        assert p.exitcode == 0
    assert len(ret) == world
    for rank, (same_keys, bad, device) in ret.items():
        assert same_keys and not bad and device == f"cuda:{rank % torch.cuda.device_count()}", (rank, bad, device)
