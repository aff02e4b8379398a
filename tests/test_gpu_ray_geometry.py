"""-m gpu: camera rays and the ray-box slab test against the references of tests/test_ray_geometry_cpu.py.

Entries: generate_rays (scene and object), get_ray_bbox_intersections, get_ray_directions, get_rays, camera_rays.
Inputs: the planted geometry; build_bbox_case and three box variants (yaw-only, signed axis permutation, rotated
pose_avg) at n in {1, 255, 257, W - 1, W + 1, 3W + 5} with W = num_sms 8 256 rays (one grid-stride wave) and at
1 000 003 rays; frames from 1x1 to 1080x1920 of a level camera and a yaw-only box, where row H / 2 of an even-height frame
has an exactly-zero box-frame dz on every pixel.  Outputs are prefilled with NaN (0xCD for hit masks) one row past n:
every row must be written and nothing past it; rays are bit-identical with and without the hit mask.
Each case prints its knife-edge count and RATIO label: x, the largest share of the rays_d gate used."""
import ctypes as C

import numpy as np
import pytest
import torch

from object_nerf_b200 import _lib, ray_utils
from tests.test_ray_geometry_cpu import (F32, PLANTED, RANDOM_BOXES, Box, bits, box_rays, directions_f32, golden_box,
                                         level_c2w, planted_rays, random_box, rays_d_ratio, reference, rigid,
                                         scene_near_far, slab_verdict, yaw)

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
NAN_BITS = 0x7FC00000
NEAR, FAR = 0.3, 7.0


def wave():
    return torch.cuda.get_device_properties(DEV).multi_processor_count * 8 * 256


def _box_arg(box):
    return C.byref(ray_utils._box_host(box, box.bbox_enlarge)) if box is not None else None


def _canvas(n):
    out = torch.full((n + 1, 8), float("nan"), device=DEV)
    hit = torch.full((n + 1,), 0xCD, dtype=torch.uint8, device=DEV)
    return out, hit


def _check_canvas(out, hit, n):
    """Row n and byte n untouched; every hit byte 0 / 1.  Returns the n rows and the hit mask on the host."""
    torch.cuda.synchronize()
    o = out.cpu().numpy()
    assert (o[n].view(np.uint32) == NAN_BITS).all(), "a row past n was written"
    h = None
    if hit is not None:
        hb = hit.cpu().numpy()
        assert hb[n] == 0xCD, "a hit byte past n was written"
        assert np.isin(hb[:n], (0, 1)).all(), "a hit byte was not written"
        h = hb[:n].astype(bool)
    return o[:n], h


def generate(o, d, box, scale):
    """onerf_generate_rays with and without the hit mask on canvases; checks the canaries and that both agree."""
    o, d = np.ascontiguousarray(o, F32), np.ascontiguousarray(d, F32)
    n = o.shape[0]
    og, dg = torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV)
    res = []
    for with_hit in (True, False):
        out, hit = _canvas(n)
        hit = hit if with_hit else None
        _lib.check(_lib.load().onerf_generate_rays(_lib.ctx(DEV), og.data_ptr(), dg.data_ptr(), n, _box_arg(box),
                                                   float(scale), NEAR, FAR, out.data_ptr(), _lib.ptr(hit), _lib.stream()))
        res.append(_check_canvas(out, hit, n))
    (rows, h), (rows2, _) = res
    assert np.array_equal(rows.view(np.uint32), rows2.view(np.uint32)), "rays differ with and without hit_out"
    assert np.array_equal(rows[:, :3].view(np.uint32), o.view(np.uint32))
    assert np.array_equal(rows[:, 3:6].view(np.uint32), d.view(np.uint32))
    return rows, h


def check_object_rays(label, o, d, box, sample=2000):
    rows, h = generate(o, d, box, box.scale_factor)
    want = reference(o, d, box, sample=sample, seed=len(o))
    n_sure = slab_verdict(h, rows[:, 6], rows[:, 7], want)
    print(f"{label}: n={len(o)} decidable {n_sure}, knife-edge {want['n_knife']}, exact {want['n_exact']}, "
          f"hits {int(h.sum())}")
    return want


def check_scene_rays(o, d, scale):
    rows, h = generate(o, d, None, scale)
    n32, f32 = scene_near_far(NEAR, FAR, scale)
    assert h.all()
    assert (rows[:, 6].view(np.uint32) == bits(n32)).all() and (rows[:, 7].view(np.uint32) == bits(f32)).all()


@pytest.mark.parametrize("name", list(PLANTED))
def test_planted_geometry(name):
    box = PLANTED[name][0]
    o, d, _ = planted_rays(name)
    want = check_object_rays(f"planted {name}", o, d, box, sample=len(o))
    assert want["sure"].all()
    # the Python entries: get_ray_bbox_intersections and generate_rays give the same rows
    og, dg = torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV)
    mask, near, far = ray_utils.get_ray_bbox_intersections(box, og, dg, box.scale_factor, box.bbox_enlarge)
    slab_verdict(mask.cpu().numpy(), near.cpu().numpy().reshape(-1), far.cpu().numpy().reshape(-1), want)
    rays, m = ray_utils.generate_rays(3, og, dg, NEAR, FAR, box.scale_factor, box=box, bbox_enlarge=box.bbox_enlarge,
                                      return_mask=True)
    slab_verdict(m.cpu().numpy(), rays[:, 6].cpu().numpy(), rays[:, 7].cpu().numpy(), want)
    rays0 = ray_utils.generate_rays(0, og, dg, NEAR, FAR, box.scale_factor)
    n32, f32 = scene_near_far(NEAR, FAR, box.scale_factor)
    assert (rays0[:, 6].cpu().numpy().view(np.uint32) == bits(n32)).all()
    assert (rays0[:, 7].cpu().numpy().view(np.uint32) == bits(f32)).all()


def _boxes():
    out = {name: golden_box(name)[0] for name in ("bbox_basic", "bbox_enlarged")}
    out.update({kind: random_box(kind, seed) for kind, seed in RANDOM_BOXES.items()})
    return out


@pytest.mark.parametrize("name", ["bbox_basic", "bbox_enlarged"])
def test_golden_box_cases(name):
    box, o, d = golden_box(name)
    want = check_object_rays(name, o, d, box, sample=len(o))
    assert want["n_knife"] == 0


def test_launch_shapes():
    """n around one grid-stride wave, each n on a different box variant; scene rays at every n with a scale that makes
    near / scale and far / scale inexact."""
    W = wave()
    boxes = list(_boxes().items())
    for k, n in enumerate((1, 255, 257, W - 1, W + 1, 3 * W + 5)):
        name, box = boxes[k % len(boxes)]
        o, d = box_rays(box, n, 700 + k)
        want = check_object_rays(f"{name} n={n}", o, d, box, sample=min(n, 1000))
        assert want["n_knife"] == 0
        check_scene_rays(o, d, 3.0)


def test_million_rays():
    """1 000 003 rays on the rotated-pose_avg box; the exact check on 20 000 of them plus every flagged one."""
    box = random_box("pose_rot", RANDOM_BOXES["pose_rot"])
    o, d = box_rays(box, 1_000_003, 801)
    want = check_object_rays("pose_rot n=1000003", o, d, box, sample=20_000)
    # a random t lies within beta (here up to ~2e-14 relative) of an fp32 midpoint with probability ~2 beta / ulp: about
    # one ray in a million; such a ray is held to the two neighbouring values instead
    assert want["n_knife"] <= 2 and want["n_exact"] >= 20_000


def _frame_box(scale):
    """A yaw-only box around the world point (0, 2, 0.1) (a level camera at the origin looking along +y sees it)."""
    A = rigid(yaw(0.4))
    A[:3, 3] = -(A[:3, :3] @ np.array([0.0, 2.0, 0.1]) * scale)
    return Box(rigid(None, (0.0, 0.0, 0.0)), A, [[-0.6, -0.5, -0.4], [0.7, 0.6, 0.5]], scale)


@pytest.mark.parametrize("HW", [(1, 1), (1, 641), (641, 1), (37, 53), (480, 640), (1080, 1920)])
def test_camera_frames(HW):
    """get_ray_directions, get_rays and camera_rays on a level camera: directions and rays_o bit for bit, rays_d inside
    its gate, near / far of every ray against the slab reference evaluated on the kernel's own rays."""
    H, W = HW
    focal = (W / 2) / np.tan(np.radians(35.0)) if W > 1 else 1.5
    c2w = level_c2w(10.0, (0.0, 0.0, 0.05))          # level, looking 10 degrees off +y
    box = _frame_box(2.0)
    n = H * W
    # get_ray_directions into a canvas one pixel longer
    dirs = torch.full(((n + 1) * 3,), float("nan"), device=DEV)
    _lib.check(_lib.load().onerf_ray_directions(_lib.ctx(DEV), H, W, float(focal), dirs.data_ptr(), _lib.stream()))
    torch.cuda.synchronize()
    dh = dirs.cpu().numpy()
    assert (dh[3 * n:].view(np.uint32) == NAN_BITS).all()
    want_dirs = directions_f32(H, W, focal).reshape(-1)
    assert np.array_equal(dh[:3 * n].view(np.uint32), want_dirs.view(np.uint32))
    assert torch.equal(ray_utils.get_ray_directions(H, W, focal, device=DEV).cpu().reshape(-1), dirs.cpu()[:3 * n])
    # get_rays into canvases
    ro = torch.full(((n + 1), 3), float("nan"), device=DEV)
    rd = torch.full(((n + 1), 3), float("nan"), device=DEV)
    cw = (C.c_float * 12)(*c2w.numpy().reshape(-1).tolist())
    _lib.check(_lib.load().onerf_get_rays(_lib.ctx(DEV), dirs.data_ptr(), n, cw, ro.data_ptr(), rd.data_ptr(), _lib.stream()))
    torch.cuda.synchronize()
    roh, rdh = ro.cpu().numpy(), rd.cpu().numpy()
    assert (roh[n].view(np.uint32) == NAN_BITS).all() and (rdh[n].view(np.uint32) == NAN_BITS).all()
    assert np.array_equal(roh[:n], np.broadcast_to(c2w.numpy()[:, 3], (n, 3)))
    r = rays_d_ratio(rdh[:n], want_dirs, c2w.numpy())
    # camera_rays with and without the hit mask
    res = []
    for with_hit in (True, False):
        out, hit = _canvas(n)
        hit = hit if with_hit else None
        _lib.check(_lib.load().onerf_camera_rays(_lib.ctx(DEV), H, W, float(focal), cw, _box_arg(box), box.scale_factor,
                                                 NEAR, FAR, out.data_ptr(), _lib.ptr(hit), _lib.stream()))
        res.append(_check_canvas(out, hit, n))
    (rows, h), (rows2, _) = res
    assert np.array_equal(rows.view(np.uint32), rows2.view(np.uint32))
    assert np.array_equal(rows[:, :3], roh[:n]) and np.array_equal(rows[:, 3:6].view(np.uint32), rdh[:n].view(np.uint32))
    want = reference(rows[:, :3].copy(), rows[:, 3:6].copy(), box, sample=min(n, 2000), seed=n)
    n_sure = slab_verdict(h, rows[:, 6], rows[:, 7], want)
    # the scene route of the same frame
    scene = ray_utils.camera_rays(H, W, focal, c2w, NEAR, FAR, box.scale_factor, device=DEV).cpu().numpy()
    n32, f32 = scene_near_far(NEAR, FAR, box.scale_factor)
    assert np.array_equal(scene[:, :6].view(np.uint32), rows[:, :6].view(np.uint32))
    assert (scene[:, 6].view(np.uint32) == bits(n32)).all() and (scene[:, 7].view(np.uint32) == bits(f32)).all()
    zero_dz = 0
    if H % 2 == 0:
        mid = rows[(H // 2) * W:(H // 2 + 1) * W, 5]
        assert (mid == 0).all()                        # world dz, and so box-frame dz, exactly zero on row H / 2
        zero_dz = int(h[(H // 2) * W:(H // 2 + 1) * W].sum())
    print(f"frame {H}x{W}: decidable {n_sure}, knife-edge {want['n_knife']}, hits {int(h.sum())}, "
          f"row H/2 hits through the 1e-14 rule {zero_dz}; RATIO rays_d {H}x{W}: {r:.3e}")
    assert r <= 1 and want["n_knife"] == 0
    if H * W >= 480 * 640:
        assert h.any() and (~h).any() and zero_dz > 0


def test_get_rays_zero_length_direction():
    """A zero-length camera direction normalises to NaN, as the reference's torch code gives."""
    x = torch.tensor([[0.0, 0.0, 0.0], [0.25, -0.5, -1.0]], device=DEV)
    c2w = level_c2w(30.0, (0.5, -0.25, 1.0))
    _, rd = ray_utils.get_rays(x, c2w)
    rd = rd.cpu()
    assert torch.isnan(rd[0]).all() and not torch.isnan(rd[1]).any()
    assert rays_d_ratio(rd.numpy(), x.cpu().numpy(), c2w.numpy()) <= 1
