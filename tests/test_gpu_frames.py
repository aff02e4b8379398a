"""The frame-store batch draw on the GPU (onerf_draw_frames / _dstep, RaySampler.from_frames): every field of every
drawn row equals the host restatement of tests/frames_cases.py at the (ray, column) pairs tests/test_batches_cpu.py
restates; from_frames draws RaySampler(fs.expand())'s batches bit for bit, eagerly and on graph replay; the rows match
the reference's own buffers (golden fixtures); a captured from_frames + train_step + Adam loop trains; the store holds
about 9 bytes per pixel."""
import ctypes as C
import math
import os

import numpy as np
import pytest
import torch

from tests import cases, helpers
from tests import frames_cases as FC
from tests.test_batches_cpu import draw_indices

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SEED = 0x0123_4567_89AB_CDEF
RAYS_D_TOL = 2.5e-7
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _rotation(rng):
    q, r = np.linalg.qr(rng.normal(size=(3, 3)))
    return q * np.sign(np.diag(r))


def _inputs(F, H, W, I, label_dtype=np.uint16, border=20, seed=0, counts=True):
    """FrameSet keyword arguments of a random scene: labels in [0, 8) (plus 40000 with uint16), column 0 all ones."""
    rng = np.random.default_rng(seed)
    poses = np.stack([np.concatenate([_rotation(rng), rng.normal(size=(3, 1))], 1) for _ in range(F)]).astype(np.float32)
    hi = 8
    labels = rng.integers(0, hi, size=(F, H, W))
    if label_dtype == np.uint16:
        labels[:, :2, :3] = 40000
    ids = [0, 3, 40000, 5, 1][:I]
    return dict(poses=poses, rgb=rng.integers(0, 256, size=(F, H, W, 3), dtype=np.uint8),
                depths=rng.uniform(0, 3, size=(F, H, W)).astype(np.float32), labels=labels.astype(label_dtype),
                focal=0.7 * W, near=0.1, far=5.0, scale_factor=1.7, instance_ids=ids, bg_instance_ids=[2, 7],
                use_instance_mask=True, fg_weight=None if counts else 2.0, bg_weight=None if counts else 0.25,
                frame_idx=np.arange(F) * 3 + 11, border=border)


def _frame_set(inp):
    from object_nerf_b200.frames import FrameSet
    return FrameSet(**inp, device=DEV)


def _draw(s, step, dstep=None):
    """onerf_draw_frames at `step` with index_out; -> (index, batch)."""
    from object_nerf_b200 import _lib
    idx = torch.full((s.batch_size, 2), -7, dtype=torch.int64, device=DEV)
    a = _lib.BatchArgs.from_buffer_copy(s._args)
    a.step, a.index_out = step, idx.data_ptr()
    lib, ctx = _lib.load(), _lib.ctx(torch.device(DEV))
    if dstep is None:
        _lib.check(lib.onerf_draw_frames(ctx, C.byref(s.frames.args), C.byref(a), _lib.stream()))
    else:
        _lib.check(lib.onerf_draw_frames_dstep(ctx, C.byref(s.frames.args), C.byref(a), dstep.data_ptr(),
                                               _lib.stream()))
    torch.cuda.synchronize()
    return idx, {k: v.clone() for k, v in s._batch.items()}


def _assert_rows(want, idx, batch, rays_d_exact=False):
    """The batch rows equal the all_* buffers `want` (host tensors) at the (ray, column) pairs."""
    ray, col = idx[:, 0].cpu(), idx[:, 1].cpu()
    b = {k: v.cpu() for k, v in batch.items()}
    B = ray.numel()
    r = want["all_rays"][ray]
    assert torch.equal(b["rays"][:, [0, 1, 2, 6, 7]], r[:, [0, 1, 2, 6, 7]])
    if rays_d_exact:
        assert torch.equal(b["rays"][:, 3:6], r[:, 3:6])
    else:
        assert (b["rays"][:, 3:6] - r[:, 3:6]).abs().max().item() <= RAYS_D_TOL
    assert torch.equal(b["rgbs"], want["all_rgbs"][ray])
    assert torch.equal(b["depths"], want["all_depths"][ray])
    assert torch.equal(b["valid_mask"], want["all_valid_masks"][ray].bool())
    assert torch.equal(b["frame_idx"], want["all_frame_indices"][ray])
    for k, key in (("instance_mask", "all_instance_masks"), ("instance_mask_weight", "all_instance_masks_weight"),
                   ("instance_ids", "all_instance_ids"), ("pass_through_mask", "all_pass_through_masks")):
        w = FC.as_sampler_dtypes(want[key], key)[ray, col].view(B, 1)
        assert torch.equal(b[k], w), k


@pytest.mark.parametrize("I", [1, 3, 5])
@pytest.mark.parametrize("W", [1, 2, 3])
def test_kernel_matches_the_host_restatement(I, W):
    """H*W = 437 (not a multiple of 128), border 12 >= H/2 on the u8 scene (no valid pixel), 3 on the u16 one."""
    from object_nerf_b200 import RaySampler
    for label_dtype, border, counts in ((np.uint8, 12, True), (np.uint16, 3, False)):
        inp = _inputs(7, 19, 23, I, label_dtype, border, seed=I * 10 + W, counts=counts)
        fs = _frame_set(inp)
        want = FC.expand_host(inp)
        R, B = fs.n_rays, 256
        for rank in range(W):
            s = RaySampler.from_frames(fs, batch_size=B, seed=SEED, rank=rank, world_size=W)
            P = s.batches_per_epoch
            for step in sorted({0, P - 1, P, 2 * P + 1}):
                idx, batch = _draw(s, step)
                ray, col = draw_indices(R, fs.n_instances, B, W, rank, SEED, step)
                assert np.array_equal(idx[:, 0].cpu().numpy(), ray), (rank, step)
                assert np.array_equal(idx[:, 1].cpu().numpy(), col), (rank, step)
                _assert_rows(want, idx, batch)


def test_expand_equals_the_host_restatement():
    for label_dtype in (np.uint8, np.uint16):
        inp = _inputs(3, 17, 29, 5, label_dtype, border=4)
        got = _frame_set(inp).expand()
        want = FC.expand_host(inp)
        for k, v in want.items():
            g = got[k].cpu()
            if k == "all_rays":
                assert torch.equal(g[:, [0, 1, 2, 6, 7]], v[:, [0, 1, 2, 6, 7]])
                assert (g[:, 3:6] - v[:, 3:6]).abs().max().item() <= RAYS_D_TOL
            else:
                assert torch.equal(FC.as_sampler_dtypes(g, k), FC.as_sampler_dtypes(v, k)), k


def _clone(batch):
    return {k: v.clone() for k, v in batch.items()}


def test_from_frames_draws_the_expanded_samplers_batches():
    """Two epochs eagerly, a set_step jump, and graph replays: bit-identical batches, rays included."""
    from object_nerf_b200 import RaySampler
    fs = _frame_set(_inputs(5, 31, 37, 3, np.uint16, border=5))
    ex = fs.expand()
    a = RaySampler.from_frames(fs, batch_size=512, seed=SEED)
    e = RaySampler(ex, batch_size=512, device=DEV, seed=SEED)
    assert a.batches_per_epoch == e.batches_per_epoch and a.n_instances == e.n_instances == 3
    for _ in range(2 * a.batches_per_epoch + 1):
        x, y = _clone(a.next()), e.next()
        for k in y:
            assert torch.equal(x[k], y[k]), k
    assert a.step == e.step and a.epoch == e.epoch == 2
    a.set_step(17)
    e.set_step(17)
    x, y = _clone(a.next()), e.next()
    for k in y:
        assert torch.equal(x[k], y[k]), k
    # graph replay
    g_s = RaySampler.from_frames(fs, batch_size=512, seed=SEED)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        g_s.next()
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = g_s.next()
    e.set_step(1)
    for k in range(1, 2 * g_s.batches_per_epoch + 3):
        g.replay()
        want = e.next()
        for key in want:
            assert torch.equal(out[key], want[key]), (k, key)
    assert g_s.step == e.step


def test_device_step_draws_what_the_host_step_draws():
    from object_nerf_b200 import RaySampler
    s = RaySampler.from_frames(_frame_set(_inputs(4, 20, 30, 2)), batch_size=300, seed=7)
    for k in (0, 3, s.batches_per_epoch, 500):
        counter = torch.full((1,), k, dtype=torch.int64, device=DEV)
        idx_d, batch_d = _draw(s, 12345, dstep=counter)
        idx_h, batch_h = _draw(s, k)
        assert torch.equal(idx_d, idx_h)
        for key in batch_h:
            assert torch.equal(batch_d[key], batch_h[key]), key
        assert counter.item() == k + 1


@pytest.mark.parametrize("name", ["i1_counts", "i3_bg_obs"])
def test_rows_equal_the_reference_buffers(name):
    """Frames decoded from the fixture's dataset and the buffers the reference's GenericDataset built from them."""
    from object_nerf_b200 import RaySampler
    g = np.load(os.path.join(GOLDEN, f"frames_{name}.npz"))
    inp = {k[3:]: g[k] for k in g.files if k.startswith("in_")}
    inp.setdefault("labels", None)
    for k in ("focal", "near", "far", "scale_factor", "border", "use_instance_mask"):
        inp[k] = inp[k].item()
    for k in ("fg_weight", "bg_weight"):
        inp[k] = inp[k].item() if k in inp else None
    inp["instance_ids"], inp["bg_instance_ids"] = inp["instance_ids"].tolist(), inp["bg_instance_ids"].tolist()
    fs = _frame_set(inp)
    want = {k[4:]: torch.from_numpy(g[k]) for k in g.files if k.startswith("ref_")}
    assert fs.n_rays == want["all_rays"].shape[0]
    s = RaySampler.from_frames(fs, batch_size=1000, seed=SEED)
    for step in range(2 * s.batches_per_epoch + 1):
        idx, batch = _draw(s, step)
        _assert_rows(want, idx, batch)


def test_store_holds_about_nine_bytes_per_pixel():
    F, H, W, I = 6, 48, 64, 5
    fs = _frame_set(_inputs(F, H, W, I))
    per_frame = 12 * 4 + 8 + I * 2 * 4
    per_column = 8 + 1 + 4 * 3
    assert fs.nbytes <= 9 * F * H * W + 12 * H * W + F * per_frame + I * per_column
    ex = fs.expand()
    expanded = sum(t.numel() * t.element_size() for t in ex.values())
    assert expanded > 8 * fs.nbytes


def _training_inputs(F=8, H=48, W=64):
    """Frames of the synthetic scene's camera (synthetic.pinhole_rays), jittered per frame, with a constant colour and
    depth target."""
    rng = np.random.default_rng(3)
    poses = []
    for _ in range(F):
        cam = np.array([-1.6, 0.1, 0.15]) + rng.normal(size=3) * 0.05
        fwd = -cam / np.linalg.norm(cam)
        right = np.cross(fwd, [0.0, 0.0, 1.0])
        right /= np.linalg.norm(right)
        up = np.cross(right, fwd)
        poses.append(np.concatenate([np.stack([right, up, -fwd], 1), cam[:, None]], 1))
    rgb = np.broadcast_to(np.array([204, 102, 51], np.uint8), (F, H, W, 3)).copy()
    labels = rng.choice([4, 6], size=(F, H, W)).astype(np.uint16)
    return dict(poses=np.stack(poses).astype(np.float32), rgb=rgb, depths=np.full((F, H, W), 1.5, np.float32),
                labels=labels, focal=0.5 * W / math.tan(math.radians(30)), near=0.15, far=3.0, scale_factor=1.0,
                instance_ids=[4, 6], use_instance_mask=True, border=0)


def test_captured_training_loop_trains():
    """from_frames' next() + train_step + Adam(capturable=True) captured once and replayed 200 times: the replays
    draw an eager sampler's batches step for step, and the colour term of the last 20 replays is below that of the
    first 20."""
    from object_nerf_b200 import Embedding, RaySampler, training
    inp = cases.build_grad_case()
    fs = _frame_set(_training_inputs())
    B = 1024
    s = RaySampler.from_frames(fs, batch_size=B, seed=SEED)
    e = RaySampler.from_frames(fs, batch_size=B, seed=SEED)
    models = {k: helpers.make_model(w, True, DEV).train() for k, w in inp["weights"].items()}
    embeddings = {"xyz": helpers.GridModule(inp["grid"]).to(DEV), "dir": Embedding(3, 4)}
    lib = helpers.CodeLib(inp["code_table"]).to(DEV)
    params = [p for m in models.values() for p in m.parameters()] + list(lib.parameters()) + \
        list(embeddings["xyz"].parameters())
    opt = torch.optim.Adam(params, lr=5e-3, capturable=True)
    kw = dict(N_samples=64, N_importance=64, perturb=1.0, noise_std=1.0, frustum_bound_th=0.025, is_eval=False,
              precision="bf16")

    def step():
        batch = s.next()
        opt.zero_grad(set_to_none=False)
        res = training.train_step(models, embeddings, lib, batch, cases.LOSS_CONF,
                                  pass_through_mask=batch["pass_through_mask"], **kw)
        opt.step()
        return batch, res

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(3):
            step()
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        batch, (_, terms, present, _) = step()
    e.set_step(3)
    color = []
    for k in range(200):
        g.replay()
        want = e.next()
        for key in want:
            assert torch.equal(batch[key], want[key]), (k, key)
        color.append(terms[0].item())
    assert present[0].item() == 1
    assert s.step == 203
    first, last = np.mean(color[:20]), np.mean(color[-20:])
    assert last < first, (first, last)
