"""The device batch sampler on the GPU (onerf_draw_batch / _dstep, batches.RaySampler): the kernel's (ray, column) pairs
equal the numpy restatement of tests/test_batches_cpu.py bit for bit, every output field is plain indexing of the
uploaded buffers, one epoch covers P*B*W distinct rays across ranks, the column draw is uniform, graph replays draw what
eager calls draw, and a captured sampler + train_step + Adam loop trains."""
import ctypes as C

import numpy as np
import pytest
import torch
from scipy import stats

from tests import cases, helpers
from tests.test_batches_cpu import dataset, draw_indices

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SEED = 0x0123_4567_89AB_CDEF


def _sampler(t, **kw):
    from object_nerf_b200 import RaySampler
    return RaySampler(t, device=DEV, **kw)


def _draw(s, step, dstep=None):
    """onerf_draw_batch at `step` (or onerf_draw_batch_dstep on the counter `dstep`) with index_out; -> (index, batch)."""
    from object_nerf_b200 import _lib
    idx = torch.full((s.batch_size, 2), -7, dtype=torch.int64, device=DEV)
    a = _lib.BatchArgs.from_buffer_copy(s._args)
    a.step, a.index_out = step, idx.data_ptr()
    lib, ctx = _lib.load(), _lib.ctx(torch.device(DEV))
    if dstep is None:
        _lib.check(lib.onerf_draw_batch(ctx, C.byref(a), _lib.stream()))
    else:
        _lib.check(lib.onerf_draw_batch_dstep(ctx, C.byref(a), dstep.data_ptr(), _lib.stream()))
    torch.cuda.synchronize()
    return idx, {k: v.clone() for k, v in s._batch.items()}


def _assert_gathered(s, idx, batch):
    """Every field is torch indexing of the uploaded buffers at the (ray, column) pairs."""
    buf = s.buffers
    ray, col = idx[:, 0], idx[:, 1]
    B = s.batch_size
    assert torch.equal(batch["rays"], buf["rays"][ray])
    assert torch.equal(batch["rgbs"], buf["rgbs"][ray])
    assert torch.equal(batch["depths"], buf["depths"][ray])
    assert torch.equal(batch["valid_mask"], buf["valid_mask"][ray].bool())
    if "frame_idx" in buf:
        assert torch.equal(batch["frame_idx"], buf["frame_idx"][ray])
    else:
        assert (batch["frame_idx"] == -1).all()
    for k in ("instance_mask", "instance_mask_weight", "instance_ids", "pass_through_mask"):
        want = buf[k][ray, col].view(B, 1)
        assert torch.equal(batch[k], want.bool() if buf[k].dtype == torch.uint8 else want), k
    assert batch["valid_mask"].dtype == batch["instance_mask"].dtype == batch["pass_through_mask"].dtype == torch.bool
    assert batch["rays"].shape == (B, 8) and batch["rgbs"].shape == (B, 3) and batch["depths"].shape == (B,)
    assert batch["frame_idx"].shape == (B,) and batch["instance_ids"].dtype == torch.int64


@pytest.mark.parametrize("R,I,B,W,frame", [(10_007, 3, 512, 1, True), (10_007, 3, 512, 3, True), (5, 2, 2, 2, False),
                                           (65_537, 1, 2048, 2, True), (1, 4, 1, 1, True)])
def test_kernel_matches_the_restatement(R, I, B, W, frame):
    t = dataset(R, I, frame)
    for seed in (SEED, 7):
        for rank in range(W):
            s = _sampler(t, batch_size=B, seed=seed, rank=rank, world_size=W)
            P = s.batches_per_epoch
            for step in sorted({0, P - 1, P, 2 * P + 1, 5 * P + 3}):
                idx, batch = _draw(s, step)
                ray, col = draw_indices(R, I, B, W, rank, seed, step)
                assert np.array_equal(idx[:, 0].cpu().numpy(), ray), (seed, rank, step)
                assert np.array_equal(idx[:, 1].cpu().numpy(), col), (seed, rank, step)
                _assert_gathered(s, idx, batch)


def test_one_dimensional_instance_buffers_count_as_one_column():
    s = _sampler(dataset(3000, None), batch_size=256, seed=SEED)
    assert s.n_instances == 1
    idx, batch = _draw(s, 4)
    assert (idx[:, 1] == 0).all()
    _assert_gathered(s, idx, batch)


@pytest.mark.parametrize("W", [1, 2])
def test_one_epoch_draws_distinct_rays_across_ranks(W):
    R, B = 1_000_003, 2048
    t = dataset(R, 2)
    samplers = [_sampler(t, batch_size=B, seed=SEED, rank=r, world_size=W) for r in range(W)]
    P = samplers[0].batches_per_epoch
    assert P == R // (B * W)
    idx = torch.empty(W, P, B, 2, dtype=torch.int64, device=DEV)
    for r, s in enumerate(samplers):
        for j in range(P):
            s._args.index_out = idx[r, j].data_ptr()   # next() writes step j's (ray, column) pairs here
            s.next()
    rays = idx[..., 0].flatten()
    assert rays.unique().numel() == P * B * W
    for s in samplers:
        assert s.step == P and s.epoch == 1
    # the next call starts epoch 1: another permutation
    s = samplers[0]
    s._args.index_out = None
    b1 = {k: v.clone() for k, v in s.next().items()}
    i1, _ = _draw(s, P)
    _assert_gathered(s, i1, b1)
    assert not torch.equal(i1[:, 0], idx[0, 0, :, 0])


def test_instance_columns_pass_a_chi_square_test():
    """I = 3, fixed seed: 10^6 column draws spread evenly (deterministic, so not flaky)."""
    R, B, I = 1_000_003, 2048, 3
    s = _sampler(dataset(R, I), batch_size=B, seed=SEED)
    steps = -(-10 ** 6 // B)
    cols = torch.cat([_draw(s, k)[0][:, 1] for k in range(steps)])
    assert cols.numel() >= 10 ** 6
    counts = torch.bincount(cols, minlength=I).cpu().numpy()
    assert counts.size == I
    p = stats.chisquare(counts).pvalue
    assert p > 1e-3, (counts, p)


def test_device_step_draws_what_the_host_step_draws():
    s = _sampler(dataset(10_007, 3), batch_size=512, seed=SEED)
    for k in (0, 3, s.batches_per_epoch, 1000):
        counter = torch.full((1,), k, dtype=torch.int64, device=DEV)
        idx_d, batch_d = _draw(s, 12345, dstep=counter)       # args.step is ignored
        idx_h, batch_h = _draw(s, k)
        assert torch.equal(idx_d, idx_h)
        for key in batch_h:
            assert torch.equal(batch_d[key], batch_h[key]), key
        assert counter.item() == k + 1


def test_set_step_and_next():
    s = _sampler(dataset(10_007, 3), batch_size=512, seed=SEED)
    assert s.step == 0 and s.epoch == 0
    s.set_step(2 * s.batches_per_epoch + 1)
    b = {k: v.clone() for k, v in s.next().items()}
    assert s.step == 2 * s.batches_per_epoch + 2 and s.epoch == 2
    idx, want = _draw(s, 2 * s.batches_per_epoch + 1)
    for k in want:
        assert torch.equal(b[k], want[k]), k


def test_graph_replay_draws_the_eager_batches():
    """A graph captured around next() and replayed k times leaves the batch of step k and advances the counter by k."""
    t = dataset(10_007, 3)
    s = _sampler(t, batch_size=512, seed=SEED)
    e = _sampler(t, batch_size=512, seed=SEED)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        s.next()                                   # warm-up (step 0)
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = s.next()
    assert s.step == 1                             # capturing runs nothing
    e.set_step(1)
    for k in range(1, 2 * s.batches_per_epoch + 3):  # crosses two epoch boundaries
        g.replay()
        want = e.next()
        for key in want:
            assert torch.equal(out[key], want[key]), (k, key)
    assert s.step == e.step == 2 * s.batches_per_epoch + 3


def test_batch_passes_through_total_loss_and_code_library():
    from object_nerf_b200 import CodeLibrary
    from object_nerf_b200.losses import TotalLoss
    R, B = 4096, 1024
    t = dataset(R, 2)
    t["all_instance_ids"] = torch.randint(0, 8, (R, 2))
    s = _sampler(t, batch_size=B, seed=SEED)
    batch = s.next()
    g = torch.Generator(device=DEV).manual_seed(0)
    out = {f"{k}_{typ}": torch.rand(shape, generator=g, device=DEV)
           for typ in ("coarse", "fine")
           for k, shape in (("rgb", (B, 3)), ("depth", (B,)), ("opacity_instance", (B,)), ("rgb_instance", (B, 3)),
                            ("depth_instance", (B,)))}
    loss, _ = TotalLoss(cases.LOSS_CONF)(out, batch)
    want = cases.total_loss(out, batch)
    assert abs(loss.item() - want.item()) <= 1e-5 * abs(want.item())
    lib = CodeLibrary({"N_max_objs": 8, "N_obj_code_length": 64}).to(DEV)
    codes = lib(batch)["embedding_instance"]
    assert torch.equal(codes, lib.embedding_instance.weight.detach()[batch["instance_ids"].view(-1)])


def test_captured_training_loop_trains():
    """sampler.next() + train_step + Adam(capturable=True) captured once and replayed 200 times on a dataset with a
    constant colour and depth target: the replays draw an eager sampler's batches step for step, and the colour term of
    the last 20 replays is below that of the first 20."""
    from object_nerf_b200 import Embedding, training
    from object_nerf_b200 import synthetic as S
    inp = cases.build_grad_case()
    R, B = 16_384, 1024
    t = dataset(R, 2)
    t["all_rays"] = S.random_rays(11, R)
    t["all_rgbs"] = torch.tensor([0.8, 0.4, 0.2]).expand(R, 3).contiguous()
    t["all_depths"] = torch.full((R,), 1.5)
    t["all_valid_masks"] = torch.ones(R, dtype=torch.bool)
    t["all_instance_ids"] = torch.from_numpy(np.random.default_rng(2).choice([4, 6], size=(R, 2)))
    s = _sampler(t, batch_size=B, seed=SEED)
    e = _sampler(t, batch_size=B, seed=SEED)
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
