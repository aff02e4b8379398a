"""A training loop fed three ways, 2048 rays per step, 64 + 64 samples, bf16, voxel model (bench.build_scene's model):
  A  a host Dataset restating GenericDataset.__getitem__ (datasets/generic_dataset.py:475-490) through
     DataLoader(shuffle=True, batch_size=2048, num_workers=6, pin_memory=True) (train.py:121-129), the batch copied to
     the device, then training.train_step eagerly and Adam(fused=True)
  B  batches.RaySampler.next() + train_step eagerly + Adam(fused=True, capturable=True)
  C  B captured once in a CUDA graph and replayed
The dataset is synthetic: FRAMES frames of bench's 640x480 pinhole rays (default 50, so 15.4 M rays) with random targets,
masks and two instance columns (ids 4 and 6).

Per route: wall-clock steps/s over STEPS steps (host clock around the window, which ends in a synchronize), the median
device time per step (CUDA events around each step), and the host process's CPU time per step from the first to the
last enqueue (time.process_time, without the final synchronize, whose wait spins; for A it excludes the six loader
workers).  Also the sampler kernel's own device time: 100 calls captured in one graph and
replayed, for onerf_draw_batch alone and for onerf_draw_batch_dstep (draw + the one-thread step advance).  The card's
name and power limit and the host CPU count are printed with the numbers."""
import ctypes as C
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch

import bench
from object_nerf_b200 import Embedding, RaySampler, _lib, training
from tests import cases, helpers

dev = torch.device("cuda", 0)
B = 2048
FRAMES = int(os.environ.get("LOOP_FRAMES", 50))
STEPS = int(os.environ.get("LOOP_STEPS", 200))
RENDER = dict(N_samples=64, perturb=1.0, noise_std=1.0, N_importance=64, frustum_bound_th=0.025, is_eval=False,
              precision="bf16")


def make_dataset(sc):
    """GenericDataset's training buffers (generic_dataset.py:216-307) for FRAMES frames, I = 2."""
    R = FRAMES * bench.N_RAYS
    rng = np.random.default_rng(7)
    g = torch.Generator().manual_seed(7)
    return {"all_rays": sc["rays"].repeat(FRAMES, 1), "all_rgbs": torch.rand(R, 3, generator=g),
            "all_depths": torch.rand(R, generator=g) * 2 + 0.3, "all_valid_masks": torch.rand(R, generator=g) < 0.9,
            "all_instance_masks": torch.rand(R, 2, generator=g) < 0.5,
            "all_instance_masks_weight": torch.where(torch.rand(R, 2, generator=g) < 0.5, 1.0, 0.05),
            "all_instance_ids": torch.from_numpy(rng.choice([4, 6], size=(R, 2))),
            "all_pass_through_masks": torch.rand(R, 2, generator=g) < 0.5,
            "all_frame_indices": torch.arange(FRAMES).repeat_interleave(bench.N_RAYS)}


class HostDataset(torch.utils.data.Dataset):
    """GenericDataset.__getitem__ for split == "train"."""

    def __init__(self, t):
        self.t = t
        self.n_instances = t["all_instance_masks"].shape[1]

    def __len__(self):
        return self.t["all_rays"].shape[0]

    def __getitem__(self, idx):
        t = self.t
        c = torch.randint(0, self.n_instances, (1,))
        return {"rays": t["all_rays"][idx], "rgbs": t["all_rgbs"][idx], "depths": t["all_depths"][idx],
                "valid_mask": t["all_valid_masks"][idx], "instance_mask": t["all_instance_masks"][idx, c],
                "instance_mask_weight": t["all_instance_masks_weight"][idx, c],
                "frame_idx": t["all_frame_indices"][idx], "instance_ids": t["all_instance_ids"][idx, c],
                "pass_through_mask": t["all_pass_through_masks"][idx, c]}


class Route:
    def __init__(self, sc, route, data):
        self.route = route
        self.models = {k: helpers.make_model(w, True, dev).train() for k, w in sc["weights"].items()}
        self.emb = helpers.GridModule(sc["grid"]).to(dev)
        self.embeddings = {"xyz": self.emb, "dir": Embedding(3, 4)}
        self.lib = helpers.CodeLib(sc["code_table"]).to(dev)
        params = [p for m in self.models.values() for p in m.parameters()] + list(self.lib.parameters()) + \
            list(self.emb.parameters())
        self.opt = torch.optim.Adam(params, lr=1e-3, fused=True, capturable=route != "A")
        self.graph = None
        if route == "A":
            loader = torch.utils.data.DataLoader(HostDataset(data), shuffle=True, batch_size=B, num_workers=6,
                                                 pin_memory=True)
            self.batches = iter(loader)
        else:
            self.sampler = RaySampler(data, batch_size=B, device=dev, seed=1)

    def _batch(self):
        if self.route == "A":
            return {k: v.to(dev, non_blocking=True) for k, v in next(self.batches).items()}
        return self.sampler.next()

    def _eager(self):
        batch = self._batch()
        self.opt.zero_grad(set_to_none=False)
        training.train_step(self.models, self.embeddings, self.lib, batch, cases.LOSS_CONF,
                            pass_through_mask=batch["pass_through_mask"], **RENDER)
        self.opt.step()

    def prepare(self):
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(5):
                self._eager()
        torch.cuda.current_stream().wait_stream(s)
        if self.route == "C":
            self.graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.graph):
                self._eager()
        torch.cuda.synchronize()

    def run(self, steps):
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
        torch.cuda.synchronize()
        c0, t0 = time.process_time(), time.perf_counter()
        for e0, e1 in ev:
            e0.record()
            if self.graph is not None:
                self.graph.replay()
            else:
                self._eager()
            e1.record()
        cpu = time.process_time() - c0          # up to the last enqueue: the synchronize below spins
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
        dt = np.array([e0.elapsed_time(e1) for e0, e1 in ev])
        return steps / wall, float(np.median(dt)), cpu / steps * 1e3


def sampler_kernel_us(sampler, dstep, calls=100, replays=20):
    """Device time per call of 100 sampler launches captured in one graph (no host work in the timed window)."""
    lib, ctx = _lib.load(), _lib.ctx(dev)
    a = _lib.BatchArgs.from_buffer_copy(sampler._args)
    a.step = 3
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            for _ in range(calls):
                if dstep:
                    _lib.check(lib.onerf_draw_batch_dstep(ctx, C.byref(a), sampler._step.data_ptr(), _lib.stream()))
                else:
                    _lib.check(lib.onerf_draw_batch(ctx, C.byref(a), _lib.stream()))
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(replays):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / (calls * replays)


def main():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print("device:", torch.cuda.get_device_name(dev), "|", q)
    print(f"host CPUs: {os.cpu_count()} (usable by this process: {len(os.sched_getaffinity(0))})")
    sc = bench.build_scene(dev)
    data = make_dataset(sc)
    R = data["all_rays"].shape[0]
    print(f"dataset: {FRAMES} frames of {bench.W}x{bench.H}, R = {R} rays, I = 2; {B} rays per step, 64 + 64 samples, "
          f"bf16, voxel model, {STEPS} timed steps per route after 5 warm-up steps")
    routes = [Route(sc, r, data) for r in ("A", "B", "C")]
    for r in routes:
        r.prepare()
    names = {"A": "host DataLoader (6 workers) + train_step + Adam",
             "B": "RaySampler.next() + train_step + Adam, eager",
             "C": "RaySampler.next() + train_step + Adam, one graph replay"}
    for r in routes:
        sps, dev_ms, cpu_ms = r.run(STEPS)
        print(f"  {r.route}  {names[r.route]:56s} {sps:7.1f} steps/s  device {dev_ms:7.2f} ms/step  "
              f"host CPU {cpu_ms:7.2f} ms/step")
    s = routes[1].sampler
    draw, dstep = sampler_kernel_us(s, False), sampler_kernel_us(s, True)
    print(f"sampler, {B} rays: onerf_draw_batch {draw:.2f} us per call, onerf_draw_batch_dstep {dstep:.2f} us per call "
          f"(graph of 100 calls)")


if __name__ == "__main__":
    main()
