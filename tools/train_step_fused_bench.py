"""One training step of 2048 rays (configs[2]: 64 + 64 samples, jitter, sigma noise, occlusion mask, pass-through rays)
by four routes, alternated step by step in one process, for the voxel model and the plain positional-encoding model,
all on the tensor cores (bf16):
  existing     render_rays -> TotalLoss -> loss.backward() -> Adam(fused=True)
  fused        training.train_step (onerf_train_step) -> Adam(fused=True, capturable=True)
  graph        the fused step and its Adam step captured once in a CUDA graph through the host-seed entry
               (onerf_train_step), then replayed: every replay draws with the seed the capture froze
  graph-dseed  the same, captured as train_step captures by default (onerf_train_step_dseed, no `_rand` buffers):
               every replay reads and advances the plan's device seed, so it draws fresh numbers
Reports per route the device time per step (CUDA events around the step), the wall time per step (host clock around the
step and a synchronize) and the library kernel launches per step (the graph replays the fused route's launches).
The card's name and power limit are printed with the numbers."""
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch

import bench
from object_nerf_b200 import Embedding, _lib, render_rays, training
from object_nerf_b200 import synthetic as S
from object_nerf_b200.losses import TotalLoss
from tests import cases, helpers

dev = torch.device("cuda", 0)
n = int(os.environ.get("TRAIN_RAYS", 2048))
STEPS = int(os.environ.get("TRAIN_STEPS", 20))
sc = bench.build_scene(dev)
rng = np.random.default_rng(0)
sel = torch.from_numpy(rng.integers(0, bench.N_RAYS, size=n))
batch = {"rays": sc["rays"][sel].to(dev), "instance_ids": torch.from_numpy(rng.choice([4, 6], size=n)).to(dev),
         "rgbs": torch.rand(n, 3, device=dev), "depths": torch.rand(n, device=dev) * 2 + 0.3,
         "valid_mask": torch.rand(n, device=dev) < 0.9, "instance_mask": torch.rand(n, device=dev) < 0.5,
         "instance_mask_weight": torch.where(torch.rand(n, device=dev) < 0.5, 1.0, 0.05)}
ptm = torch.rand(n, 1, device=dev) < 0.5
RENDER = dict(N_samples=64, perturb=1.0, noise_std=1.0, N_importance=64, frustum_bound_th=0.025, pass_through_mask=ptm,
              is_eval=False, precision="bf16")
loss_fn = TotalLoss(cases.LOSS_CONF)


class Arm:
    def __init__(self, use_voxel, route):
        self.name = f"{'voxel' if use_voxel else 'plain'} {route}"
        self.route = route
        if use_voxel:
            weights, self.emb = sc["weights"], helpers.GridModule(sc["grid"]).to(dev)
        else:
            weights = {"coarse": S.make_weights(0, False, sigma_gain=8.0, sigma_bias=1.0, rgb_gain=24.0),
                       "fine": S.make_weights(1000, False, sigma_gain=8.0, sigma_bias=1.0, rgb_gain=24.0)}
            self.emb = Embedding(3, 10)
        self.models = {k: helpers.make_model(w, use_voxel, dev).train() for k, w in weights.items()}
        self.embeddings = {"xyz": self.emb, "dir": Embedding(3, 4)}
        self.lib = helpers.CodeLib(S.make_codes(2)).to(dev)
        params = [p for m in self.models.values() for p in m.parameters()] + list(self.lib.parameters()) + \
            list(self.emb.parameters())
        self.opt = torch.optim.Adam(params, lr=1e-3, fused=True, capturable=route != "existing")
        self.graph = None

    def _eager(self):
        if self.route == "existing":
            self.opt.zero_grad(set_to_none=True)
            codes = self.lib.embedding_instance(batch["instance_ids"])
            out = render_rays(self.models, self.embeddings, batch["rays"], embedding_instance=codes, **RENDER)
            loss, _ = loss_fn(out, batch)
            loss.backward()
        else:
            self.opt.zero_grad(set_to_none=False)
            training.train_step(self.models, self.embeddings, self.lib, batch, cases.LOSS_CONF, **RENDER)
        self.opt.step()

    def prepare(self):
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(3):
                self._eager()
        torch.cuda.current_stream().wait_stream(s)
        if self.route.startswith("graph"):
            self.graph = torch.cuda.CUDAGraph()
            capturing = training._capturing
            if self.route == "graph":       # the host-seed entry: the capture freezes the seed
                training._capturing = lambda dev: False
            try:
                with torch.cuda.graph(self.graph):
                    self._eager()
            finally:
                training._capturing = capturing
        torch.cuda.synchronize()

    def step(self):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter()
        e0.record()
        if self.graph is not None:
            self.graph.replay()
        else:
            self._eager()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1), (time.perf_counter() - t0) * 1e3


def main():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print("device:", torch.cuda.get_device_name(dev), "|", q)
    arms = [Arm(v, r) for v in (True, False) for r in ("existing", "fused", "graph", "graph-dseed")]
    lib, ctx = _lib.load(), _lib.ctx(dev)
    launches = {}
    for arm in arms:
        arm.prepare()
        if not arm.route.startswith("graph"):
            c0 = lib.onerf_ctx_launch_count(ctx)
            arm._eager()
            torch.cuda.synchronize()
            launches[arm.name] = lib.onerf_ctx_launch_count(ctx) - c0
    for arm in arms:
        if arm.route.startswith("graph"):
            launches[arm.name] = launches[arm.name.split()[0] + " fused"]
    ts = {arm.name: [] for arm in arms}
    for _ in range(STEPS):
        for arm in arms:
            ts[arm.name].append(arm.step())
    print(f"train step, {n} rays, 64 + 64 samples, bf16, {STEPS} steps per route, routes alternated step by step")
    for arm in arms:
        dt = np.array([t[0] for t in ts[arm.name]])
        wt = np.array([t[1] for t in ts[arm.name]])
        print(f"  {arm.name:18s} device {np.median(dt):7.2f} ms (min {dt.min():6.2f})  wall {np.median(wt):7.2f} ms "
              f"(min {wt.min():6.2f})  library launches {launches[arm.name]}")


if __name__ == "__main__":
    main()
