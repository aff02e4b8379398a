"""configs[2] in the bench scene: one training step of 2048 rays (render_rays train mode -> TotalLoss -> backward -> Adam),
timed with CUDA events.  Reports ms per step and the split forward / backward.

TRAIN_PLAIN=1 times three arms in one process, alternating them step by step: the plain positional-encoding model
(use_voxel_embedding: false) on the fp32 path and on the tensor cores, and the voxel model on the tensor cores as the
reference point.  It also reports the library kernel launches of one step of each arm."""
import os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
import bench
from object_nerf_b200 import Embedding, _lib, render_rays
from object_nerf_b200 import synthetic as S
from tests import cases, helpers

dev = torch.device("cuda", 0)
sc = bench.build_scene(dev)
n = int(os.environ.get("TRAIN_RAYS", 2048))
rng = np.random.default_rng(0)
sel = torch.from_numpy(rng.integers(0, bench.N_RAYS, size=n))
rays = sc["rays"][sel].to(dev)
ids = torch.from_numpy(rng.choice([4, 6], size=n)).to(dev)
batch = {"rgbs": torch.rand(n, 3, device=dev), "depths": torch.rand(n, device=dev) * 2 + 0.3,
         "valid_mask": torch.rand(n, device=dev) < 0.9, "instance_mask": torch.rand(n, device=dev) < 0.5,
         "instance_mask_weight": torch.where(torch.rand(n, device=dev) < 0.5, 1.0, 0.05)}
ptm = torch.rand(n, 1, device=dev) < 0.5
from object_nerf_b200.losses import TotalLoss
loss_fn = TotalLoss({k: v for k, v in cases.LOSS_CONF.items()})
STEPS = int(os.environ.get("TRAIN_STEPS", 10))


class Arm:
    """One trainable setup: models, xyz embedding, code library, Adam, forward precision."""

    def __init__(self, use_voxel, precision):
        self.name = f"{'voxel' if use_voxel else 'plain'} {precision}"
        self.precision = precision
        if use_voxel:
            weights = sc["weights"]
            self.emb = helpers.GridModule(sc["grid"]).to(dev)
        else:   # the bench scene's weight recipe at the plain model's input widths
            weights = {"coarse": S.make_weights(0, False, sigma_gain=8.0, sigma_bias=1.0, rgb_gain=24.0),
                       "fine": S.make_weights(1000, False, sigma_gain=8.0, sigma_bias=1.0, rgb_gain=24.0)}
            self.emb = Embedding(3, 10)
        self.models = {k: helpers.make_model(w, use_voxel, dev).train() for k, w in weights.items()}
        self.lib = helpers.CodeLib(S.make_codes(2)).to(dev)
        params = [p for m in self.models.values() for p in m.parameters()] + list(self.lib.parameters()) + \
            list(self.emb.parameters())
        self.opt = torch.optim.Adam(params, lr=1e-3, fused=True)

    def step(self):
        self.opt.zero_grad(set_to_none=True)
        codes = self.lib.embedding_instance(ids)
        e = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        e[0].record()
        out = render_rays(self.models, {"xyz": self.emb, "dir": Embedding(3, 4)}, rays, N_samples=64, perturb=1.0,
                          noise_std=1.0, N_importance=64, embedding_instance=codes, frustum_bound_th=0.025,
                          pass_through_mask=ptm, is_eval=False, precision=self.precision)
        loss, _ = loss_fn(out, batch)
        e[1].record()
        loss.backward()
        e[2].record()
        self.opt.step()
        e[3].record()
        torch.cuda.synchronize()
        return loss.item(), [e[i].elapsed_time(e[i + 1]) for i in range(3)]


def report(name, ts):
    fw = np.mean([t[1][0] for t in ts]); bw = np.mean([t[1][1] for t in ts]); ad = np.mean([t[1][2] for t in ts])
    tot = [sum(t[1]) for t in ts]
    print(f"train step, {n} rays, {name}: forward+loss {fw:.1f} ms, backward {bw:.1f} ms, adam {ad:.1f} ms, "
          f"total {fw+bw+ad:.1f} ms (median {np.median(tot):.1f}, min {np.min(tot):.1f}) = {n/(fw+bw+ad)*1e3:.0f} rays/s; "
          f"losses {[round(t[0],4) for t in ts]}")


if os.environ.get("TRAIN_PLAIN") == "1":
    print("device:", torch.cuda.get_device_name(dev))
    arms = [Arm(False, "fp32"), Arm(False, "bf16"), Arm(True, "bf16")]
    lib, ctx = _lib.load(), _lib.ctx(dev)
    for arm in arms:
        for _ in range(3):
            arm.step()
        c0 = lib.onerf_ctx_launch_count(ctx)
        arm.step()
        print(f"{arm.name}: {lib.onerf_ctx_launch_count(ctx) - c0} library kernel launches per step")
    ts = {arm.name: [] for arm in arms}
    for _ in range(STEPS):
        for arm in arms:
            ts[arm.name].append(arm.step())
    for arm in arms:
        report(arm.name, ts[arm.name])
else:
    arm = Arm(True, os.environ.get("ONERF_PRECISION", "bf16"))
    for _ in range(3):
        arm.step()
    report(f"forward precision {arm.precision}", [arm.step() for _ in range(STEPS)])
