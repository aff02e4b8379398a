"""The reference's own ObjectNeRFSystem.training_step (train.py:147-180, byte-compiled into oracle/_ref) by two routes,
alternated step by step in one process, for the voxel model and the plain positional-encoding model, bf16:
  reference  training_step over dropin.install() (render_rays -> TotalLoss -> psnr), loss.backward(), Adam(fused=True)
  installed  training.install_training(ObjectNeRFSystem): the one-call step through TrainStepFn, loss.backward(), Adam
  direct     for comparison, no Lightning: training.train_step into .grad (zero_grad(set_to_none=False)), then Adam
2048 rays per step, 64 + 64 samples, jitter and sigma noise on, on tests/dropin_fixture.py's synthetic scene with
default_conf.yml's 800 000-row voxel table.  Under torchrun (NCCL) the reference and installed routes run inside
DistributedDataParallel around a module whose forward is training_step (world 1 measures DDP's own cost):

    python tools/train_lightning_bench.py
    torchrun --nproc-per-node 1 tools/train_lightning_bench.py

Per route: median device time per step (CUDA events around zero_grad, training_step, backward and the Adam step) and
steps/s (host clock around each step and a synchronize).  Also the device time of the installed backward's gradient
copy alone (one multiply per trained tensor, as TrainStepFn.backward).  The card's name and power limit are printed
with the numbers."""
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch

from oracle import ref_loader as R

N = int(os.environ.get("TRAIN_RAYS", 2048))
STEPS = int(os.environ.get("TRAIN_STEPS", 50))


class _Step(torch.nn.Module):
    """DDP wraps a module's forward: this one's is the system's training_step."""

    def __init__(self, system):
        super().__init__()
        self.system = system

    def forward(self, batch):
        return self.system.training_step(batch, 0)


class Arm:
    def __init__(self, use_voxel, route, conf, batch, dev, ddp):
        import object_nerf_b200.dropin as dropin
        from object_nerf_b200 import training
        from tests import dropin_fixture as F
        from tests.test_gpu_install_training import _fill
        self.name, self.route = f"{'voxel' if use_voxel else 'plain'} {route}", route
        conf = dict(conf, model=dict(conf["model"], use_voxel_embedding=use_voxel))
        F.purge_reference_modules()
        R.install(cuda_noop=False)
        dropin.install()
        train, self.system = F.make_system(conf, dev)
        _fill(self.system, use_voxel)
        self.system.train()
        if route == "installed":
            training.install_training(train.ObjectNeRFSystem)
        params = [p for p in self.system.parameters() if p.requires_grad]
        self.system.optimizer = self.opt = torch.optim.Adam(params, lr=1e-3, fused=True)
        self.step_module = _Step(self.system)
        if ddp:
            self.step_module = torch.nn.parallel.DistributedDataParallel(
                self.step_module, device_ids=[dev.index], broadcast_buffers=False)
        self.batch = batch

    def run(self):
        if self.route == "direct":
            from object_nerf_b200 import training
            s, m = self.system, self.system.config.model
            self.opt.zero_grad(set_to_none=False)
            training.train_step(s.models, s.embeddings, s.code_library, self.batch, s.config.loss, N_samples=m.N_samples,
                                use_disp=m.use_disp, perturb=m.perturb, noise_std=m.noise_std,
                                N_importance=m.N_importance, pass_through_mask=self.batch["pass_through_mask"],
                                frustum_bound_th=m.frustum_bound / s.config.dataset_extra.scale_factor)
        else:
            self.opt.zero_grad(set_to_none=True)
            self.step_module(self.batch).backward()
        self.opt.step()

    def step(self):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        e0.record()
        self.run()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1), time.perf_counter() - t0


def copy_ms(arm, reps=20):
    """Device time of TrainStepFn.backward's work alone: every sink gradient times a device scalar, new tensors."""
    from object_nerf_b200 import training
    (plan,) = training._plans[arm.system.models["coarse"]].values()
    one = torch.ones((), device=plan.sink.flat.device)
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = [g * one for g in plan.sink.views]
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
        del out
    return float(np.median(ts)), plan.sink.flat.numel() * 4 / 1e6


def main():
    if not R.available():
        sys.exit("oracle/_ref not built: build() byte-compiles the reference there where a reference checkout exists")
    ddp = "RANK" in os.environ
    dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", 0)))
    torch.cuda.set_device(dev)
    if ddp:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=dev)
    os.environ.setdefault("ONERF_PRECISION", "bf16")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print("device:", torch.cuda.get_device_name(dev), "|", q)
    from tests import dropin_fixture as F
    with tempfile.TemporaryDirectory() as tmp:
        conf, _ = F.write_scene(tmp)
        conf["model"].update(perturb=1, noise_std=1, N_max_voxels=800000)
        batch = {k: v.to(dev) for k, v in F.training_batch(n=N).items()}
        try:
            routes = ("reference", "installed") if ddp else ("reference", "installed", "direct")
            arms = [Arm(v, r, conf, batch, dev, ddp) for v in (True, False) for r in routes]
            for arm in arms:
                for _ in range(5):
                    arm.run()
            torch.cuda.synchronize()
            ts = {arm.name: [] for arm in arms}
            for _ in range(STEPS):
                for arm in arms:
                    ts[arm.name].append(arm.step())
            copies = {arm.name: copy_ms(arm) for arm in arms if arm.name.endswith("installed")}
        finally:
            F.purge_reference_modules()
    print(f"ObjectNeRFSystem.training_step + backward + Adam, {N} rays, 64 + 64 samples, bf16, "
          f"{'DDP world 1 (NCCL)' if ddp else 'no DDP'}, {STEPS} steps per route, routes alternated step by step")
    for arm in arms:
        dt = np.array([t[0] for t in ts[arm.name]])
        wt = np.array([t[1] for t in ts[arm.name]])
        print(f"  {arm.name:16s} device {np.median(dt):7.2f} ms (min {dt.min():6.2f})  "
              f"{len(wt) / wt.sum():6.1f} steps/s")
    for name, (ms, mb) in copies.items():
        print(f"  {name:16s} backward gradient copy alone: {ms:.3f} ms for {mb:.1f} MB")
    if ddp:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
