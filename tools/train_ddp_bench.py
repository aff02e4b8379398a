"""Data-parallel training three ways, run under torchrun (NCCL, one process per GPU); per rank 2048 rays per step,
64 + 64 samples, bf16, voxel model (bench.build_scene's model), batches from batches.RaySampler(group=) over
tools/train_loop_bench.py's synthetic dataset:
  a  DistributedDataParallel around render_rays + TotalLoss, loss.backward(), Adam(fused=True)
  b  training.train_step(group=) eagerly + Adam(fused=True, capturable=True)
  c  b captured once in a CUDA graph (sampler + step + Adam) and replayed
Per rank and arm: wall-clock steps/s over STEPS steps (host clock around a window that ends in a synchronize) and the
median device time per step (CUDA events around each step).  Also the all-reduce alone (SUM + 1/W scale, 50 calls
captured in one graph and replayed) over the whole gradient bucket and over the prefix train_step reduces.  The card's
name and power limit are printed with the numbers.

    torchrun --nproc-per-node N tools/train_ddp_bench.py"""
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np
import torch
import torch.distributed as dist

import bench
from object_nerf_b200 import Embedding, RaySampler, render_rays, training
from object_nerf_b200.losses import TotalLoss
from tests import cases, helpers
from train_loop_bench import B, RENDER, make_dataset

STEPS = int(os.environ.get("DDP_STEPS", 100))


class System(torch.nn.Module):
    """The reference's ObjectNeRFSystem forward (train.py:147-176): codes, render_rays, TotalLoss."""

    def __init__(self, models, emb, lib):
        super().__init__()
        self.coarse, self.fine, self.emb, self.lib = models["coarse"], models["fine"], emb, lib
        self.loss = TotalLoss(cases.LOSS_CONF)

    def forward(self, batch):
        codes = self.lib.embedding_instance(batch["instance_ids"].view(-1))
        out = render_rays({"coarse": self.coarse, "fine": self.fine}, {"xyz": self.emb, "dir": Embedding(3, 4)},
                          batch["rays"], embedding_instance=codes, pass_through_mask=batch["pass_through_mask"],
                          **RENDER)
        return self.loss(out, batch)[0]


class Arm:
    def __init__(self, sc, arm, data, dev, group):
        self.arm, self.group = arm, group
        self.models = {k: helpers.make_model(w, True, dev).train() for k, w in sc["weights"].items()}
        self.emb = helpers.GridModule(sc["grid"]).to(dev)
        self.embeddings = {"xyz": self.emb, "dir": Embedding(3, 4)}
        self.lib = helpers.CodeLib(sc["code_table"]).to(dev)
        params = [p for m in self.models.values() for p in m.parameters()] + list(self.lib.parameters()) + \
            list(self.emb.parameters())
        self.sampler = RaySampler(data, batch_size=B, device=dev, seed=1, group=group)
        if arm == "a":
            self.ddp = torch.nn.parallel.DistributedDataParallel(
                System(self.models, self.emb, self.lib), device_ids=[dev.index], broadcast_buffers=False,
                bucket_cap_mb=128, gradient_as_bucket_view=True)
        else:
            training.sync_replicas(self.models, self.embeddings, self.lib, group)
        self.opt = torch.optim.Adam(params, lr=1e-3, fused=True, capturable=arm != "a")
        self.graph = None

    def _eager(self):
        batch = self.sampler.next()
        self.opt.zero_grad(set_to_none=False)
        if self.arm == "a":
            self.ddp(batch).backward()
        else:
            training.train_step(self.models, self.embeddings, self.lib, batch, cases.LOSS_CONF,
                                pass_through_mask=batch["pass_through_mask"], group=self.group, **RENDER)
        self.opt.step()

    def prepare(self):
        # the graphed arm warms up on a side stream (as a capture needs); DDP keeps its autograd nodes, so arm a warms
        # up on the stream it is timed on
        s = torch.cuda.Stream() if self.arm == "c" else torch.cuda.current_stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(5):
                self._eager()
        torch.cuda.current_stream().wait_stream(s)
        if self.arm == "c":
            self.graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.graph):
                self._eager()
        torch.cuda.synchronize()

    def run(self, steps):
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
        dist.barrier()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for e0, e1 in ev:
            e0.record()
            if self.graph is not None:
                self.graph.replay()
            else:
                self._eager()
            e1.record()
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
        return steps / wall, float(np.median([e0.elapsed_time(e1) for e0, e1 in ev]))


def allreduce_ms(t, group, calls=50, replays=10):
    """Device time of one SUM all-reduce + 1/W scale of t, from a graph of `calls` of them."""
    world = dist.get_world_size(group)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        dist.all_reduce(t, group=group)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            for _ in range(calls):
                dist.all_reduce(t, op=dist.ReduceOp.SUM, group=group)
                t.mul_(1.0 / world)
    torch.cuda.current_stream().wait_stream(s)
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(replays):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / (calls * replays)


def main():
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", 0)))
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl", device_id=dev)
    group = dist.group.WORLD
    if rank == 0:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True).stdout.strip()
        print("device:", torch.cuda.get_device_name(dev), "|", q)
    sc = bench.build_scene(dev)
    data = make_dataset(sc)
    if rank == 0:
        print(f"world {world}; per rank {B} rays per step, 64 + 64 samples, bf16, voxel model; "
              f"R = {data['all_rays'].shape[0]} rays; {STEPS} timed steps per arm after 5 warm-up steps")
    names = {"a": "DDP(render_rays + TotalLoss) + backward + Adam",
             "b": "train_step(group=) + Adam, eager",
             "c": "sampler + train_step(group=) + Adam, one graph replay"}
    lines = []
    arms = {}
    for a in ("a", "b", "c"):
        arms[a] = Arm(sc, a, data, dev, group)
        arms[a].prepare()
    for a, arm in arms.items():
        sps, dev_ms = arm.run(STEPS)
        lines.append(f"  rank {rank}  {a}  {names[a]:54s} {sps:7.1f} steps/s  device {dev_ms:7.2f} ms/step")
    (plan,) = training._plans[arms["b"].models["coarse"]].values()
    bucket, n_used = plan.bucket, training._synced[arms["b"].models["coarse"]][1]
    n_prefix = bucket.prefix(n_used)
    full, prefix = bucket.flat.clone(), bucket.flat[:n_prefix].clone()
    full_ms, prefix_ms = allreduce_ms(full, group), allreduce_ms(prefix, group)
    lines.append(f"  rank {rank}  all-reduce + scale: whole bucket {bucket.flat.numel()} floats "
                 f"({bucket.flat.numel() * 4 / 1e6:.1f} MB) {full_ms:.3f} ms; prefix {n_prefix} floats "
                 f"({n_prefix * 4 / 1e6:.1f} MB, n_used = {n_used}) {prefix_ms:.3f} ms")
    out = [None] * world
    dist.all_gather_object(out, lines)
    if rank == 0:
        for ls in out:
            print("\n".join(ls))
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
