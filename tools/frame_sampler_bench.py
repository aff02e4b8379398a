"""Training batches from the frame store (RaySampler.from_frames) against the same batches from GenericDataset's
expanded per-ray buffers (RaySampler(frame_set.expand())), on one synthetic scene: FRAMES frames of 640x480 pixels
(default 50, so 15.4 M rays) seen by bench's pinhole camera, jittered per frame, with random colours, depths and labels,
at I = 1 and I = 5 instance columns.  Both samplers draw bit-identical batches (tests/test_gpu_frames.py).

Per I:
  - device bytes each sampler holds (frame store: its tensors; expanded: the uploaded per-ray buffers);
  - device time per next() at B = 2048 and 8192: 100 calls captured in one graph, replayed REPEATS times, the two
    samplers alternated, median and spread over the repeats;
  - steps/s of the captured next() + training.train_step + Adam(capturable) loop at B = 2048 (bench's model, bf16,
    64 + 64 samples): STEPS replays after warm-up, host clock around a window ending in a synchronize, alternated.
The card's name and power limit are printed with the numbers.

    python tools/frame_sampler_bench.py            # FRAMES=50 STEPS=200 REPEATS=3 by default
"""
import json
import math
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch

import bench
from object_nerf_b200 import Embedding, RaySampler, training
from object_nerf_b200.frames import FrameSet
from tests import cases, helpers

dev = torch.device("cuda", 0)
FRAMES = int(os.environ.get("FRAMES", 50))
STEPS = int(os.environ.get("STEPS", 200))
REPEATS = int(os.environ.get("REPEATS", 3))
H, W = 480, 640
RENDER = dict(N_samples=64, perturb=1.0, noise_std=1.0, N_importance=64, frustum_bound_th=0.025, is_eval=False,
              precision="bf16")


def frame_set(I):
    rng = np.random.default_rng(5)
    poses = []
    for _ in range(FRAMES):
        cam = np.array([-1.6, 0.1, 0.15]) + rng.normal(size=3) * 0.05
        fwd = -cam / np.linalg.norm(cam)
        right = np.cross(fwd, [0.0, 0.0, 1.0])
        right /= np.linalg.norm(right)
        up = np.cross(right, fwd)
        poses.append(np.concatenate([np.stack([right, up, -fwd], 1), cam[:, None]], 1))
    ids = [4, 6, 1, 2, 3][:I]
    return FrameSet(np.stack(poses).astype(np.float32), rng.integers(0, 256, (FRAMES, H, W, 3), dtype=np.uint8),
                    rng.uniform(0, 3, (FRAMES, H, W)).astype(np.float32),
                    rng.choice(ids + [0], size=(FRAMES, H, W)).astype(np.uint16),
                    focal=0.5 * W / math.tan(math.radians(30)), near=0.15, far=3.0, scale_factor=1.0,
                    instance_ids=ids, bg_instance_ids=[0], device=dev)


def draw_us(sampler, calls=100):
    """Device microseconds per next(): `calls` calls captured in one graph, timed with events around one replay."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        sampler.next()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(calls):
            sampler.next()
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / calls


class Loop:
    """next() + train_step + Adam(capturable) captured in one graph."""

    def __init__(self, sc, sampler):
        self.sampler = sampler
        self.models = {k: helpers.make_model(w, True, dev).train() for k, w in sc["weights"].items()}
        emb = helpers.GridModule(sc["grid"]).to(dev)
        self.embeddings = {"xyz": emb, "dir": Embedding(3, 4)}
        self.lib = helpers.CodeLib(sc["code_table"]).to(dev)
        params = [p for m in self.models.values() for p in m.parameters()] + list(self.lib.parameters()) + \
            list(emb.parameters())
        self.opt = torch.optim.Adam(params, lr=1e-3, fused=True, capturable=True)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(5):
                self._step()
        torch.cuda.current_stream().wait_stream(s)
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self._step()
        torch.cuda.synchronize()

    def _step(self):
        batch = self.sampler.next()
        self.opt.zero_grad(set_to_none=False)
        training.train_step(self.models, self.embeddings, self.lib, batch, cases.LOSS_CONF,
                            pass_through_mask=batch["pass_through_mask"], **RENDER)
        self.opt.step()

    def steps_per_s(self, steps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(steps):
            self.graph.replay()
        torch.cuda.synchronize()
        return steps / (time.perf_counter() - t0)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def spread(xs):
    return {"median": float(np.median(xs)), "min": float(np.min(xs)), "max": float(np.max(xs))}


def main():
    sc = bench.build_scene()
    print(json.dumps({"card": card(), "frames": FRAMES, "H": H, "W": W, "repeats": REPEATS, "steps": STEPS}),
          flush=True)
    for I in (1, 5):
        fs = frame_set(I)
        res = {"I": I, "rays": fs.n_rays}
        ex = fs.expand()
        for B in (2048, 8192):
            f = RaySampler.from_frames(fs, batch_size=B, seed=1)
            e = RaySampler(ex, batch_size=B, device=dev, seed=1)
            if B == 2048:
                res["bytes_frames"] = fs.nbytes
                res["bytes_expanded"] = sum(t.numel() * t.element_size() for t in e.buffers.values())
            t = {"frames": [], "expanded": []}
            for _ in range(REPEATS):
                t["frames"].append(draw_us(f))
                t["expanded"].append(draw_us(e))
            res[f"draw_us_B{B}"] = {k: spread(v) for k, v in t.items()}
            del f, e
        del ex
        torch.cuda.empty_cache()
        e_fs = frame_set(I)
        loops = {"frames": Loop(sc, RaySampler.from_frames(fs, batch_size=2048, seed=1)),
                 "expanded": Loop(sc, RaySampler(e_fs.expand(), batch_size=2048, device=dev, seed=1))}
        del e_fs
        sps = {"frames": [], "expanded": []}
        for _ in range(REPEATS):
            for k, lp in loops.items():
                sps[k].append(lp.steps_per_s(STEPS))
        res["loop_steps_per_s_B2048"] = {k: spread(v) for k, v in sps.items()}
        print(json.dumps(res), flush=True)
        del loops, fs
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
