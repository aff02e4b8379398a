"""bench.py — headline metric of BASELINE.json: rays/s rendering 640x480 frames (64 coarse + 64 importance
samples => 128-sample fine pass, scene + object branch, voxel embedding) through the reference call surface
`render_rays()`, plus the fused-MLP tensor-core roofline.

  python bench.py [--gpus N] [--steps K] [--warmup W] [--impl ours|reference] [--precision bf16|fp32] [--no-extras]
                  [--dump-outputs DIR]

One process per GPU (torchrun for N > 1).  Headline (`value`, `e2e`, `roofline`): a step = one full frame (307 200 rays)
per rank, rendered in 65 536-ray chunks; N > 1: every rank renders its own frame and the (rgb, depth) tiles are
all-gathered over NCCL inside the timed region (weak scaling, no other collective).
The same JSON line carries, unless --no-extras:
  "train"   BASELINE configs[2]/[3]: one training step of 2 048 rays per rank (render_rays train mode -> fused TotalLoss ->
            tensor-core backward -> DDP gradient all-reduce over NCCL -> Adam), rays/s and per-kernel times
  "strong"  BASELINE configs[4] sharding: ONE frame tile-sharded over the N ranks, gather inside the timed region
  "edit"    BASELINE configs[4] path: render_rays_multi with ray sets [0, 4, 4], chunk 4096 (edit_scannet_0113.yaml shape)
  "parity"  the GPU render of the cpu_baseline sample against the reference / oracle output of the same rays
  "gpu_torch_baseline"  the unmodified reference (PyTorch) running on the same GPU (fp32 and TF32)
Prints ONE JSON line (rank 0).  See DESIGN.md §5 for the definitions.
--dump-outputs DIR writes what the last timed headline step returned (rank 0's frame: rgb_fine (H*W, 3) and depth_fine
(H*W,), float32) as DIR/<name>.npy.  The scene and rays are generated from fixed seeds, so two builds run with the same
arguments can be compared output for output.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import statistics
import subprocess
import sys
import tempfile
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

H, W = 480, 640
N_RAYS = H * W
N_SAMPLES, N_IMPORTANCE = 64, 64
CHUNK = 65536
TRAIN_RAYS = 2048                  # config/default_conf.yml:40 batch_size
FLOP_PER_SAMPLE = 1776128          # 2 x MAC of the reference's nn.Linear layers, voxel config (SURVEY.md §8d)
FLOP_PER_RAY = (N_SAMPLES + N_SAMPLES + N_IMPORTANCE) * FLOP_PER_SAMPLE
WORKLOAD = "configs[1]: 640x480 frame, 64 coarse + 64 importance (128-sample fine pass), scene+object two-branch, voxel embedding, eval"
LOSS_CONF = dict(color_loss_weight=1.0, depth_loss_weight=0.1, opacity_loss_weight=100.0,
                 instance_color_loss_weight=1.0, instance_depth_loss_weight=0.1)   # default_conf.yml:61-66 + scannet override


def load_peaks():
    path = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(path):
        with open(path) as f:
            return json.load(f), "measured"
    # NVIDIA H100 SXM data sheet (700 W card): 3.35 TB/s HBM3, 989 TFLOP/s dense BF16; a data-sheet figure, not a measurement
    return {"hbm_gbs": 3350.0, "bf16_tflops": 989.0, "bf16_tflops_sustained": 989.0}, "datasheet"


class ClockSampler:
    """SM clock and throttle reasons of ONE GPU every 100 ms while the timed region runs.  NVML in-process (the library
    nvidia-smi prints from): eight `nvidia-smi -lms` children starting inside an 8-rank timed region each enumerate every
    GPU of the box and stalled the launching threads for tens of milliseconds.  Falls back to an nvidia-smi child."""
    FIELDS = ("clocks.sm,clocks.max.sm,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
              "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")
    NAMES = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]

    def __init__(self, index):
        self.index, self.proc, self.tmp, self.rows, self.thread, self.h = index, None, None, [], None, None
        self.stop = threading.Event()
        try:
            import pynvml
            pynvml.nvmlInit()
            visible = os.environ.get("CUDA_VISIBLE_DEVICES")
            phys = int(visible.split(",")[index]) if visible and visible.split(",")[index].strip().isdigit() else index
            self.h = pynvml.nvmlDeviceGetHandleByIndex(phys)
            self.nv = pynvml
            self.max_mhz = float(pynvml.nvmlDeviceGetMaxClockInfo(self.h, pynvml.NVML_CLOCK_SM))
        except Exception:
            self.h = None

    def _poll(self):
        nv = self.nv
        masks = [nv.nvmlClocksThrottleReasonHwSlowdown, nv.nvmlClocksThrottleReasonHwThermalSlowdown,
                 nv.nvmlClocksThrottleReasonSwThermalSlowdown, nv.nvmlClocksThrottleReasonSwPowerCap]
        while True:
            try:
                mhz = float(nv.nvmlDeviceGetClockInfo(self.h, nv.NVML_CLOCK_SM))
                r = nv.nvmlDeviceGetCurrentClocksThrottleReasons(self.h)
                self.rows.append((mhz, [bool(r & m) for m in masks]))
            except Exception:
                pass
            if self.stop.wait(0.1):
                return

    def __enter__(self):
        if self.h is not None:
            self.thread = threading.Thread(target=self._poll, daemon=True)
            self.thread.start()
            return self
        try:
            self.tmp = tempfile.NamedTemporaryFile("w+", suffix=".csv", delete=False)
            self.proc = subprocess.Popen(["nvidia-smi", "-i", str(self.index), f"--query-gpu={self.FIELDS}",
                                          "--format=csv,noheader,nounits", "-lms", "100"], stdout=self.tmp,
                                         stderr=subprocess.DEVNULL)
        except Exception:
            self.proc = None
        return self

    def __exit__(self, *exc):
        if self.thread is not None:
            self.stop.set()
            self.thread.join(timeout=2)
        if self.proc is not None:
            self.proc.terminate()
            try:
                self.proc.wait(timeout=5)
            except Exception:
                self.proc.kill()

    def summary(self):
        out = {"sm_mhz": None, "sm_max_mhz": None, "reasons": []}
        if self.thread is not None:
            if self.rows:
                out["sm_mhz"] = statistics.median(r[0] for r in self.rows)
                out["sm_max_mhz"] = self.max_mhz
                out["reasons"] = [n for i, n in enumerate(self.NAMES) if any(r[1][i] for r in self.rows)]
                out["samples"] = len(self.rows)
                out["source"] = "nvml"
            return out
        if self.tmp is None:
            return out
        try:
            self.tmp.flush()
            rows = [r.strip().split(",") for r in open(self.tmp.name) if r.strip()]
            os.unlink(self.tmp.name)
            sm = [float(r[0]) for r in rows if len(r) >= 6]
            if sm:
                out["sm_mhz"] = statistics.median(sm)
                out["sm_max_mhz"] = float(rows[0][1])
                for i, n in enumerate(self.NAMES):
                    if any(r[2 + i].strip().lower().startswith("active") for r in rows if len(r) >= 6):
                        out["reasons"].append(n)
                out["samples"] = len(sm)
                out["source"] = "nvidia-smi"
        except Exception:
            pass
        return out


# ------------------------------------------------------------------------------------------------
# synthetic scene (no datasets / checkpoints offline: SURVEY.md §8d)
# ------------------------------------------------------------------------------------------------
def build_scene(device=None):
    from object_nerf_b200 import synthetic as S
    # density heads sharpened and colour heads scaled so that the render has structure (opacity and colours spread over
    # their range); default nn.Linear init renders a flat grey on which every renderer agrees trivially
    wc = S.make_weights(0, True, sigma_gain=8.0, sigma_bias=1.0, rgb_gain=24.0)
    wf = S.make_weights(1000, True, sigma_gain=8.0, sigma_bias=1.0, rgb_gain=24.0)
    grid = S.make_grid(seed=5, shape=(42, 42, 22), occupancy=0.6, voxel_size=0.05, n_rows=800000)
    rays = S.pinhole_rays(H, W)                      # (307200, 8), pinhole 640x480, unit directions
    code_table = S.make_codes(2)
    ids = torch.from_numpy(np.random.default_rng(3).choice([4, 6], size=N_RAYS))
    return {"weights": {"coarse": wc, "fine": wf}, "grid": grid, "rays": rays, "code_table": code_table, "ids": ids,
            "codes": code_table[ids]}


def train_batches(n_batches, rank, n=TRAIN_RAYS):
    """Per-rank training batches in the shape ObjectNeRFSystem.training_step consumes (train.py:147-180,
    datasets/generic_dataset.py): rays, instance ids in {4, 6} (scannet_base_0113_multi.yml:36), targets and masks."""
    rng = np.random.default_rng(1000 + rank)
    sc_rays = build_scene.cache["rays"]
    out = []
    f = lambda a: torch.from_numpy(np.ascontiguousarray(a.astype(np.float32)))
    for _ in range(n_batches):
        sel = torch.from_numpy(rng.integers(0, N_RAYS, size=n))
        out.append({
            "rays": sc_rays[sel].contiguous(),
            "instance_ids": torch.from_numpy(rng.choice([4, 6], size=n)).view(n, 1),
            "rgbs": f(rng.random((n, 3))), "depths": f(rng.uniform(0.3, 2.5, size=n)),
            "valid_mask": torch.from_numpy(rng.random(n) < 0.9),
            "instance_mask": torch.from_numpy(rng.random(n) < 0.5),
            "instance_mask_weight": f(np.where(rng.random(n) < 0.5, 1.0, 0.05)),
            "pass_through_mask": torch.from_numpy(rng.random((n, 1)) < 0.5),
        })
    return out


# ------------------------------------------------------------------------------------------------
# the reference side: oracle/_ref (the unmodified reference, byte-compiled by oracle/build_ref.py) when present,
# else the oracle port (oracle/onerf_oracle.py, pinned bit-exactly to the reference)
# ------------------------------------------------------------------------------------------------
def reference_renderer(sc, device="cpu"):
    """-> (kind, fn(rays, codes) -> result dict) rendering configs[1] rays with the reference's own render_rays."""
    from oracle import ref_loader as R
    on_cpu = torch.device(device).type == "cpu"
    if R.available():
        R.install(cuda_noop=on_cpu)
        from models.rendering import render_rays as ref_render_rays
        stdout = sys.stdout
        sys.stdout = open(os.devnull, "w")       # the voxel helper prints while it builds its throw-away grid
        try:
            models, emb = R.ref_render_setup(sc["weights"], sc["grid"], device)
        finally:
            sys.stdout.close()
            sys.stdout = stdout

        def fn(rays, codes):
            R.cuda_noop(on_cpu)       # the reference calls .cuda() inside forward: keep CPU runs on the CPU
            try:
                with torch.no_grad():
                    return ref_render_rays(models, emb, rays, N_samples=N_SAMPLES, use_disp=False, perturb=0, noise_std=0,
                                           N_importance=N_IMPORTANCE, chunk=32768, white_back=False,
                                           embedding_instance=codes, is_eval=True)
            finally:
                R.cuda_noop(not torch.cuda.is_available())
        return "reference", fn
    from oracle import onerf_oracle as O
    g = sc["grid"]
    grid = O.VoxelGrid(g["offset"], g["voxel_size"], g["shape"].tolist(), g["idx_map"], g["table"])

    def fn(rays, codes):
        with torch.no_grad():
            return O.render_rays(sc["weights"], grid, rays, codes, n_samples=N_SAMPLES, n_importance=N_IMPORTANCE, is_eval=True)
    return "port", fn


def pick_cpu_threads(fn):
    """torch's CPU matmuls on these small (32768 x 256) chunks can get slower when oversubscribed, so "all the host
    threads it can use" is found by timing a small probe at a few thread counts and keeping the fastest."""
    cores = os.cpu_count() or 1
    best, best_t = cores, None
    for t in sorted({cores, max(1, cores // 2), max(1, cores // 4), 32, 16}, reverse=True):
        if t > cores:
            continue
        torch.set_num_threads(t)
        fn()
        t0 = time.perf_counter()
        fn()
        dt = time.perf_counter() - t0
        if best_t is None or dt < best_t:
            best, best_t = t, dt
    torch.set_num_threads(best)
    return best


def run_reference(args, rank, world):
    """The reference's own CPU implementation of the path on the host cores, a bounded ray sample per step."""
    if rank != 0:
        return
    cores = os.cpu_count() or 1
    sc = build_scene()
    kind, render = reference_renderer(sc)
    n = 2048
    sel = torch.linspace(0, N_RAYS - 1, n).long()
    rays, codes = sc["rays"][sel], sc["codes"][sel]
    threads = pick_cpu_threads(lambda: render(rays[:256], codes[:256]))
    for _ in range(args.warmup):
        render(rays, codes)
    t0 = time.perf_counter()
    for _ in range(args.steps):
        render(rays, codes)
    dt = time.perf_counter() - t0
    val = n * args.steps / dt
    what = ("the unmodified reference (oracle/_ref, models/rendering.py::render_rays, torch CPU fp32)" if kind == "reference"
            else "oracle port (torch CPU fp32)")
    sample = (f"{n} rays of the frame (every {N_RAYS // n}th) per step, {what}, {threads} torch "
              f"threads (fastest of a probe; host has {cores} logical cores)")
    print(json.dumps({
        "impl": "reference", "metric": "rays/s", "value": val, "unit": "rays/s", "n_gpus": args.gpus,
        "steps": args.steps, "warmup": args.warmup, "ms_per_step": 1e3 * dt / args.steps, "higher_is_better": True,
        "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": {"workload": WORKLOAD, "rays_per_step": n},
        "cpu_baseline": {"value": val, "unit": "rays/s", "cores": threads, "kind": kind, "sample": sample},
        "e2e": {"value": val, "unit": "rays/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
    }))


def cpu_baseline_sample(sc):
    """-> (cpu_baseline dict, sample ray indices, reference output dict of the sample)."""
    cores = os.cpu_count() or 1
    kind, render = reference_renderer(sc)
    n = 4096
    sel = torch.linspace(0, N_RAYS - 1, n).long()
    rays, codes = sc["rays"][sel], sc["codes"][sel]
    threads = pick_cpu_threads(lambda: render(rays[:256], codes[:256]))
    t0 = time.perf_counter()
    reps = 0
    out = None
    while reps < 2 or (time.perf_counter() - t0 < 10.0 and reps < 8):
        out = render(rays, codes)
        reps += 1
    dt = time.perf_counter() - t0
    what = "the unmodified reference (oracle/_ref)" if kind == "reference" else "oracle port"
    return ({"value": n * reps / dt, "unit": "rays/s", "cores": threads, "kind": kind,
             "sample": f"{reps} x {n} rays of the frame, {what} (torch CPU fp32), {threads} torch threads "
                       f"(fastest of a probe over thread counts; host has {cores} logical cores)"}, sel, out)


def psnr(a, b):
    mse = torch.mean((a.double() - b.double()) ** 2).item()
    return float("inf") if mse == 0 else -10.0 * math.log10(mse)


def gpu_torch_baseline(sc, dev):
    """The reference as its users run it: unmodified PyTorch code on the same GPU (cuBLAS SGEMM, then TF32)."""
    try:
        kind, render = reference_renderer(sc, dev)
        if kind != "reference":
            return {"unavailable": "oracle/_ref not built"}
        res = {"kind": "unmodified reference (oracle/_ref) on the same GPU, torch " + torch.__version__}
        for n in (2048, 32768):
            sel = torch.linspace(0, N_RAYS - 1, n).long()
            rays, codes = sc["rays"][sel].to(dev), sc["codes"][sel].to(dev)
            for tf32 in (False, True):
                torch.backends.cuda.matmul.allow_tf32 = tf32
                torch.backends.cudnn.allow_tf32 = tf32
                for _ in range(2):
                    render(rays, codes)
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                reps = 5
                e0.record()
                for _ in range(reps):
                    render(rays, codes)
                e1.record()
                torch.cuda.synchronize()
                res[f"rays_per_s_{n}_{'tf32' if tf32 else 'fp32'}"] = n * reps / (e0.elapsed_time(e1) * 1e-3)
        # ---- the reference's training step (train.py:147-180 with its own models / loss / autograd) on the same GPU ----
        from oracle import ref_loader as R
        from models.code_library import CodeLibrary
        from models.losses import TotalLoss
        from models.rendering import render_rays as ref_render_rays
        models, emb = R.ref_render_setup(sc["weights"], sc["grid"], dev)
        for m in models.values():
            m.train()
        lib = CodeLibrary(R.default_model_config()).to(dev)
        loss_fn = TotalLoss(R.AttrDict(LOSS_CONF))
        params = [p for m in models.values() for p in m.parameters()] + list(lib.parameters()) + list(emb["xyz"].parameters())
        opt = torch.optim.Adam(params, lr=1e-3, eps=1e-8)
        batch = {k: v.to(dev) for k, v in train_batches(1, 0)[0].items()}

        def ref_step():
            opt.zero_grad(set_to_none=True)
            codes = lib(batch)["embedding_instance"]
            out = ref_render_rays(models, emb, batch["rays"], N_samples=N_SAMPLES, use_disp=False, perturb=1.0, noise_std=1.0,
                                  N_importance=N_IMPORTANCE, chunk=32768, white_back=False, embedding_instance=codes,
                                  frustum_bound_th=0.025, pass_through_mask=batch["pass_through_mask"], is_eval=False)
            loss, _ = loss_fn(out, batch)
            loss.backward()
            opt.step()

        for tf32 in (False, True):
            torch.backends.cuda.matmul.allow_tf32 = tf32
            torch.backends.cudnn.allow_tf32 = tf32
            res[f"train_rays_per_s_{TRAIN_RAYS}_{'tf32' if tf32 else 'fp32'}"] = TRAIN_RAYS / (event_ms(ref_step, reps=5) * 1e-3)
        torch.backends.cuda.matmul.allow_tf32 = False
        torch.backends.cudnn.allow_tf32 = False
        return res
    except Exception as ex:  # a baseline must never take the product line down
        return {"unavailable": f"{type(ex).__name__}: {ex}"[:200]}


# ------------------------------------------------------------------------------------------------
# our side
# ------------------------------------------------------------------------------------------------
class Timer:
    def __init__(self, dev, world):
        self.dev, self.world = dev, world

    def barrier(self):
        if self.world > 1:
            import torch.distributed as dist
            dist.barrier()
        torch.cuda.synchronize()

    def timed(self, fn, steps):
        """ms for `steps` calls: barrier + synchronize on both sides, CUDA events, max over ranks."""
        import torch.distributed as dist
        self.barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            fn()
        e1.record()
        self.barrier()
        ms = torch.tensor([e0.elapsed_time(e1)], device=self.dev)
        if self.world > 1:
            dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        return ms.item()


def event_ms(fn, reps=5):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def run_train(args, rank, world, dev, sc, timer, peaks):
    """configs[2] / configs[3]: 2 048 rays per rank per step, ray-sharded data parallel, NCCL gradient all-reduce (DDP)."""
    import ctypes as C
    import torch.distributed as dist
    from torch import nn
    from object_nerf_b200 import Embedding, _lib, render_rays, synthetic as S
    from object_nerf_b200.losses import TotalLoss

    class System(nn.Module):
        """What train.ObjectNeRFSystem holds and does in training_step (train.py:36-105, 147-180)."""

        def __init__(self):
            super().__init__()
            self.nerf_coarse = S.make_model(sc["weights"]["coarse"], True, dev).train()
            self.nerf_fine = S.make_model(sc["weights"]["fine"], True, dev).train()
            self.embedding_xyz = S.GridModule(sc["grid"]).to(dev)
            self.code_library = S.make_code_library(sc["code_table"]).to(dev)
            self.loss = TotalLoss(LOSS_CONF)
            self.embedding_dir = Embedding(3, 4)

        def forward(self, b):
            codes = self.code_library({"instance_ids": b["instance_ids"]})["embedding_instance"]
            out = render_rays({"coarse": self.nerf_coarse, "fine": self.nerf_fine},
                              {"xyz": self.embedding_xyz, "dir": self.embedding_dir}, b["rays"], N_samples=N_SAMPLES,
                              use_disp=False, perturb=1.0, noise_std=1.0, N_importance=N_IMPORTANCE, chunk=32768,
                              white_back=False, embedding_instance=codes, frustum_bound_th=0.025,
                              pass_through_mask=b["pass_through_mask"], is_eval=False, precision=args.precision)
            return self.loss(out, b)[0]

    torch.manual_seed(0)
    system = System()
    model = system
    if world > 1:
        model = nn.parallel.DistributedDataParallel(system, device_ids=[dev.index], gradient_as_bucket_view=True,
                                                    bucket_cap_mb=128, broadcast_buffers=False)
    params = [p for p in system.parameters() if p.requires_grad]
    n_grad = sum(p.numel() for p in params)
    opt = torch.optim.Adam(params, lr=1e-3, eps=1e-8, fused=True)
    host = [{k: v.pin_memory() for k, v in b.items()} for b in train_batches(4, rank)]
    resident = [{k: v.to(dev) for k, v in b.items()} for b in host]
    h2d = sum(v.numel() * v.element_size() for v in host[0].values())
    it = {"i": 0}
    loss_host = torch.empty(1, dtype=torch.float32).pin_memory()

    def step(batch):
        opt.zero_grad(set_to_none=True)
        loss = model(batch)
        loss.backward()           # DDP: gradient all-reduce (mean) over NCCL, overlapped with the tail of the backward
        opt.step()
        return loss

    def step_device():
        it["i"] += 1
        return step(resident[it["i"] % len(resident)])

    def step_e2e():
        it["i"] += 1
        b = {k: v.to(dev, non_blocking=True) for k, v in host[it["i"] % len(host)].items()}
        loss = step(b)
        loss_host.copy_(loss.detach().reshape(1), non_blocking=True)
        torch.cuda.current_stream().synchronize()

    steps = max(args.steps * 4, 20)
    for _ in range(20):      # DDP rebuilds its buckets after the first step and NCCL connects channels lazily: at 8 ranks
        step_device()        # the first dozen steps carry one-off stalls of hundreds of milliseconds
    l0 = _lib.launch_count(dev)
    ms = timer.timed(step_device, steps)
    launches = (_lib.launch_count(dev) - l0) / steps
    step_e2e()
    ms_e2e = timer.timed(step_e2e, steps)
    res = {
        "workload": "configs[2]/[3]: ScanNet-0113-shaped train step: 2048 rays per rank (64 coarse + 128 fine samples, "
                    "two-branch, voxel), perturb=1, noise_std=1, frustum_bound_th=0.025, fused TotalLoss, tensor-core "
                    "backward, Adam (fused), DDP all-reduce inside the timed region",
        "metric": "train rays/s", "value": TRAIN_RAYS * world * steps / (ms * 1e-3), "unit": "rays/s", "ms_per_step": ms / steps,
        "steps": steps, "rays_per_step_per_gpu": TRAIN_RAYS, "dtype": args.precision, "scaling": "weak",
        "e2e": {"value": TRAIN_RAYS * world * steps / (ms_e2e * 1e-3), "unit": "rays/s", "h2d_bytes_per_step": h2d,
                "d2h_bytes_per_step": 4},
        "gpu_launches_per_step": launches, "grad_floats_allreduced": n_grad if world > 1 else 0,
    }
    if world > 1:     # the collective alone: one all-reduce of the full gradient size
        buf = torch.zeros(n_grad, device=dev)
        res["allreduce_ms_alone"] = event_ms(lambda: dist.all_reduce(buf))
        res["allreduce_bytes"] = n_grad * 4
    if rank == 0 and args.precision == "bf16":
        # per-kernel times of the fine pass (262 144 samples), stage entry points on a field training workspace
        try:
            res["kernels"] = train_kernel_times(dev, sc, system, peaks)
        except Exception as ex:
            res["kernels"] = {"error": f"{type(ex).__name__}: {ex}"[:200]}
    return res


def train_kernel_times(dev, sc, system, peaks):
    """CUDA-event times of the tensor-core training kernels on one fine pass of 2 048 rays x 128 samples."""
    import ctypes as C
    from object_nerf_b200 import _lib, engine
    lib = _lib.load()
    ctx = _lib.ctx(dev)
    S = N_SAMPLES + N_IMPORTANCE
    n, B = TRAIN_RAYS, TRAIN_RAYS * S
    rays = train_batches(1, 0)[0]["rays"].to(dev)
    z = engine.sample_coarse(rays, S)
    packed = engine.packed_for(system.nerf_fine, True, fresh=True)
    grid = engine.GridBuffers.from_module(system.embedding_xyz)
    codes = torch.randn(n, 64, device=dev)
    ws = torch.empty(lib.onerf_field_train_bytes(1, B) + 1024, dtype=torch.uint8, device=dev)
    ws = ws[(-ws.data_ptr()) % 1024:]
    a = _lib.FieldArgs()
    scene, obj, rc = (torch.empty(n, S, 4, device=dev), torch.empty(n, S, 4, device=dev), torch.empty(n, 448, device=dev))
    a.rays, a.z, a.z_stride, a.codes = rays.data_ptr(), z.data_ptr(), S, codes.data_ptr()
    a.n_rays, a.n_samples = n, S
    a.grid, a.packed = C.pointer(grid.c), packed.data_ptr()
    a.want_scene, a.want_object, a.precision = 1, 1, _lib.PREC_BF16
    a.scene_out, a.obj_out, a.out_stride, a.ray_const = scene.data_ptr(), obj.data_ptr(), S, rc.data_ptr()
    st = _lib.stream
    t = {}
    a.train_ws = None
    t["field_fwd_inference"] = event_ms(lambda: _lib.check(lib.onerf_field_fwd(ctx, C.byref(a), st())))
    a.train_ws = ws.data_ptr()
    t["field_fwd_training_dump"] = event_ms(lambda: _lib.check(lib.onerf_field_fwd(ctx, C.byref(a), st())))
    dA_s, dA_o = torch.randn(B, 4, device=dev) * 1e-3, torch.randn(B, 4, device=dev) * 1e-3
    grad = torch.zeros(lib.onerf_grad_buffer_floats(1), device=dev)
    table_grad = torch.zeros_like(system.embedding_xyz.embedding_space_ftr.weight)
    rs = torch.empty(n, 448, device=dev)
    t["bwd_chain"] = event_ms(lambda: _lib.check(lib.onerf_bwd_chain(ctx, 1, 1, packed.data_ptr(), ws.data_ptr(), B, dA_s.data_ptr(), dA_o.data_ptr(), st())))
    t["bwd_wgrad"] = event_ms(lambda: _lib.check(lib.onerf_bwd_wgrad(ctx, 1, 1, ws.data_ptr(), B, grad.data_ptr(), st())))
    t["bwd_colsums"] = event_ms(lambda: _lib.check(lib.onerf_bwd_colsums(ctx, 1, 1, ws.data_ptr(), B, dA_s.data_ptr(), dA_o.data_ptr(), grad.data_ptr(), st())))
    t["bwd_raysums"] = event_ms(lambda: _lib.check(lib.onerf_bwd_raysums(ctx, 1, 1, ws.data_ptr(), n, S, rs.data_ptr(), st())))
    t["bwd_dx_encode"] = event_ms(lambda: _lib.check(lib.onerf_bwd_dx(ctx, 1, packed.data_ptr(), ws.data_ptr(), rays.data_ptr(), z.data_ptr(), n, S, C.byref(grid.c), table_grad.data_ptr(), st())))
    # algorithmic work of the fine pass: chain = hidden blocks of every layer, wgrad = every GEMM layer, dx = X blocks
    mac_chain = 128 * 256 + 8 * 256 * 256 + 64 * 128 + 4 * 128 * 128
    mac_wgrad = (699904 - 256 - 384 - 27 * 128) + (188160 - 128 - 192 - 27 * 64 - 2 * 64 * 128)
    mac_dx = 2 * 271 * 256 + 2 * (271 + 104) * 128
    out = {"ms": t, "samples": B,
           "tflops": {"bwd_chain": 2 * mac_chain * B / (t["bwd_chain"] * 1e-3) / 1e12,
                      "bwd_wgrad": 2 * mac_wgrad * B / (t["bwd_wgrad"] * 1e-3) / 1e12,
                      "bwd_dx_encode": 2 * mac_dx * B / (t["bwd_dx_encode"] * 1e-3) / 1e12,
                      "field_fwd_training_dump": FLOP_PER_SAMPLE * B / (t["field_fwd_training_dump"] * 1e-3) / 1e12}}
    # the weight-gradient GEMM streams every operand tile once per column block: HBM-bound (layout in DESIGN.md §4.5)
    wg_bytes = 1088 * 1024 * 2 * (B // 128)
    out["wgrad_hbm"] = {"bytes": wg_bytes, "gbs": wg_bytes / (t["bwd_wgrad"] * 1e-3) / 1e9, "peak_gbs": peaks["hbm_gbs"],
                        "frac": wg_bytes / (t["bwd_wgrad"] * 1e-3) / 1e9 / peaks["hbm_gbs"]}
    return out


def run_edit(args, dev, sc, models, embeddings):
    """configs[4] path on one GPU: render_rays_multi, ray sets [scene, object 4, object 4 (duplicate, moved)], chunk 4096,
    two removed-object boxes on the scene set (test/config/edit_scannet_0113.yaml:4-12, demo_editable_render.py:33-42)."""
    from object_nerf_b200 import synthetic as S
    from object_nerf_b200.multi_rendering import render_rays_multi

    class Box:          # the attributes of utils/bbox_utils.py::BBoxRayHelper that the removed-object mask reads
        def __init__(self, b):
            self.scale_factor = 2.0
            self.pose_avg = np.eye(4)
            self.axis_align_mat = np.eye(4)
            self.axis_align_mat[:3, 3] = [0.05 * b, -0.1, 0.0]
            lo = np.array([-0.5, -0.4, -0.3]) + 0.1 * b
            self.bbox_bounds = np.array([lo, lo + 0.6])

    lib = S.make_code_library(sc["code_table"]).to(dev)
    rays0 = sc["rays"].to(dev)
    rng = np.random.default_rng(7)
    sets = [rays0]
    for k in range(2):       # object ray sets: per-ray near / far from a box hit, misses get near = far = 0
        r = rays0.clone()
        near = torch.from_numpy(rng.uniform(0.4, 1.2, size=N_RAYS).astype(np.float32)).to(dev)
        far = near + torch.from_numpy(rng.uniform(0.2, 0.9, size=N_RAYS).astype(np.float32)).to(dev)
        miss = torch.from_numpy(rng.random(N_RAYS) < 0.3).to(dev)
        near[miss] = 0
        far[miss] = 0
        r[:, 6], r[:, 7] = near, far
        sets.append(r)
    boxes = {"4": Box(0), "6": Box(1)}
    chunk = 4096

    n_frame = min(N_RAYS, int(os.environ.get("ONERF_EDIT_CHUNKS", "0")) * chunk or N_RAYS)   # (profiling runs: first chunks only)

    def frame():
        with torch.no_grad():
            for i in range(0, n_frame, chunk):
                render_rays_multi(models, embeddings, lib, [s[i:i + chunk] for s in sets], [0, 4, 4], N_samples=N_SAMPLES,
                                  N_importance=N_IMPORTANCE, chunk=chunk, white_back=False, background_skip_bbox=boxes,
                                  precision=args.precision)

    ms = event_ms(frame, reps=2)
    return {"workload": "configs[4] path: render_rays_multi, 640x480, 3 ray sets (ids [0,4,4]), 64 + 64 samples per set, "
                        "chunk 4096, 2 removed-object boxes, single GPU", "ms_per_frame": ms,
            "rays_per_s": N_RAYS / (ms * 1e-3), "ray_set_evaluations_per_s": 3 * N_RAYS / (ms * 1e-3),
            "tflops_algorithmic": N_RAYS * 2 * 192 * (699904 + 2 * 188160) / (ms * 1e-3) / 1e12}


def run_ours(args, rank, world, local_rank):
    import torch.distributed as dist
    from object_nerf_b200 import Embedding, _lib, engine, parallel, render_rays, synthetic as S

    dev = torch.device("cuda", local_rank)
    torch.cuda.set_device(dev)
    sc = build_scene()
    build_scene.cache = sc
    timer = Timer(dev, world)
    peaks, peaks_kind = load_peaks()
    models = {k: S.make_model(w, True, dev) for k, w in sc["weights"].items()}
    emb = S.GridModule(sc["grid"]).to(dev)
    embeddings = {"xyz": emb, "dir": Embedding(3, 4)}
    code_lib = S.make_code_library(sc["code_table"]).to(dev)
    rays_dev, ids_dev = sc["rays"].to(dev), sc["ids"].to(dev)
    with torch.no_grad():
        codes_dev = code_lib.lookup(ids_dev)
    rays_host, ids_host = sc["rays"].pin_memory(), sc["ids"].pin_memory()
    out_host = torch.empty(N_RAYS, 4, dtype=torch.float32).pin_memory()

    def render(rays, codes, precision=None, keys=("rgb_fine", "depth_fine")):
        n = rays.shape[0]
        rgbd = torch.empty(n, 4, device=dev)
        with torch.no_grad():
            for i in range(0, n, CHUNK):
                r = render_rays(models, embeddings, rays[i:i + CHUNK], N_samples=N_SAMPLES, use_disp=False, perturb=0,
                                noise_std=0, N_importance=N_IMPORTANCE, chunk=32768, white_back=False,
                                embedding_instance=codes[i:i + CHUNK], is_eval=True, precision=precision or args.precision)
                rgbd[i:i + CHUNK, :3] = r[keys[0]]
                rgbd[i:i + CHUNK, 3] = r[keys[1]]
        return rgbd

    last = {}

    def step_device():          # weak scaling: every rank renders its own frame, no collective on the data path
        last["rgbd"] = render(rays_dev, codes_dev)
        return last["rgbd"]

    def step_e2e():
        r = rays_host.to(dev, non_blocking=True)
        ids = ids_host.to(dev, non_blocking=True)
        with torch.no_grad():
            c = code_lib.lookup(ids)             # the code-library gather runs on the device: 8 B of ids per ray cross PCIe
        rgbd = render(r, c)
        out_host.copy_(rgbd, non_blocking=True)
        torch.cuda.current_stream().synchronize()

    cs = ClockSampler(local_rank)       # NVML is initialised here, outside the timed region
    for _ in range(max(args.warmup, 3)):
        step_device()
    launches0 = _lib.launch_count(dev)
    with cs:
        ms = timer.timed(step_device, args.steps)
    launches = _lib.launch_count(dev) - launches0
    clocks = cs.summary()
    if args.dump_outputs and rank == 0:
        rgbd = last["rgbd"].float().cpu().numpy()
        os.makedirs(args.dump_outputs, exist_ok=True)
        np.save(os.path.join(args.dump_outputs, "rgb_fine.npy"), np.ascontiguousarray(rgbd[:, :3]))
        np.save(os.path.join(args.dump_outputs, "depth_fine.npy"), np.ascontiguousarray(rgbd[:, 3]))
    step_e2e()
    ms_e2e = timer.timed(step_e2e, args.steps)

    # ---- roofline of the dominant kernel: the fine-pass field kernel (65 536 rays x 128 samples) ----
    engine.PROFILE_EVENTS = []
    step_device()
    torch.cuda.synchronize()
    fine = [a.elapsed_time(b) for (a, b, n, s) in engine.PROFILE_EVENTS if s == N_SAMPLES + N_IMPORTANCE and n == CHUNK]
    coarse = [a.elapsed_time(b) for (a, b, n, s) in engine.PROFILE_EVENTS if s == N_SAMPLES and n == CHUNK]
    field_ms_total = sum(a.elapsed_time(b) for (a, b, n, s) in engine.PROFILE_EVENTS)
    engine.PROFILE_EVENTS = None
    fine_ms = statistics.mean(fine)
    flops = CHUNK * (N_SAMPLES + N_IMPORTANCE) * FLOP_PER_SAMPLE
    achieved = flops / (fine_ms * 1e-3) / 1e12
    peak = peaks["bf16_tflops_sustained"] if args.precision == "bf16" else 67.0   # H100 SXM data sheet, FP32 non-tensor

    extras = {}
    if not args.no_extras:
        if world > 1:
            # ---- strong scaling: ONE frame, contiguous ray tiles over the ranks, gather inside the timed region ----
            def step_strong():
                return parallel.render_sharded(lambda r, pr: {"rgbd": render(r, pr["codes"])}, rays_dev, {"codes": codes_dev},
                                               ["rgbd"])["rgbd"]
            for _ in range(3):
                step_strong()
            ms_s = timer.timed(step_strong, args.steps * 2)
            extras["strong"] = {"workload": "ONE 640x480 frame tile-sharded over the ranks (parallel.render_sharded), all-gather "
                                            "of (rgb, depth) inside the timed region", "ms_per_frame": ms_s / (args.steps * 2),
                                "rays_per_s": N_RAYS * args.steps * 2 / (ms_s * 1e-3), "rays_per_rank": math.ceil(N_RAYS / world),
                                "scaling": "strong"}
        extras["train"] = run_train(args, rank, world, dev, sc, timer, peaks)
        if rank == 0 and world == 1:
            try:
                extras["edit"] = run_edit(args, dev, sc, models, embeddings)
            except Exception as ex:
                extras["edit"] = {"error": f"{type(ex).__name__}: {ex}"[:200]}
    timer.barrier()
    if rank != 0:
        return
    value = N_RAYS * world * args.steps / (ms * 1e-3)
    e2e = N_RAYS * world * args.steps / (ms_e2e * 1e-3)
    line = {
        "metric": "rays/s", "value": value, "unit": "rays/s", "n_gpus": world, "steps": args.steps,
        "warmup": max(args.warmup, 3), "ms_per_step": ms / args.steps, "higher_is_better": True, "scaling": "weak",
        "vs_baseline": None, "dtype": args.precision, "data": "synthetic",
        "config": {"workload": WORKLOAD, "rays_per_step_per_gpu": N_RAYS, "chunk_rays": CHUNK,
                   "parallelism": f"ray-sharded dp{world}" if world > 1 else "single GPU",
                   "l2": "no explicit flush: each step streams ~3 GB of intermediates (>> 50 MB L2)",
                   "tflops_algorithmic_whole_step": N_RAYS * world * FLOP_PER_RAY * args.steps / (ms * 1e-3) / 1e12},
        "clocks": clocks,
        "e2e": {"value": e2e, "unit": "rays/s", "h2d_bytes_per_step": N_RAYS * (8 * 4 + 8),
                "d2h_bytes_per_step": N_RAYS * 4 * 4},
        "gpu_launches": launches,
        "roofline": {"bound": "tensor", "kernel": "field_tc_kernel (wgmma, voxel) fine pass (65536 rays x 128 samples)",
                     "achieved": achieved, "peak": peak, "unit": "TFLOP/s", "frac": achieved / peak,
                     "peak_source": f"{peaks_kind} bf16_tflops_sustained (kernel timed inside the step)",
                     "flops_per_launch": flops, "ms_per_launch": fine_ms,
                     "ms_per_launch_coarse": statistics.mean(coarse) if coarse else None,
                     "field_kernel_share_of_step": field_ms_total / (ms / args.steps)},
    }
    line.update(extras)
    if world == 1 and not args.no_cpu:
        cpu, sel, ref = cpu_baseline_sample(sc)
        line["cpu_baseline"] = cpu
        # ---- parity at the benchmark configuration: the same 4 096 rays on the GPU vs the reference output ----
        sel_d = sel.to(dev)
        with torch.no_grad():
            got = {p: render_rays(models, embeddings, rays_dev[sel_d], N_samples=N_SAMPLES, perturb=0, noise_std=0,
                                  N_importance=N_IMPORTANCE, embedding_instance=codes_dev[sel_d], is_eval=True, precision=p)
                   for p in ("bf16", "fp32")}
        cpu_ = lambda t: t.detach().float().cpu()
        par = {"rays": int(sel.numel()), "against": cpu["kind"], "bench_precision": args.precision}
        for p in ("bf16", "fp32"):
            par[f"psnr_rgb_fine_{p}"] = psnr(cpu_(got[p]["rgb_fine"]), ref["rgb_fine"])
            par[f"max_abs_rgb_fine_{p}"] = (cpu_(got[p]["rgb_fine"]) - ref["rgb_fine"]).abs().max().item()
            par[f"max_abs_depth_fine_{p}"] = (cpu_(got[p]["depth_fine"]) - ref["depth_fine"]).abs().max().item()
            par[f"max_abs_rgb_instance_fine_{p}"] = (cpu_(got[p]["rgb_instance_fine"]) - ref["rgb_instance_fine"]).abs().max().item()
        # PSNR of each render against a noisy "photograph" of the reference render (30 dB): the delta is what a user sees
        g = torch.Generator().manual_seed(0)
        photo = (ref["rgb_fine"] + torch.randn(ref["rgb_fine"].shape, generator=g) * 10 ** (-30 / 20)).clamp(0, 1)
        base = psnr(ref["rgb_fine"], photo)
        par["psnr_delta_vs_reference_bf16"] = psnr(cpu_(got["bf16"]["rgb_fine"]), photo) - base
        par["psnr_delta_vs_reference_fp32"] = psnr(cpu_(got["fp32"]["rgb_fine"]), photo) - base
        line["parity"] = par
        if not args.no_extras:
            line["gpu_torch_baseline"] = gpu_torch_baseline(sc, dev)
    print(json.dumps(line))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--precision", default="bf16", choices=["bf16", "fp32"])
    ap.add_argument("--no-cpu", action="store_true", help="skip the cpu_baseline / parity legs (development runs)")
    ap.add_argument("--no-extras", action="store_true", help="headline only: skip train / strong / edit / gpu baseline")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write the last timed step's outputs (rgb_fine, depth_fine) as DIR/<name>.npy (float32)")
    args = ap.parse_args()
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    if args.impl == "reference":
        run_reference(args, rank, world)
        return
    if world > 1:
        import torch.distributed as dist
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        if os.environ.get("NCCL_DEBUG", "").upper() == "VERSION":
            os.environ["NCCL_DEBUG"] = "WARN"      # the version banner goes to stdout: keep stdout to the one JSON line
        dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
    try:
        run_ours(args, rank, world, local_rank)
    finally:
        if world > 1:
            import torch.distributed as dist
            dist.destroy_process_group()


if __name__ == "__main__":
    main()
