"""One voxel-pruning pass (EmbeddingVoxel.self_pruning_empty_voxels, 16^3 samples per occupied voxel) two ways, on the
bench grid (synthetic.make_grid(seed=5, 42 x 42 x 22, 60 % occupied), occupancy = idx_map >= 0, the fine weights of
bench.build_scene) before and after one voxel_subdivision:

  a  the route before the device pass: the host loop over 32-voxel chunks, torch jitter and points,
     rendering.query_sigma (bf16 fused field, every point a one-sample ray), torch alpha and max
     (`_sigma_fn=lambda p: rendering.query_sigma(model, emb, p, precision="bf16")`)
  b  the device pass: onerf_prune_measure (one fused tensor-core launch, bf16) + onerf_prune_apply

First, with one injected jitter, both arms must prune the same voxels.  Then the arms alternate, each run on a fresh
copy of the grid.  Per grid and arm: median / min / max of the pass's wall time (ending in the count's host read, which
both arms make), samples/s, algorithmic TFLOP/s at 1 195 520 FLOP per sample (xyz_encoding_1..8 + sigma,
models/nerf_model.py:97-112), the peak of torch's allocator, and the card's name and power limit read in this run.
There is no CPU mode.

    python tools/prune_bench.py [--runs 5]
"""
import argparse
import copy
import json
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

FLOP_PER_SAMPLE = 1_195_520
SAMPLES = 4096


def card():
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip()
    name, limit = [s.strip() for s in out.split(",")]
    return {"gpu": name, "power_limit": limit}


def arm_a(emb, model, rand=None):
    from object_nerf_b200 import rendering
    return emb.self_pruning_empty_voxels(model, _rand=rand,
                                         _sigma_fn=lambda p: rendering.query_sigma(model, emb, p, precision="bf16"))


def arm_b(emb, model, rand=None):
    return emb.self_pruning_empty_voxels(model, precision="bf16", _rand=rand)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("prune_bench.py measures on a CUDA device; none is available")
    import bench
    from object_nerf_b200 import synthetic as S
    dev = torch.device("cuda:0")
    info = card()
    sc = bench.build_scene()
    model = S.make_model(sc["weights"]["fine"], True, dev).eval()
    base = S.make_embedding(sc["grid"]).to(dev)
    subdivided = copy.deepcopy(base)
    subdivided.voxel_subdivision()
    arms = {"a_host_loop_query_sigma": arm_a, "b_device_pass": arm_b}
    result = {**info, "runs": args.runs, "flop_per_sample": FLOP_PER_SAMPLE, "grids": {}}
    for gname, grid in (("bench", base), ("bench_subdivided", subdivided)):
        k = int(grid.voxel_occupancy.sum())
        # agreement: one injected jitter, the same voxels pruned
        g = torch.Generator(device=dev).manual_seed(1)
        rand = [torch.rand(32 * SAMPLES, 3, device=dev, generator=g) for _ in range((k + 31) // 32)]
        grids = {}
        for name, fn in arms.items():
            e = copy.deepcopy(grid)
            n = fn(e, model, rand)
            grids[name] = (n, e.voxel_occupancy.clone(), e.voxel_idx_map.clone())
        (na, oa, ia), (nb, ob, ib) = grids.values()
        assert na == nb and torch.equal(oa, ob) and torch.equal(ia, ib), f"{gname}: the arms prune different voxels"
        del rand, grids
        torch.cuda.empty_cache()
        wall, peak, pruned = ({a: [] for a in arms} for _ in range(3))
        for _ in range(args.runs):
            for name, fn in arms.items():
                e = copy.deepcopy(grid)
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                t0 = time.perf_counter()
                pruned[name].append(fn(e, model))
                torch.cuda.synchronize()
                wall[name].append((time.perf_counter() - t0) * 1e3)
                peak[name].append(torch.cuda.max_memory_allocated())
                del e
        out = {"occupied_voxels": k, "samples": k * SAMPLES, "pruned_agreement_check": na, "arms": {}}
        for name in arms:
            med = statistics.median(wall[name])
            out["arms"][name] = {
                "ms": {"median": round(med, 2), "min": round(min(wall[name]), 2), "max": round(max(wall[name]), 2)},
                "samples_per_s": round(k * SAMPLES / (med / 1e3)),
                "algorithmic_tflops": round(k * SAMPLES * FLOP_PER_SAMPLE / (med / 1e3) / 1e12, 1),
                "peak_allocated_bytes": max(peak[name]), "pruned": pruned[name]}
        out["speedup_b_over_a"] = round(statistics.median(wall["a_host_loop_query_sigma"]) /
                                        statistics.median(wall["b_device_pass"]), 2)
        result["grids"][gname] = out
    print(json.dumps(result))


if __name__ == "__main__":
    main()
