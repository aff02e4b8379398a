"""Phase timeline of the fused forward kernel (field_tc_kernel) in the bench frame's fine pass.

Builds an instrumented copy of the library (-DONERF_FIELD_TIMELINE) into a temporary directory, renders one bench-shaped
chunk (65 536 rays, 64 + 64 samples: the last field launch is the 65 536 x 128 fine pass, voxel model, both branches)
and prints cycles per tile for each phase, from clock64 stamps of lane 0 of each warpgroup in the first 16 tiles of
CTAs 0-7.  The first tile of each CTA is reported apart from the steady-state tiles (median over the others).

    python tools/field_timeline.py [--json OUT]

Slots of a consumer record (field_tc.cu): 0 tile start, 1 X ready, 2 rows read (layers start), for the layer with
activation slot s (1..16, GEMM index + 1) 3s first MMA issue, 3s + 1 after wgmma.wait_group 0, 3s + 2 epilogue end,
51 heads written, 52 tile end, 55 + s cycles spent in the layer's ring full-barrier waits.  Encoder record (warpgroup 2):
0 tile start, 1 every job written (the gathers run before, the shared-memory stores after the wait for X to be free),
2 x_full arrived.
"""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import shutil
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "object_nerf_b200", "csrc")
TL_CTAS, TL_TILES, TL_SLOTS = 8, 16, 80
LAYERS = ["S0", "S1", "S2", "S3", "S4", "S5", "S6", "S7", "SFIN", "SDIR", "O0", "O1", "O2", "O3", "OFIN", "ODIR"]


def build_instrumented(out_dir: str) -> str:
    """Copy the sources (csrc/ and include/, same relative layout) to out_dir and build them there."""
    src = os.path.join(out_dir, "object_nerf_b200", "csrc")
    shutil.copytree(CSRC, src, ignore=shutil.ignore_patterns("build", "*.so"))
    shutil.copytree(os.path.join(ROOT, "include"), os.path.join(out_dir, "include"))
    r = subprocess.run(["make", "-C", src, "EXPERIMENT=ONERF_FIELD_TIMELINE", "-j16"], capture_output=True, text=True)
    if r.returncode != 0:
        sys.exit("instrumented build failed:\n" + r.stdout[-3000:] + r.stderr[-3000:])
    return os.path.join(out_dir, "object_nerf_b200", "libonerf_sm90.so")


def run(lib_path: str):
    os.environ["ONERF_LIB_PATH"] = lib_path
    sys.path.insert(0, ROOT)
    import torch
    import bench
    from object_nerf_b200 import Embedding, _lib, render_rays, synthetic as S

    dev = torch.device("cuda", 0)
    sc = bench.build_scene()
    models = {k: S.make_model(w, True, dev) for k, w in sc["weights"].items()}
    emb = S.GridModule(sc["grid"]).to(dev)
    rays, codes = sc["rays"][:bench.CHUNK].to(dev), sc["codes"][:bench.CHUNK].to(dev)
    buf = torch.zeros(TL_CTAS * 3 * TL_TILES * TL_SLOTS, dtype=torch.int64, device=dev)
    lib = _lib.load()
    lib.onerf_field_timeline.argtypes = [ctypes.c_void_p]

    def render():
        with torch.no_grad():
            render_rays(models, {"xyz": emb, "dir": Embedding(3, 4)}, rays, N_samples=bench.N_SAMPLES, use_disp=False,
                        perturb=0, noise_std=0, N_importance=bench.N_IMPORTANCE, chunk=32768, white_back=False,
                        embedding_instance=codes, is_eval=True)
        torch.cuda.synchronize()

    render()                                  # warm-up: module load, first-touch of the weights
    lib.onerf_field_timeline(ctypes.c_void_p(buf.data_ptr()))
    render()                                  # the fine pass is the last field launch: its stamps remain
    lib.onerf_field_timeline(None)
    props = torch.cuda.get_device_properties(dev)
    return buf.view(TL_CTAS, 3, TL_TILES, TL_SLOTS).cpu().numpy(), props.name


def phases(rec):
    """-> {phase: cycles} for one consumer tile record (rec[slot]); absent phases are skipped."""
    out = {"encode / wait for X (tile start -> X ready)": rec[1] - rec[0], "rows read / X dump": rec[2] - rec[1]}
    ends = []
    for s in range(1, 17):
        if rec[3 * s] == 0:
            continue
        name = LAYERS[s - 1]
        out[f"{name} MMA"] = rec[3 * s + 1] - rec[3 * s]
        out[f"{name} full-barrier wait"] = rec[55 + s]
        out[f"{name} epilogue"] = rec[3 * s + 2] - rec[3 * s + 1]
        ends.append(rec[3 * s + 2])
    out["heads (last epilogue -> heads written)"] = rec[51] - max(ends)
    out["tile tail (heads -> tile end)"] = rec[52] - rec[51]
    out["tile total"] = rec[52] - rec[0]
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--json", help="also write the table as JSON to this path")
    args = ap.parse_args()
    with tempfile.TemporaryDirectory(prefix="onerf_timeline_") as tmp:
        stamps, gpu = run(build_instrumented(tmp))
    rows = {}
    for cta in range(TL_CTAS):
        for wg in range(2):
            for k in range(TL_TILES):
                rec = [int(v) for v in stamps[cta, wg, k]]
                if rec[52] == 0:
                    continue
                for name, v in phases(rec).items():
                    rows.setdefault(name, {"first": [], "steady": []})["first" if k == 0 else "steady"].append(v)
    enc = {"tile start -> X written (gathers + wait for X free + stores)": [], "fence + x_full arrive": []}
    for cta in range(TL_CTAS):
        for k in range(TL_TILES):
            rec = [int(v) for v in stamps[cta, 2, k]]
            if rec[2] == 0:
                continue
            enc["tile start -> X written (gathers + wait for X free + stores)"].append(rec[1] - rec[0])
            enc["fence + x_full arrive"].append(rec[2] - rec[1])
    med = lambda v: statistics.median(v) if v else float("nan")
    total = med(rows["tile total"]["steady"])
    print(f"{gpu}: field_tc_kernel fine pass, cycles per tile (median over {len(rows['tile total']['steady'])} "
          f"steady-state tile records; first tile of each CTA apart)")
    print(f"{'phase':42s} {'steady':>9s} {'share':>7s} {'first':>9s}")
    for name, v in rows.items():
        s = med(v["steady"])
        print(f"{name:42s} {s:9.0f} {100 * s / total:6.1f}% {med(v['first']):9.0f}")
    for name, v in enc.items():
        if v:
            print(f"encoder warps: {name:60s} {med(v):9.0f}")
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"gpu": gpu, "consumer": {k: {"steady": med(v["steady"]), "first": med(v["first"])}
                                                for k, v in rows.items()},
                       "encoder": {k: med(v) for k, v in enc.items() if v}}, f, indent=1)


if __name__ == "__main__":
    main()
