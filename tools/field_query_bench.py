"""Points per second of field queries (ObjectNeRF.forward on embedded points, voxel model): the forward without grad
and forward + backward of sum(rgb * c) + sum(sigma * c'), at 2^20 points, bf16 and fp32.  Each timed call includes
the stand-alone encodings emb(pts) and Embedding(3, 4)(dirs) a caller makes (the fused kernel re-encodes from the
points they carry).  Where oracle/_ref is built, the unmodified reference ObjectNeRF / EmbeddingVoxel / Embedding run
the same calls on the same GPU (PyTorch eager, fp32 and TF32 matmuls).  CUDA events around `--iters` calls after
`--warmup` calls; the card's name and power limit are printed with the numbers.

  python tools/field_query_bench.py [--points 1048576] [--iters 5] [--warmup 2] [--out FILE.json]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from object_nerf_b200 import Embedding, synthetic as S   # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:   # noqa: BLE001
        q = f"unknown ({e})"
    return q


def _time(fn, a):
    for _ in range(a.warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / a.iters


def reference_arm(a, dev, g, pts, dirs, cot):
    """The same queries through the unmodified reference modules (oracle/_ref), or why they were not run."""
    from oracle import ref_loader as R
    if not R.available():
        return {"unavailable": "oracle/_ref not built"}
    R.install(cuda_noop=False)
    from models.embedding_helper import Embedding as RefEmbedding
    stdout = sys.stdout
    sys.stdout = open(os.devnull, "w")       # the voxel helper prints while it builds its throw-away grid
    try:
        model = R.ref_model(S.make_weights(11, True, 8.0, 1.0), True, dev).train()
        emb = R.ref_voxel_embedding(g, dev)
    finally:
        sys.stdout.close()
        sys.stdout = stdout
    emb_dir = RefEmbedding(3, 4)
    res = {"kind": "unmodified reference (oracle/_ref) on the same GPU, torch " + torch.__version__}

    def query():
        x, _ = emb(pts)
        out = model({"emb_xyz": x, "emb_dir": emb_dir(dirs)})
        return torch.cat([out["rgb"], out["sigma"]], 1)

    def forward():
        with torch.no_grad():
            query()

    def fwd_bwd():
        model.zero_grad(set_to_none=True)
        emb.zero_grad(set_to_none=True)
        (query() * cot).sum().backward()

    for tf32 in (False, True):
        torch.backends.cuda.matmul.allow_tf32 = tf32
        tag = "tf32" if tf32 else "fp32"
        for name, fn in (("forward", forward), ("forward_backward", fwd_bwd)):
            ms = _time(fn, a)
            res[f"{tag}_{name}_ms"] = ms
            res[f"{tag}_{name}_points_per_s"] = a.points / (ms * 1e-3)
    torch.backends.cuda.matmul.allow_tf32 = False
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, default=1 << 20)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("field_query_bench measures on a CUDA device; none found")
    dev = "cuda:0"
    model = S.make_model(S.make_weights(11, True, 8.0, 1.0), True, dev).train()
    g = S.make_grid(seed=5, shape=(42, 42, 22), occupancy=0.6, voxel_size=0.05)
    emb = S.make_embedding(g).to(dev)
    gen = torch.Generator(device=dev).manual_seed(0)
    ext = (g["shape"].float() * float(g["voxel_size"])).to(dev)
    pts = torch.rand(a.points, 3, device=dev, generator=gen) * ext - g["offset"].to(dev)
    dirs = torch.nn.functional.normalize(torch.randn(a.points, 3, device=dev, generator=gen), dim=1)
    cot = torch.randn(a.points, 4, device=dev, generator=gen)
    res = {"card": card(), "points": a.points, "iters": a.iters}

    def query():
        e = emb(pts)
        out = model({"emb_xyz": e[0], "emb_dir": Embedding(3, 4)(dirs)})
        return torch.cat([out["rgb"], out["sigma"]], 1)

    def forward():
        with torch.no_grad():
            query()

    def fwd_bwd():
        model.zero_grad(set_to_none=True)
        emb.zero_grad(set_to_none=True)
        (query() * cot).sum().backward()

    for prec in ("bf16", "fp32"):
        os.environ["ONERF_PRECISION"] = prec
        for name, fn in (("forward", forward), ("forward_backward", fwd_bwd)):
            ms = _time(fn, a)
            res[f"{prec}_{name}_ms"] = ms
            res[f"{prec}_{name}_points_per_s"] = a.points / (ms * 1e-3)
    res["peak_mem_gb"] = torch.cuda.max_memory_allocated() / 1e9
    res["reference"] = reference_arm(a, dev, g, pts, dirs, cot)

    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
