"""Generate tests/golden/*.npz by running the REAL reference (/root/reference, CPU) on the
deterministic synthetic scenes of tests/synth.py.  Run in the build container only:

    python tools/make_golden.py                    # every fixture
    python tools/make_golden.py grad_case_plain    # only the named generators (see GENERATORS)

The fixtures hold reference OUTPUTS (and the case parameters); inputs are regenerated from seeds by
tests/cases.py (tests/grad_plain.py for the plain-PE training step), which is shared by this script, the CPU oracle
tests and the GPU parity tests.
The reference draws RNG inside the path (models/rendering.py:40,156,187,276); to pin those branches
the torch.rand* entry points are patched for the duration of a reference call so that it consumes
the pre-drawn buffers of synth.random_buffers in call order.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import ref_import as R  # noqa: E402

R.install()
from models.rendering import render_rays as ref_render_rays, sample_pdf as ref_sample_pdf  # noqa: E402
from models.nerf_model import ObjectNeRF  # noqa: E402
from models.embedding_helper import Embedding, EmbeddingVoxel  # noqa: E402
from render_tools.multi_rendering import render_rays_multi as ref_render_rays_multi  # noqa: E402
from utils.bbox_utils import BBoxRayHelper  # noqa: E402

from tests import cases, grad_plain, synth  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")

REF_NAMES = {  # oracle layout -> reference attribute (models/nerf_model.py:41-58,77-95)
    **{f"scene.l{i}": f"xyz_encoding_{i+1}.0" for i in range(8)},
    "scene.final": "xyz_encoding_final", "scene.sigma": "sigma", "scene.dir": "dir_encoding.0",
    "scene.rgb": "rgb.0",
    **{f"obj.l{i}": f"instance_encoding_{i+1}.0" for i in range(4)},
    "obj.final": "instance_encoding_final.0", "obj.sigma": "instance_sigma",
    "obj.dir": "inst_dir_encoding.0", "obj.rgb": "inst_rgb.0",
}


def ref_model(w, use_voxel):
    m = ObjectNeRF(R.default_model_config(use_voxel))
    sd = {}
    for k, (W, b) in w.items():
        sd[REF_NAMES[k] + ".weight"] = W
        sd[REF_NAMES[k] + ".bias"] = b
    m.load_state_dict(sd, strict=True)
    return m.eval()


def ref_voxel_embedding(grid):
    """Build the reference EmbeddingVoxel on a throw-away cloud, then overwrite the buffers the hot path
    reads with the synthetic grid (the cold-path constructor is pinned separately in case 'gridbuild')."""
    R.register_pointcloud("tiny.ply", np.array([[0.0, 0, 0], [0.2, 0.2, 0.2]]))
    extra = R.AttrDict(pcd_path="tiny.ply", scene_center=[0, 0, 0], scale_factor=1.0, voxel_size=0.1,
                       neighbor_marks=3)
    emb = EmbeddingVoxel(24, 6, grid["table"].shape[0], extra)
    emb.voxel_size = grid["voxel_size"].clone()
    emb.voxel_offset = grid["offset"].clone()
    emb.voxel_shape = grid["shape"].clone()
    emb.voxel_idx_map = grid["idx_map"].clone()
    with torch.no_grad():
        emb.embedding_space_ftr.weight.copy_(grid["table"])
    return emb


class InjectRandom:
    """Patch torch.rand / rand_like / randn_like to hand out pre-drawn buffers in call order."""

    def __init__(self, rand_like_seq, rand_seq, randn_like_seq):
        self.seqs = {"rand_like": list(rand_like_seq), "rand": list(rand_seq), "randn_like": list(randn_like_seq)}

    def __enter__(self):
        self.saved = (torch.rand_like, torch.rand, torch.randn_like)
        torch.rand_like = lambda t, *a, **k: self._next("rand_like", t.shape)
        torch.rand = lambda *a, **k: self._next("rand", tuple(a))
        torch.randn_like = lambda t, *a, **k: self._next("randn_like", t.shape)
        return self

    def _next(self, kind, shape):
        buf = self.seqs[kind].pop(0)
        assert tuple(buf.shape) == tuple(shape), (kind, buf.shape, shape)
        return buf.clone()

    def __exit__(self, *exc):
        torch.rand_like, torch.rand, torch.randn_like = self.saved


def save(name, **arrays):
    os.makedirs(OUT, exist_ok=True)
    path = os.path.join(OUT, name + ".npz")
    np.savez_compressed(path, **{k: (v.detach().numpy() if torch.is_tensor(v) else np.asarray(v))
                                 for k, v in arrays.items()})
    print("wrote", path, os.path.getsize(path), "bytes")


def gen_stage_cases():
    # positional encoding
    x = cases.stage_inputs()["posenc_x"]
    save("stage_posenc", pe10=Embedding(3, 10)(x), pe4=Embedding(3, 4)(x))
    # voxel embedding
    grid = synth.make_grid(**cases.GRID_KW)
    emb = ref_voxel_embedding(grid)
    xyz = cases.stage_inputs()["voxel_xyz"]
    with torch.no_grad():
        scene_in, obj_in = emb(xyz.clone())
    save("stage_voxel", scene_in=scene_in, obj_in=obj_in)
    # MLP branches on synthetic embeddings
    si = cases.stage_inputs()
    for use_voxel in (True, False):
        w = synth.make_weights(11, use_voxel, sigma_gain=8.0, sigma_bias=1.0)
        m = ref_model(w, use_voxel)
        ex = si["emb_xyz_v"] if use_voxel else si["emb_xyz_p"]
        with torch.no_grad():
            o = m({"emb_xyz": ex, "emb_dir": si["emb_dir"]})
            oi = m.forward_instance({"emb_xyz": ex, "emb_dir": si["emb_dir"],
                                     "obj_voxel": si["obj_voxel"] if use_voxel else None,
                                     "obj_code": si["obj_code"]})
        save(f"stage_mlp_{'voxel' if use_voxel else 'plain'}", sigma=o["sigma"][:, 0], rgb=o["rgb"],
             inst_sigma=oi["inst_sigma"][:, 0], inst_rgb=oi["inst_rgb"])
    # sample_pdf, deterministic and with injected u
    bins, wts, u = si["pdf_bins"], si["pdf_weights"], si["pdf_u"]
    det = ref_sample_pdf(bins, wts, 64, det=True)
    with InjectRandom([], [u], []):
        rnd = ref_sample_pdf(bins, wts, 64, det=False)
    save("stage_sample_pdf", det=det, rnd=rnd)


def gen_render_cases():
    for name, c in cases.RENDER_CASES.items():
        inp = cases.build_render_case(c)
        use_voxel = c["use_voxel"]
        models = {"coarse": ref_model(inp["weights"]["coarse"], use_voxel)}
        if c["n_importance"] > 0:
            models["fine"] = ref_model(inp["weights"]["fine"], use_voxel)
        emb_xyz = ref_voxel_embedding(inp["grid"]) if use_voxel else Embedding(3, 10)
        embeddings = {"xyz": emb_xyz, "dir": Embedding(3, 4)}
        r = inp["rand"]
        kw = dict(N_samples=c["n_samples"], use_disp=c["use_disp"], perturb=c["perturb"],
                  noise_std=c["noise_std"], N_importance=c["n_importance"], chunk=c.get("chunk", 32768),
                  white_back=c["white_back"], forward_instance=c["forward_instance"],
                  embedding_instance=inp["codes"], frustum_bound_th=c["frustum_bound_th"],
                  pass_through_mask=inp["pass_through_mask"], rays_in_bbox=c["rays_in_bbox"],
                  is_eval=c["is_eval"])
        rand_like = [r["jitter"]] if c["perturb"] > 0 else []
        rand = [r["u"]] if (c["perturb"] > 0 and c["n_importance"] > 0) else []
        randn = [r["noise_scene_coarse"]] + ([r["noise_obj_coarse"]] if c["forward_instance"] else [])
        if c["n_importance"] > 0:
            randn += [r["noise_scene_fine"]] + ([r["noise_obj_fine"]] if c["forward_instance"] else [])
        with torch.no_grad(), InjectRandom(rand_like, rand, randn):
            out = ref_render_rays(models, embeddings, inp["rays"], **kw)
        save("render_" + name, **out)


def _ref_multi_inputs(inp):
    """The reference's models, embeddings, code library and removed-object box helpers of a multi case."""
    models = {"coarse": ref_model(inp["weights"]["coarse"], True), "fine": ref_model(inp["weights"]["fine"], True)}
    embeddings = {"xyz": ref_voxel_embedding(inp["grid"]), "dir": Embedding(3, 4)}

    class Lib(torch.nn.Module):
        def __init__(self, table):
            super().__init__()
            self.embedding_instance = torch.nn.Embedding.from_pretrained(table)

    boxes = None
    if inp["boxes"]:
        boxes = {}
        for k, b in enumerate(inp["boxes"]):
            h = object.__new__(BBoxRayHelper)   # bypass the file-reading ctor (utils/bbox_utils.py:10-24)
            h.scale_factor = b["scale_factor"]
            h.pose_avg = b["pose_avg"]
            h.axis_align_mat = b["axis_align_mat"]
            h.bbox_bounds = b["bbox_bounds"]
            boxes[k] = h
    return models, embeddings, Lib(inp["code_table"]), boxes


def gen_multi_cases():
    for name, c in cases.MULTI_CASES.items():
        inp = cases.build_multi_case(c)
        models, embeddings, lib, boxes = _ref_multi_inputs(inp)
        with torch.no_grad():
            out = ref_render_rays_multi(models, embeddings, lib, inp["rays_list"],
                                        c["obj_ids"], N_samples=c["n_samples"], use_disp=False, perturb=0,
                                        noise_std=0, N_importance=c["n_importance"], chunk=c.get("chunk", 32768),
                                        white_back=c["white_back"], background_skip_bbox=boxes)
        save("multi_" + name, **out)


def gen_multi_noise_clip_cases():
    """render_rays_multi with sigma noise, perturbed importance sampling and 10-column ray sets
    (tests/multi_noise_cases.py).  The reference draws randn_like over the sorted sigmas once per pass
    (render_tools/multi_rendering.py:131) and torch.rand (N, K) once per set in sample_pdf (models/rendering.py:40);
    InjectRandom hands it the case's buffers in that order."""
    from tests import multi_noise_cases as M
    for name, c in M.NOISE_CLIP_CASES.items():
        inp = M.build_noise_clip_case(c)
        models, embeddings, lib, boxes = _ref_multi_inputs(inp)
        r = inp["rand"]
        rand = list(r["u"]) if c["perturb"] != 0 else []
        with torch.no_grad(), InjectRandom([], rand, [r["noise_coarse"], r["noise_fine"]]) as inj:
            out = ref_render_rays_multi(models, embeddings, lib, inp["rays_list"], c["obj_ids"],
                                        N_samples=c["n_samples"], use_disp=False, perturb=c["perturb"],
                                        noise_std=c["noise_std"], N_importance=c["n_importance"], chunk=32768,
                                        white_back=c["white_back"], background_skip_bbox=boxes)
        assert not any(inj.seqs.values()), "the reference drew fewer random tensors than the case injects"
        save("multi_" + name, **out)


def gen_grad_case():
    """Training step through the REAL reference: render_rays (train mode, injected RNG) -> reference TotalLoss ->
    backward.  The fixture keeps the loss and, per parameter tensor, its L2 norm, sum and sampled entries."""
    _gen_grad(cases.GRAD_CASE, cases.build_grad_case(), "grad_train_step")


def gen_grad_case_plain():
    """The same training step on the plain positional-encoding model (Embedding(3, 10) as the xyz embedding): the
    fixture has the keys of grad_train_step minus voxel|*."""
    _gen_grad(grad_plain.GRAD_CASE_PLAIN, grad_plain.build_grad_case_plain(), "grad_train_step_plain")


def _gen_grad(c, inp, name):
    from models.losses import TotalLoss
    from models.code_library import CodeLibrary
    use_voxel = c["use_voxel"]
    models = {"coarse": ref_model(inp["weights"]["coarse"], use_voxel).train(),
              "fine": ref_model(inp["weights"]["fine"], use_voxel).train()}
    emb = ref_voxel_embedding(inp["grid"]) if use_voxel else Embedding(3, 10)
    lib = CodeLibrary(R.default_model_config())
    with torch.no_grad():
        lib.embedding_instance.weight.copy_(inp["code_table"])
    codes = lib({"instance_ids": inp["instance_ids"]})["embedding_instance"]
    r = inp["rand"]
    with InjectRandom([r["jitter"]], [r["u"]], [r["noise_scene_coarse"], r["noise_obj_coarse"], r["noise_scene_fine"],
                                               r["noise_obj_fine"]]):
        out = ref_render_rays(models, {"xyz": emb, "dir": Embedding(3, 4)}, inp["rays"], N_samples=c["n_samples"],
                              use_disp=False, perturb=c["perturb"], noise_std=c["noise_std"],
                              N_importance=c["n_importance"], chunk=32768, white_back=False,
                              embedding_instance=codes, frustum_bound_th=c["frustum_bound_th"],
                              pass_through_mask=inp["pass_through_mask"], rays_in_bbox=False, is_eval=False)
    loss, _ = TotalLoss(R.AttrDict(cases.LOSS_CONF))(out, inp["batch"])
    # our restatement of the loss must agree with the reference's
    assert abs(cases.total_loss(out, inp["batch"]).item() - loss.item()) < 1e-5 * max(1.0, abs(loss.item()))
    loss.backward()
    fix = {"loss": loss.detach()}
    named = [(f"{typ}.{k}", p) for typ, m in models.items() for k, p in m.named_parameters()]
    named += [("codes", lib.embedding_instance.weight)]
    if use_voxel:
        named += [("voxel", emb.embedding_space_ftr.weight)]
    for pname, p in named:
        g = p.grad.reshape(-1)
        fix[pname + "|norm"] = g.norm()
        fix[pname + "|sum"] = g.sum()
        fix[pname + "|samples"] = g[cases.sample_indices(pname, g.numel())]
    if use_voxel:
        nz = torch.nonzero(emb.embedding_space_ftr.weight.grad.abs().sum(1)).view(-1)
        fix["voxel|nonzero_rows"] = nz
        print("voxel rows touched", nz.numel())
    save(name, **fix)
    print(name, "loss", loss.item())


def gen_gridbuild():
    """Cold path pin: the reference's EmbeddingVoxel constructor on a synthetic cloud (ScanNet-0113-like
    voxel_size / scale_factor / scene_center, config/scannet_base_0113_multi.yml:7-11,43-44)."""
    pts = np.random.default_rng(0).uniform([0, 0, -1], [4, 4, 1], size=(20000, 3))
    R.register_pointcloud("synthetic", pts)
    extra = R.AttrDict(pcd_path="synthetic", scene_center=[2.0, 2.0, 0.0], scale_factor=2.0, voxel_size=0.1,
                       neighbor_marks=3)
    emb = EmbeddingVoxel(24, 6, 50000, extra)
    save("gridbuild", voxel_shape=emb.voxel_shape, voxel_idx_map=emb.voxel_idx_map, voxel_offset=emb.voxel_offset,
         voxel_size=emb.voxel_size)


def gen_ray_cases():
    """SURVEY section 8f rows 1-2: the reference's own get_ray_directions / get_rays (datasets/ray_utils.py) and
    BBoxRayHelper.get_ray_bbox_intersections (utils/bbox_utils.py:132-156, numba slab test of datasets/geo_utils.py).
    The helper's constructor parses dataset files, so an instance is made without it and given the three attributes
    the method reads."""
    from datasets.ray_utils import get_ray_directions, get_rays
    from utils.bbox_utils import BBoxRayHelper
    for name, c in cases.CAMERA_CASES.items():
        inp = cases.build_camera_case(c)
        directions = get_ray_directions(inp["H"], inp["W"], inp["focal"])
        rays_o, rays_d = get_rays(directions, inp["c2w"])
        save("rays_" + name, directions=directions, rays_o=rays_o.contiguous(), rays_d=rays_d)
    for name, c in cases.BBOX_CASES.items():
        inp = cases.build_bbox_case(c)
        h = object.__new__(BBoxRayHelper)
        h.pose_avg, h.axis_align_mat, h.bbox_bounds = inp["pose_avg"], inp["axis_align_mat"], inp["bbox_bounds"]
        h.scale_factor = inp["scale_factor"]
        mask, near, far = h.get_ray_bbox_intersections(inp["rays_o"], inp["rays_d"], inp["scale_factor"],
                                                       bbox_enlarge=inp["bbox_enlarge"])
        save("rays_" + name, mask=mask, near=near, far=far)
        print(name, "hits", int(mask.sum()), "of", mask.numel())


def gen_loss_cases():
    """SURVEY section 8f row 3: the reference's TotalLoss (models/losses.py) and its autograd gradients on random maps."""
    from models.losses import TotalLoss
    for name, c in cases.LOSS_CASES.items():
        maps, batch = cases.build_loss_case(c)
        maps = {k: v.clone().requires_grad_(True) for k, v in maps.items()}
        loss_sum, loss_dict = TotalLoss(dict(cases.LOSS_CONF))(maps, batch)
        loss_sum.backward()
        fix = {"loss_sum": loss_sum.detach()}
        for k, v in loss_dict.items():
            fix["term|" + k] = v.detach()
        for k, v in maps.items():
            fix["grad|" + k] = v.grad if v.grad is not None else torch.zeros_like(v)
        save(name, **fix)
        print(name, float(loss_sum.detach()), sorted(loss_dict))


def _maint_embedding():
    inp = cases.build_maint_case()
    c = cases.MAINT_CASE
    R.register_pointcloud(c["extra"]["pcd_path"], inp["points"])
    emb = EmbeddingVoxel(24, 6, c["max_voxels"], R.AttrDict(c["extra"]))
    with torch.no_grad():
        emb.embedding_space_ftr.weight.copy_(inp["table"])
    return emb, inp


def _grid_state(emb, prefix):
    n = int(torch.nonzero(emb.voxel_occupancy).shape[0])
    return {prefix + "voxel_size": emb.voxel_size.clone(), prefix + "voxel_shape": emb.voxel_shape.clone(),
            prefix + "voxel_occupancy": emb.voxel_occupancy.clone(), prefix + "voxel_idx_map": emb.voxel_idx_map.clone(),
            prefix + "table_rows": emb.embedding_space_ftr.weight.detach()[:n].clone()}


def gen_maint_cases():
    """SURVEY section 8f row 4: EmbeddingVoxel.voxel_subdivision and self_pruning_empty_voxels of the reference
    (models/embedding_helper.py:202-302).  The pruning routine calls `model(voxel_ftrs, sigma_only=True)` and unpacks two
    results (:223) although ObjectNeRF.forward takes a dict and returns a dict; the adapter below gives it exactly that
    call shape on top of the reference model (sigma of the scene branch), nothing else is touched."""
    c = cases.MAINT_CASE
    emb, inp = _maint_embedding()
    fix = _grid_state(emb, "before|")
    emb.voxel_subdivision()
    fix.update(_grid_state(emb, "subdiv|"))
    save("maint_subdivision", **fix)

    emb, inp = _maint_embedding()
    model = ref_model(inp["weights"], True)

    def adapter(voxel_ftrs, sigma_only=True):
        with torch.no_grad():
            return model({"emb_xyz": voxel_ftrs}, sigma_only=True)["sigma"], None

    n_occu = int(torch.nonzero(emb.voxel_occupancy).shape[0])
    n_chunks = (n_occu + 31) // 32
    rand = cases.maint_rand(n_chunks)
    seq = []
    for k in range(n_chunks):
        n_here = min(32, n_occu - 32 * k) * 16 ** 3
        seq.append(rand[k][:n_here])
    with InjectRandom(seq, [], []):
        emb.self_pruning_empty_voxels(adapter, max_alpha_th=c["max_alpha_th"])
    fix = _grid_state(emb, "pruned|")
    fix["n_before"] = torch.tensor(n_occu)
    save("maint_pruning", **fix)
    print("pruning:", n_occu, "->", int(torch.nonzero(emb.voxel_occupancy).shape[0]))


GENERATORS = ("ray_cases", "maint_cases", "loss_cases", "gridbuild", "grad_case", "grad_case_plain", "stage_cases",
              "render_cases", "multi_cases", "multi_noise_clip_cases")

if __name__ == "__main__":
    torch.set_num_threads(8)
    if len(sys.argv) > 1:      # python tools/make_golden.py grad_case_plain ...: only the named generators
        unknown = [a for a in sys.argv[1:] if a not in GENERATORS]
        if unknown:
            sys.exit(f"unknown generator(s) {unknown}; choose from {list(GENERATORS)}")
        for a in sys.argv[1:]:
            globals()["gen_" + a]()
        sys.exit(0)
    gen_ray_cases()
    gen_maint_cases()
    gen_loss_cases()
    gen_gridbuild()
    gen_grad_case()
    gen_grad_case_plain()
    gen_stage_cases()
    gen_render_cases()
    gen_multi_cases()
    gen_multi_noise_clip_cases()
