"""Training the plain positional-encoding model (the reference's use_voxel_embedding: false) on the tensor cores: the
training forward's dump, the backward stages at the one-X-atom layout against PyTorch fp32 references of the same ops,
and the whole step against the reference's own backward (fixture grad_train_step_plain) and against the fp32 path."""
import ctypes as C

import pytest
import torch

from tests import cases, grad_plain, helpers

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

GEMM_OF_DZ = ["S0", "S1", "S2", "S3", "S4", "S5", "S6", "S7", "SFIN", "SDIR", "O0", "O1", "O2", "O3", "OFIN", "ODIR"]
GEMM_N = dict(S0=256, S1=256, S2=256, S3=256, S4=256, S5=256, S6=256, S7=256, SFIN=256, SDIR=128,
              O0=128, O1=128, O2=128, O3=128, OFIN=128, ODIR=64)
# kernel-K widths of the plain layout (layout.h: KX = KO = 64, X column 63 is padding)
GEMM_K = dict(S0=64, S1=256, S2=256, S3=256, S4=320, S5=256, S6=256, S7=256, SFIN=256, SDIR=256,
              O0=64, O1=128, O2=192, O3=128, OFIN=128, ODIR=128)
WIDTHS = [64] + [256] * 8 + [256, 128] + [128] * 4 + [128, 64]    # activation slots, X first
XIN, OIN = 63, 127                                                  # reference scene / object input widths


def _lib():
    from object_nerf_b200 import _lib
    return _lib


def grad_layout():
    off, w_off, b_off = 0, {}, {}
    for g in GEMM_OF_DZ:
        w_off[g] = off
        off += GEMM_N[g] * GEMM_K[g]
        b_off[g] = off
        off += GEMM_N[g]
        off = (off + 3) // 4 * 4
    for n in (256, 1, 384, 3, 128, 1, 192, 3):
        off += (n + 3) // 4 * 4
    return w_off, b_off, off


def _plain_field_inputs(n_rays, S=64):
    from object_nerf_b200 import engine
    inp = cases.build_render_case(dict(cases.RENDER_CASES["eval_plain"], n_rays=n_rays))
    model = helpers.make_model(inp["weights"]["coarse"], False, DEV)
    rays = inp["rays"].to(DEV)
    z = engine.sample_coarse(rays, S)
    packed = engine.packed_for(model, False)
    return inp, model, rays, z, packed, inp["codes"].to(DEV)


def _training_forward(rays, z, packed, codes, T):
    """onerf_field_fwd with a training workspace (field_tc_kernel<false, true>) -> (scene, obj, ws)."""
    L = _lib()
    n, S = z.shape
    ws = helpers.aligned_u8(T["total"], DEV, fill=0)
    a = L.FieldArgs()
    scene = torch.empty(n, S, 4, device=DEV)
    obj = torch.empty(n, S, 4, device=DEV)
    rc = torch.empty(n, 448, device=DEV)
    a.rays, a.z, a.z_stride, a.codes = rays.data_ptr(), z.data_ptr(), S, codes.data_ptr()
    a.n_rays, a.n_samples = n, S
    a.grid = None
    a.packed = packed.data_ptr()
    a.want_scene, a.want_object, a.precision = 1, 1, L.PREC_BF16
    a.scene_out, a.obj_out, a.out_stride, a.ray_const = scene.data_ptr(), obj.data_ptr(), S, rc.data_ptr()
    a.train_ws = ws.data_ptr()
    L.check(L.load().onerf_field_fwd(L.ctx(torch.device(DEV)), C.byref(a), L.stream()))
    return scene, obj, ws


def test_plain_training_forward_dump_matches_fp32_activations():
    """The plain bf16 forward with a training dump: same fields as the inference forward; its one X atom, every layer's
    activation tiles and the sign masks against the fp32 kernel's activation dump."""
    from object_nerf_b200 import engine
    inp, model, rays, z, packed, codes = _plain_field_inputs(96)
    n, S = z.shape
    B = n * S
    T = helpers.train_layout(False, B)
    assert _lib().load().onerf_field_train_bytes(0, B) == T["total"]
    scene, obj, ws = _training_forward(rays, z, packed, codes, T)
    scene2, obj2 = engine.field(rays, z, packed, None, codes=codes, precision="bf16")
    torch.cuda.synchronize()
    assert torch.equal(scene, scene2) and torch.equal(obj, obj2)
    acts = [torch.empty(B, w, device=DEV) for w in WIDTHS]
    ptrs = (C.c_void_p * 17)(*[t.data_ptr() for t in acts])
    engine.field(rays, z, packed, None, codes=codes, precision="fp32", activations=ptrs)
    torch.cuda.synchronize()
    X = helpers.from_atoms(ws, T["act_off"][0], T["n_tiles"], 1)
    assert torch.equal(X[:, 63], torch.zeros_like(X[:, 63]))     # the padding column
    masks = helpers.read_masks(ws, T)
    for slot in range(17):
        got = helpers.from_atoms(ws, T["act_off"][slot], T["n_tiles"], T["act_atoms"][slot])[:B, :WIDTHS[slot]]
        want = acts[slot]
        tol = 2e-2 + 2e-2 * want.abs()
        bad = ((got - want).abs() > tol).float().mean().item()
        assert bad < 2e-3, (slot, bad, (got - want).abs().max().item())
    word0 = {**{s: (s - 1) * 8 for s in range(1, 9)}, 10: 64, **{s: 68 + (s - 11) * 4 for s in range(11, 15)}, 16: 84}
    for slot, w0 in word0.items():
        Wd = WIDTHS[slot]
        nbits = 16 if Wd == 64 else 32
        bits = torch.stack([(masks[:, w0 + w, :] >> j) & 1 for w in range(Wd // nbits) for j in range(nbits)], -1)
        bits = bits.reshape(-1, Wd)[:B]
        want = acts[slot] > 0
        clear = acts[slot].abs() > 2e-2
        agree = ((bits == 1) == want)[clear].float().mean().item()
        assert agree > 0.999, (slot, agree)


def _torch_chain(acts_bf, w, dA_s, dA_o):
    """fp32 reference of the input-gradient chain of the plain model from the dumped (bf16) activations."""
    lk = lambda h: torch.where(h > 0, 1.0, 0.01)
    W = {k: v[0].to(DEV) for k, v in w.items()}
    dz = {}
    dz["SDIR"] = (dA_s[:, :3] @ W["scene.rgb"]) * lk(acts_bf[10])
    dz["SFIN"] = dz["SDIR"] @ W["scene.dir"][:, :256]
    dz["S7"] = (dz["SFIN"] @ W["scene.final"] + dA_s[:, 3:4] * W["scene.sigma"]) * lk(acts_bf[8])
    for l in range(7, 0, -1):
        Wl = W[f"scene.l{l}"][:, XIN:] if l == 4 else W[f"scene.l{l}"]
        dz[f"S{l-1}"] = (dz[f"S{l}"] @ Wl) * lk(acts_bf[l])
    dz["ODIR"] = (dA_o[:, :3] @ W["obj.rgb"]) * lk(acts_bf[16])
    dz["OFIN"] = dz["ODIR"] @ W["obj.dir"][:, :128]
    dz["O3"] = (dz["OFIN"] @ W["obj.final"] + dA_o[:, 3:4] * W["obj.sigma"]) * lk(acts_bf[14])
    dz["O2"] = (dz["O3"] @ W["obj.l3"]) * lk(acts_bf[13])
    dz["O1"] = (dz["O2"] @ W["obj.l2"][:, OIN:]) * lk(acts_bf[12])
    dz["O0"] = (dz["O1"] @ W["obj.l1"]) * lk(acts_bf[11])
    return dz


def test_plain_bwd_chain_matches_torch_reference():
    """onerf_bwd_chain at the plain layout: the skip layers' hidden blocks start at kernel column 64 (S4, O2)."""
    L = _lib()
    inp, model, rays, z, packed, codes = _plain_field_inputs(70)   # 70 x 64 = 4480 samples = 35 tiles
    n, S = z.shape
    B = n * S
    T = helpers.train_layout(False, B)
    _, _, ws = _training_forward(rays, z, packed, codes, T)
    g = torch.Generator(device=DEV).manual_seed(1)
    dA_s = torch.randn(B, 4, device=DEV, generator=g)
    dA_o = torch.randn(B, 4, device=DEV, generator=g)
    L.check(L.load().onerf_bwd_chain(L.ctx(torch.device(DEV)), 0, 1, packed.data_ptr(), ws.data_ptr(), B, dA_s.data_ptr(),
                                     dA_o.data_ptr(), L.stream()))
    torch.cuda.synchronize()
    acts = [helpers.from_atoms(ws, T["act_off"][s], T["n_tiles"], T["act_atoms"][s])[:B, :WIDTHS[s]] for s in range(17)]
    want = _torch_chain(acts, inp["weights"]["coarse"], dA_s, dA_o)
    for d, gname in enumerate(GEMM_OF_DZ):
        got = helpers.from_atoms(ws, T["dz_off"][d], T["n_tiles"], T["dz_atoms"][d])[:B, :GEMM_N[gname]]
        ref = want[gname]
        scale = ref.abs().mean().item() + 1e-12
        err = (got - ref).abs()
        assert err.mean().item() <= 2e-2 * scale, (gname, err.mean().item(), scale)
        assert (err > 0.25 * scale + 0.05 * ref.abs()).float().mean().item() < 5e-3, (gname, err.max().item(), scale)


def test_plain_wgrad_and_unpack_match_torch_matmul():
    """onerf_bwd_wgrad at the plain layout (one X atom, 64 valid columns) on random bf16 operand tiles, and
    onerf_unpack_grads from the plain kernel layout to the reference shapes: column 63 of X (padding) is dropped, the
    hoisted code columns of object layers 0 / 2 are left to the per-ray sums."""
    from object_nerf_b200 import engine
    L = _lib()
    lib = L.load()
    ctx = L.ctx(torch.device(DEV))
    n_samples = 128 * 37
    T = helpers.train_layout(False, n_samples)
    ws = helpers.aligned_u8(T["total"], DEV, fill=0)
    g = torch.Generator(device=DEV).manual_seed(0)
    acts = [torch.randn(n_samples, 64 * a, device=DEV, generator=g) for a in T["act_atoms"]]
    dzs = [torch.randn(n_samples, 64 * a, device=DEV, generator=g) for a in T["dz_atoms"]]
    for i, m in enumerate(acts):
        helpers.write_atoms(ws, T["act_off"][i], m)
    for i, m in enumerate(dzs):
        helpers.write_atoms(ws, T["dz_off"][i], m)
    w_off, b_off, total = grad_layout()
    assert lib.onerf_grad_buffer_floats(0) == total
    grad = torch.zeros(total, device=DEV)
    L.check(lib.onerf_bwd_wgrad(ctx, 0, 1, ws.data_ptr(), n_samples, grad.data_ptr(), L.stream()))
    torch.cuda.synchronize()
    bf = lambda t: t.to(torch.bfloat16).float()
    X = bf(acts[0])
    inputs = {"S0": X, "S4": torch.cat([X, bf(acts[4])], 1), "O0": X, "O2": torch.cat([X, bf(acts[12])], 1),
              "SFIN": bf(acts[8]), "SDIR": bf(acts[9]), "O1": bf(acts[11]), "O3": bf(acts[13]), "OFIN": bf(acts[14]),
              "ODIR": bf(acts[15])}
    for l in (1, 2, 3, 5, 6, 7):
        inputs[f"S{l}"] = bf(acts[l])
    for d, gname in enumerate(GEMM_OF_DZ):
        dz = bf(dzs[d])[:, :GEMM_N[gname]]
        want = dz.t().double() @ inputs[gname].double()
        got = grad[w_off[gname]:w_off[gname] + GEMM_N[gname] * GEMM_K[gname]].view(GEMM_N[gname], GEMM_K[gname]).double()
        assert got.shape == want.shape, gname
        err = (got - want).abs().max().item()
        scale = want.abs().max().item()
        assert err <= 2e-3 * scale, (gname, err, scale)
        db_want = dz.double().sum(0)
        db_got = grad[b_off[gname]:b_off[gname] + GEMM_N[gname]].double()
        assert (db_got - db_want).abs().max().item() <= 2e-3 * db_want.abs().max().item(), gname
    # unpack into the reference's [out, in] tensors (zero-filled: onerf_unpack_grads accumulates)
    model = helpers.make_model(cases.build_render_case(cases.RENDER_CASES["eval_plain"])["weights"]["coarse"], False, DEV)
    lin = engine.model_linears(model)
    dW = [torch.zeros_like(w) for w, _ in lin]
    db = [torch.zeros_like(b) for _, b in lin]
    assert [tuple(dW[i].shape) for i in (0, 4, 12, 14)] == [(256, 63), (256, 319), (128, 127), (128, 255)]
    L.check(lib.onerf_unpack_grads(ctx, 0, grad.data_ptr(), (C.c_void_p * 20)(*[t.data_ptr() for t in dW]),
                                   (C.c_void_p * 20)(*[t.data_ptr() for t in db]), L.stream()))
    torch.cuda.synchronize()
    k = lambda gname: grad[w_off[gname]:w_off[gname] + GEMM_N[gname] * GEMM_K[gname]].view(GEMM_N[gname], GEMM_K[gname])
    kb = lambda gname: grad[b_off[gname]:b_off[gname] + GEMM_N[gname]]
    assert torch.equal(dW[0], k("S0")[:, :XIN]) and torch.equal(db[0], kb("S0"))
    assert torch.equal(dW[4], torch.cat([k("S4")[:, :XIN], k("S4")[:, 64:]], 1)) and torch.equal(db[4], kb("S4"))
    assert torch.equal(dW[12][:, :XIN], k("O0")[:, :XIN]) and (dW[12][:, XIN:] == 0).all()
    assert torch.equal(dW[14][:, :XIN], k("O2")[:, :XIN]) and (dW[14][:, XIN:OIN] == 0).all()
    assert torch.equal(dW[14][:, OIN:], k("O2")[:, 64:]) and torch.equal(db[14], kb("O2"))


def _train_step(precision, inp, c, rand):
    from object_nerf_b200 import Embedding, render_rays
    models = {k: helpers.make_model(w, False, DEV).train() for k, w in inp["weights"].items()}
    lib = helpers.CodeLib(inp["code_table"]).to(DEV)
    codes = lib.embedding_instance(inp["instance_ids"].view(-1).to(DEV))
    out = render_rays(models, {"xyz": Embedding(3, 10), "dir": Embedding(3, 4)}, inp["rays"].to(DEV),
                      N_samples=c["n_samples"], perturb=c["perturb"], noise_std=c["noise_std"],
                      N_importance=c["n_importance"], embedding_instance=codes, frustum_bound_th=c["frustum_bound_th"],
                      pass_through_mask=inp["pass_through_mask"].to(DEV), is_eval=False, precision=precision, _rand=rand)
    batch = {k: v.to(DEV) for k, v in inp["batch"].items()}
    loss = cases.total_loss(out, batch)
    loss.backward()
    named = [(f"{typ}.{k}", p) for typ, m in models.items() for k, p in m.named_parameters()]
    named += [("codes", lib.embedding_instance.weight)]
    return loss, named


def test_plain_training_backward_runs_in_the_forward_precision():
    """A bf16 training call on the plain model runs the tensor-core backward; fp32 runs the fp32 one.  Both reach
    onerf_render_rays_bwd with the forward's precision in the argument block: the tensor-core backward is a few dozen
    library launches, the fp32 one (FFMA forward re-run, then layer by layer) far more."""
    c = grad_plain.GRAD_CASE_PLAIN
    inp = grad_plain.build_grad_case_plain()
    rand = {k: v.to(DEV) for k, v in inp["rand"].items()}
    L = _lib()
    lib, dev = L.load(), torch.device(DEV)
    orig = lib.onerf_render_rays_bwd
    seen = []

    def spy(ctx, fwd, bwd, stream):
        n0 = L.launch_count(dev)
        rc = orig(ctx, fwd, bwd, stream)
        seen.append((fwd._obj.precision, L.launch_count(dev) - n0))
        return rc

    lib.onerf_render_rays_bwd = spy
    try:
        _train_step("bf16", inp, c, rand)
        _train_step("fp32", inp, c, rand)
    finally:
        lib.onerf_render_rays_bwd = orig
    assert [p for p, _ in seen] == [L.PREC_BF16, L.PREC_FP32], seen
    assert seen[0][1] < 64 < seen[1][1], seen


def test_plain_training_step_bf16_gradients_match_reference_golden(golden):
    """The plain model's step on the tensor cores against the REFERENCE's own backward (fixture): loss within 2 %,
    per-tensor norm within 5 %, direction (cosine against the fp32 path) >= 0.995 for the 80 MLP tensors and the codes."""
    g = golden("grad_train_step_plain")
    c = grad_plain.GRAD_CASE_PLAIN
    inp = grad_plain.build_grad_case_plain()
    rand = {k: v.to(DEV) for k, v in inp["rand"].items()}
    loss, named = _train_step("bf16", inp, c, rand)
    assert abs(loss.item() - g["loss"].item()) <= 2e-2 * abs(g["loss"].item()), (loss.item(), g["loss"].item())
    loss32, named32 = _train_step("fp32", inp, c, rand)
    assert len(named) == 81
    report = []
    for (name, p), (_, p32) in zip(named, named32):
        assert p.grad is not None, name
        gr, g32 = p.grad.detach().reshape(-1).double(), p32.grad.detach().reshape(-1).double()
        ref_norm = g[name + "|norm"].item()
        cos = (gr @ g32 / (gr.norm() * g32.norm() + 1e-30)).item()
        report.append((name, gr.norm().item() / max(ref_norm, 1e-12), cos))
    print("plain bf16 step vs reference: loss", loss.item(), "ref", g["loss"].item())
    for r in report:
        print(f"  {r[0]:40s} norm ratio {r[1]:.4f}  cos {r[2]:.5f}")
    bad = [r for r in report if not (0.95 <= r[1] <= 1.05 and r[2] >= 0.995)]
    assert not bad, bad


def _oracle_grads_fp64(c):
    """The reference's step restated by the CPU oracle in float64: the fixture's entries without fp32 rounding."""
    from oracle import onerf_oracle as O
    inp = grad_plain.build_grad_case_plain()
    f64 = lambda t: t.double() if t is not None and t.is_floating_point() else t
    leaves = {}

    def leaf(name, t):
        leaves[name] = t.double().clone().requires_grad_(True)
        return leaves[name]

    weights = {typ: {k: (leaf(f"{typ}.{helpers.REF_NAMES[k]}.weight", W), leaf(f"{typ}.{helpers.REF_NAMES[k]}.bias", b))
                     for k, (W, b) in w.items()} for typ, w in inp["weights"].items()}
    codes = leaf("codes", inp["code_table"])[inp["instance_ids"].view(-1)]
    out = O.render_rays(weights, None, inp["rays"].double(), codes, n_samples=c["n_samples"], perturb=c["perturb"],
                        noise_std=c["noise_std"], n_importance=c["n_importance"], frustum_bound_th=c["frustum_bound_th"],
                        pass_through_mask=inp["pass_through_mask"], is_eval=False,
                        rand={k: f64(v) for k, v in inp["rand"].items()})
    cases.total_loss(out, {k: f64(v) for k, v in inp["batch"].items()}).backward()
    return {k: t.grad.reshape(-1) for k, t in leaves.items()}


def test_plain_training_step_fp32_gradients_match_reference_golden(golden):
    """The fp32 path (precision="fp32") on the plain model against the reference's backward, with the fp32 tolerances
    of the voxel model's fixture test: loss 2e-4, per-tensor norm 2e-3, sampled entries within 1 % of the tensor's RMS
    entry.  The plain model's deep-layer gradients are sensitive enough that the fixture's own fp32 rounding moves some
    entries by more than that 1 % (the float64 restatement differs from the fixture by up to ~6 % of the RMS on this
    case).  Such entries cannot decide the gate either way and are reported, not asserted; every other entry is."""
    g = golden("grad_train_step_plain")
    c = grad_plain.GRAD_CASE_PLAIN
    inp = grad_plain.build_grad_case_plain()
    rand = {k: v.to(DEV) for k, v in inp["rand"].items()}
    loss, named = _train_step("fp32", inp, c, rand)
    assert abs(loss.item() - g["loss"].item()) <= 2e-4 * abs(g["loss"].item()), (loss.item(), g["loss"].item())
    exact = _oracle_grads_fp64(c)
    undecidable, checked = [], 0
    for name, p in named:
        assert p.grad is not None, name
        gr = p.grad.detach().cpu().reshape(-1)
        ref_norm = g[name + "|norm"].item()
        assert abs(gr.norm().item() - ref_norm) <= 2e-3 * max(ref_norm, 1e-7), (name, gr.norm().item(), ref_norm)
        idx = cases.sample_indices(name, gr.numel())
        rms = max(ref_norm, 1e-7) / max(1.0, gr.numel() ** 0.5)
        gate = 1e-2 * rms + 1e-8
        ref = g[name + "|samples"]
        noise = (exact[name][idx] - ref.double()).abs()       # the fixture's own fp32 rounding
        decidable = noise <= gate
        err = (gr[idx] - ref).abs()
        assert (err[decidable] <= gate).all(), (name, err[decidable].max().item(), rms)
        checked += int(decidable.sum())
        if not decidable.all():
            undecidable.append((name, int((~decidable).sum()), round(noise.max().item() / rms, 4),
                                round(err[~decidable].max().item() / rms, 4)))
    print("plain fp32 step: entries checked", checked, "; (tensor, entries, fixture noise / rms, our error / rms) "
          "not decidable at 1 % of rms:", undecidable)
    assert checked >= 0.95 * sum(min(cases.GRAD_SAMPLES, p.numel()) for _, p in named)


@pytest.mark.parametrize("n_rays", [2048])
def test_plain_training_step_bf16_vs_fp32_at_batch_size(n_rays):
    """2048 rays (config/default_conf.yml:40) on the plain model: tensor-core gradients against the fp32 path."""
    c = dict(grad_plain.GRAD_CASE_PLAIN, n_rays=n_rays)
    inp = grad_plain.build_grad_case_plain(n_rays=n_rays)
    rand = {k: v.to(DEV) for k, v in inp["rand"].items()}
    loss, named = _train_step("bf16", inp, c, rand)
    loss32, named32 = _train_step("fp32", inp, c, rand)
    assert abs(loss.item() - loss32.item()) <= 2e-2 * abs(loss32.item())
    bad = []
    for (name, p), (_, p32) in zip(named, named32):
        gr, g32 = p.grad.detach().reshape(-1).double(), p32.grad.detach().reshape(-1).double()
        ratio = (gr.norm() / (g32.norm() + 1e-30)).item()
        cos = (gr @ g32 / (gr.norm() * g32.norm() + 1e-30)).item()
        if not (0.95 <= ratio <= 1.05 and cos >= 0.995):
            bad.append((name, ratio, cos))
    assert not bad, bad


def test_plain_backward_rejects_a_table_gradient():
    """onerf_render_rays_bwd on the plain model (grid NULL) with a table_grad buffer: ONERF_ERR_BAD_ARG and a message,
    before any kernel runs."""
    L = _lib()
    lib = L.load()
    n, ns, ni = 4, 64, 0
    buf = torch.zeros(1 << 16, device=DEV)
    tws = helpers.aligned_u8(lib.onerf_train_workspace_bytes(0, n, ns, ni), DEV, fill=0)
    a = L.RenderArgs()
    a.rays, a.n_rays, a.n_samples, a.n_importance = buf.data_ptr(), n, ns, ni
    a.grid = None
    a.packed_coarse = buf.data_ptr()
    a.precision = L.PREC_BF16
    a.train_ws, a.train_ws_bytes = tws.data_ptr(), tws.numel()
    ptrs = (C.c_void_p * 20)(*([buf.data_ptr()] * 20))
    b = L.RenderBwdArgs()
    b.W_coarse, b.dW_coarse, b.db_coarse = ptrs, ptrs, ptrs
    b.table_grad = buf.data_ptr()
    rc = lib.onerf_render_rays_bwd(L.ctx(torch.device(DEV)), C.byref(a), C.byref(b), L.stream())
    assert rc == -1, rc      # ONERF_ERR_BAD_ARG
    assert b"table_grad" in lib.onerf_last_error()
    torch.cuda.synchronize()
    assert (buf == 0).all()
