"""Host-side rules of the differentiable field queries: which calls are refused before any kernel runs, and which
Linear tensors each query's gradient reaches (the reference's graph, models/nerf_model.py:97-152)."""
import pytest
import torch

from object_nerf_b200 import Embedding, engine, field_query, synthetic as S


def _model():
    return S.make_model(S.make_weights(1, False), False, "cpu").train()


def _tagged(x, module):
    t = torch.zeros(x.shape[0], module.out_channels)
    t._onerf_src = (x, module)
    return t


def test_untagged_inputs_are_refused():
    with pytest.raises(NotImplementedError):
        _model().forward({"emb_xyz": torch.zeros(4, 63), "emb_dir": torch.zeros(4, 27)})
    with pytest.raises(NotImplementedError):
        _model().forward_instance({"emb_xyz": torch.zeros(4, 63), "obj_code": torch.zeros(4, 64)}, sigma_only=True)


def test_missing_direction_embedding_is_a_value_error():
    pts = torch.zeros(4, 3)
    with pytest.raises(ValueError, match="emb_dir"):
        _model().forward({"emb_xyz": _tagged(pts, Embedding(3, 10))})


def test_direction_embedding_must_be_pe4():
    pts = torch.zeros(4, 3)
    with pytest.raises(NotImplementedError):
        _model().forward({"emb_xyz": _tagged(pts, Embedding(3, 10)), "emb_dir": _tagged(pts, Embedding(3, 10))})


def test_positions_or_directions_that_require_grad_are_refused():
    pts = torch.zeros(4, 3, requires_grad=True)
    d = torch.zeros(4, 3)
    with pytest.raises(ValueError, match="no gradient"):
        _model().forward({"emb_xyz": _tagged(pts, Embedding(3, 10)), "emb_dir": _tagged(d, Embedding(3, 4))})
    with pytest.raises(ValueError, match="no gradient"):
        _model().forward({"emb_xyz": _tagged(d, Embedding(3, 10)),
                          "emb_dir": _tagged(d.clone().requires_grad_(True), Embedding(3, 4))})


def test_unsupported_positional_encodings_raise():
    for c, f in ((3, 6), (2, 4), (3, 5)):
        with pytest.raises(NotImplementedError):
            Embedding(c, f)(torch.zeros(4, c))
    with pytest.raises(NotImplementedError):   # CPU tensors: the encoding is a CUDA kernel
        Embedding(3, 4)(torch.zeros(4, 3))


def test_object_code_shape_is_checked():
    pts = torch.zeros(4, 3)
    with pytest.raises(ValueError, match="obj_code"):
        _model().forward_instance({"emb_xyz": _tagged(pts, Embedding(3, 10)), "emb_dir": _tagged(pts, Embedding(3, 4)),
                                   "obj_code": torch.zeros(3, 64)})


def test_reached_tensors_follow_the_reference_graph():
    """forward never touches instance_* (their gradient stays None, not zero), sigma_only stops at the sigma head."""
    names = [a.split(".")[0] for a in engine.LINEAR_ATTRS]
    assert [names[i] for i in field_query.SCENE] == [f"xyz_encoding_{i}" for i in range(1, 9)] + [
        "sigma", "xyz_encoding_final", "dir_encoding", "rgb"]
    assert [names[i] for i in field_query.SCENE_SIGMA] == [f"xyz_encoding_{i}" for i in range(1, 9)] + ["sigma"]
    assert [names[i] for i in field_query.OBJECT] == [f"instance_encoding_{i}" for i in range(1, 5)] + [
        "instance_sigma", "instance_encoding_final", "inst_dir_encoding", "inst_rgb"]
    assert [names[i] for i in field_query.OBJECT_SIGMA] == [f"instance_encoding_{i}" for i in range(1, 5)] + [
        "instance_sigma"]


class _FakeArgs:
    precision, grid, n_rays, n_samples = 0, None, 0, 1


def _stub_engine(monkeypatch, calls):
    """engine with the library calls replaced: the field writes zeros, the backward returns ones for every tensor"""
    monkeypatch.setattr(field_query._lib, "load", lambda: None)
    monkeypatch.setattr(field_query.engine, "packed_for", lambda *a, **k: None)

    def field(rays, z, packed, grid, codes=None, want_object=True, scene_out=None, obj_out=None, _args_out=None, **k):
        scene_out.zero_()
        if obj_out is not None:
            obj_out.zero_()
        _args_out += [_FakeArgs(), ()]
        return scene_out, obj_out

    def field_bwd(args, d_scene, d_obj, linears, grads=None, d_codes=None, table_grad=None, workspace=None):
        calls.append((d_scene is not None, d_obj is not None))
        if d_codes is not None:
            d_codes += 1
        return [(torch.ones_like(w), torch.ones_like(b)) for w, b in linears]

    monkeypatch.setattr(field_query.engine, "field", field)
    monkeypatch.setattr(field_query.engine, "field_bwd", field_bwd)
    monkeypatch.setattr(field_query.engine, "field_bwd_workspace_bytes", lambda *a: 0)
    monkeypatch.setattr(field_query.engine, "aligned_bytes", lambda *a: None)


@pytest.mark.parametrize("fi,sigma_only", [(False, False), (False, True), (True, False), (True, True)])
def test_unreached_tensors_get_none_not_zero(monkeypatch, fi, sigma_only):
    """FieldEvalFn.backward hands autograd None for every Linear tensor outside the evaluated branch (and, with sigma_only,
    after the sigma head), a gradient for the others, and a code gradient only with the object branch."""
    calls = []
    _stub_engine(monkeypatch, calls)
    model = _model()
    n = 5
    codes = torch.zeros(n, 64, requires_grad=True)
    reached = (field_query.OBJECT_SIGMA if sigma_only else field_query.OBJECT) if fi else (
        field_query.SCENE_SIGMA if sigma_only else field_query.SCENE)
    scene, obj = field_query.field_eval(model, None, torch.zeros(n, 8), torch.zeros(n, 1), torch.zeros(n, 1, 3),
                                        codes if fi else None, fi, "fp32", reached)
    out = obj if fi else scene
    (out[..., 3:] if sigma_only else out).sum().backward()
    assert calls == [(not fi, fi)]
    names = [a for a in engine.LINEAR_ATTRS]
    for i, attr in enumerate(names):
        mod = model
        for part in attr.split("."):
            mod = mod[int(part)] if part.isdigit() else getattr(mod, part)
        for p in (mod.weight, mod.bias):
            if i in reached:
                assert p.grad is not None and torch.equal(p.grad, torch.ones_like(p)), attr
            else:
                assert p.grad is None, attr
    assert (codes.grad is not None) == fi


def test_empty_batch_backward_gives_zero_gradients(monkeypatch):
    calls = []
    _stub_engine(monkeypatch, calls)
    model = _model()
    scene, _ = field_query.field_eval(model, None, torch.zeros(0, 8), torch.zeros(0, 1), torch.zeros(0, 1, 3), None,
                                      False, "fp32", field_query.SCENE)
    scene.sum().backward()
    assert calls == []
    assert torch.equal(model.sigma.weight.grad, torch.zeros_like(model.sigma.weight))


def test_positions_requiring_grad_are_refused_with_a_frozen_model():
    model = _model().requires_grad_(False)
    pts = torch.zeros(4, 3, requires_grad=True)
    with pytest.raises(ValueError, match="no gradient"):
        model.forward({"emb_xyz": _tagged(pts, Embedding(3, 10))}, sigma_only=True)
