"""CPU checks of the Python binding's shared pieces: every module reaches the library through _lib.call (the device
guard, the context first and the stream last, a failed status raised), engine alone builds the 20-entry pointer tables
and aligns blobs to 1024 bytes, and those helpers, the gradient buffer and pack_weights(out=...) behave as documented
on CPU tensors."""
import contextlib
import glob
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PACKAGE = os.path.join(ROOT, "object_nerf_b200")


def _modules():
    return {os.path.basename(p): open(p).read() for p in sorted(glob.glob(os.path.join(PACKAGE, "*.py")))}


def test_only_the_binding_takes_contexts_and_streams():
    bad = [(name, m) for name, src in _modules().items() if name != "_lib.py"
           for m in re.findall(r"_lib\.(?:ctx|stream|check)\(", src)]
    assert not bad, bad


def test_only_engine_aligns_blobs_and_builds_pointer_tables():
    mods = _modules()
    assert [name for name, src in mods.items() if "% 1024" in src] == ["engine.py"]
    table = re.compile(r"c_void_p\s*\*\s*(?:20|(?:_lib\.)?N_LINEAR)\b")
    assert [name for name, src in mods.items() if table.search(src)] == ["engine.py"]


def test_pointer_tables_hold_the_tensors_addresses_in_order():
    from object_nerf_b200 import engine
    pairs = [(torch.randn(i + 2, 3), torch.randn(i + 2)) for i in range(20)]
    first, second = engine.pointer_tables(pairs)
    assert list(first) == [w.data_ptr() for w, _ in pairs] and list(second) == [b.data_ptr() for _, b in pairs]


def test_gradient_buffer_views_are_zeroed_disjoint_16_byte_aligned_and_shaped_like_the_tensors():
    from object_nerf_b200 import engine
    tensors = [torch.empty(256, 63), torch.empty(1), torch.empty(3, 128), torch.empty(3), torch.empty(7, 5)]
    flat, views, offsets = engine.grad_buffer(tensors, "cpu")
    assert flat.dtype == torch.float32 and not flat.any()
    assert [v.shape for v in views] == [t.shape for t in tensors]
    assert [v.data_ptr() - flat.data_ptr() for v in views] == [4 * o for o in offsets]
    assert all(o % 4 == 0 for o in offsets) and offsets[0] == 0
    ends = [o + t.numel() for o, t in zip(offsets, tensors)]
    assert all(e <= o for e, o in zip(ends, offsets[1:])) and ends[-1] <= flat.numel()
    for i, v in enumerate(views):
        v.fill_(i + 1)
    assert [v.unique().tolist() for v in views] == [[i + 1] for i in range(len(views))]


@pytest.mark.parametrize("nbytes", [1, 1000, 1024, 5 * 1024 * 1024 + 3])
def test_aligned_bytes_start_on_a_1024_byte_boundary_and_hold_what_was_asked(nbytes):
    from object_nerf_b200 import engine
    t = engine.aligned_bytes(nbytes, "cpu")
    assert t.dtype == torch.uint8 and t.numel() == nbytes and t.is_contiguous() and t.data_ptr() % 1024 == 0


class _Recorder:
    def __init__(self, rc=0):
        self.rc, self.calls = rc, []

    def onerf_pack_weights(self, *args):
        self.calls.append(("onerf_pack_weights", args))
        return self.rc

    def onerf_last_error(self):
        return b"bad argument"


@pytest.fixture
def stubbed(monkeypatch):
    from object_nerf_b200 import _lib
    fake, guards = _Recorder(), []

    @contextlib.contextmanager
    def device(dev):
        guards.append(dev)
        yield

    monkeypatch.setattr(_lib, "load", lambda: fake)
    monkeypatch.setattr(_lib, "ctx", lambda dev: ("ctx", dev))
    monkeypatch.setattr(_lib, "stream", lambda: "stream")
    monkeypatch.setattr(torch.cuda, "device", device)
    return fake, guards


def test_call_passes_context_first_and_stream_last_under_the_device_guard_and_raises_on_failure(stubbed):
    from object_nerf_b200 import _lib
    fake, guards = stubbed
    dev = torch.device("cpu")
    assert _lib.call("onerf_pack_weights", dev, 1, 2) is None
    assert fake.calls == [("onerf_pack_weights", (("ctx", dev), 1, 2, "stream"))] and guards == [dev]
    fake.rc = -1
    with pytest.raises(RuntimeError, match="bad argument"):
        _lib.call("onerf_pack_weights", dev)


def test_pack_weights_fills_the_given_blob(stubbed):
    from object_nerf_b200 import engine
    fake, _ = stubbed
    lin = [(torch.randn(4, 3), torch.randn(4)) for _ in range(20)]
    blob = engine.aligned_bytes(4096, "cpu")
    assert engine.pack_weights(lin, True, out=blob) is blob
    ((name, (ctx, use_voxel, W, B, packed, nbytes, stream)),) = fake.calls
    assert (use_voxel, packed, nbytes) == (1, blob.data_ptr(), 4096)
    assert list(W) == [w.data_ptr() for w, _ in lin] and list(B) == [b.data_ptr() for _, b in lin]


def test_training_precision_rule():
    from object_nerf_b200 import engine
    assert [engine.train_precision(p) for p in ("bf16", "fp32", "tf32")] == ["bf16", "fp32", "fp32"]
    assert engine.train_precision(None) == ("bf16" if engine.default_precision() == "bf16" else "fp32")
