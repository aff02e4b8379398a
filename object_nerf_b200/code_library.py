"""Per-object latent codes (reference models/code_library.py:5-28): an embedding table looked up by instance id.
On a CUDA device the lookup and its gradient (scatter-add of the per-ray code gradients into the table) are kernels of
libonerf_sm90.so (`onerf_code_gather` / `onerf_code_scatter_add`); the parameter keeps the reference's name
(`embedding_instance.weight`), so checkpoints and optimizers are interchangeable.  An id outside [0, n_codes) reads the
nearest row (0 or n_codes - 1), and its gradient goes to that same row."""
import torch
from torch import nn

from . import _lib


class _CodeLookup(torch.autograd.Function):
    @staticmethod
    def forward(ctx, table, ids):
        dev = table.device
        ids = ids.reshape(-1).to(torch.int64).contiguous()
        t = table.detach().contiguous().float()
        out = torch.empty(ids.numel(), t.shape[1], dtype=torch.float32, device=dev)
        _lib.call("onerf_code_gather", dev, t.data_ptr(), ids.data_ptr(), ids.numel(), t.shape[0], out.data_ptr())
        ctx.save_for_backward(ids)
        ctx.shape = tuple(t.shape)
        return out

    @staticmethod
    def backward(ctx, g):
        (ids,) = ctx.saved_tensors
        g = g.contiguous().float()
        grad = torch.zeros(ctx.shape, dtype=torch.float32, device=g.device)
        _lib.call("onerf_code_scatter_add", g.device, g.data_ptr(), ids.data_ptr(), ids.numel(), ctx.shape[0],
                  grad.data_ptr())
        return grad, None


class CodeLibrary(nn.Module):
    def __init__(self, model_config):
        super().__init__()
        get = model_config.get if hasattr(model_config, "get") else (lambda k, d: getattr(model_config, k, d))
        self.embedding_instance = nn.Embedding(get("N_max_objs", 64), get("N_obj_code_length", 64))

    def lookup(self, instance_ids: torch.Tensor) -> torch.Tensor:
        """(N,) or (N,1) int64 ids -> (N,64) codes."""
        w = self.embedding_instance.weight
        if w.shape[1] != 64:
            raise RuntimeError("object_nerf_b200 kernels are built for 64-long object codes")
        return _CodeLookup.apply(w, instance_ids)

    def forward(self, inputs):
        out = {}
        if "instance_ids" in inputs:
            out["embedding_instance"] = self.lookup(inputs["instance_ids"])
        return out
