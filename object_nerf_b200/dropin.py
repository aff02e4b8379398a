"""Make the reference's own entry scripts import this package's hot path.

    import object_nerf_b200.dropin as dropin
    dropin.install()            # before `import train` / `from render_tools.editable_renderer import ...`

After install(), these module names resolve to the H100 implementations (same public names, signatures and
result keys as the reference files they shadow):

    models.rendering              -> object_nerf_b200.rendering         (render_rays, sample_pdf, inference_model)
    models.nerf_model             -> object_nerf_b200.nerf_model        (ObjectNeRF)
    models.embedding_helper       -> object_nerf_b200.embedding_helper  (Embedding, EmbeddingVoxel)
    models.code_library           -> object_nerf_b200.code_library      (CodeLibrary)
    render_tools.multi_rendering  -> object_nerf_b200.multi_rendering   (render_rays_multi)
    models.losses                 -> object_nerf_b200.losses            (TotalLoss, get_loss: fused loss + gradient)

Every other reference module (train.py, render_tools/editable_renderer.py, datasets/, utils/)
is imported from the reference checkout as is: their `from models.rendering import render_rays` etc. bind to
the modules above because Python consults sys.modules before the file system.
"""
import importlib
import sys
import types

ALIASES = {
    "models.rendering": "object_nerf_b200.rendering",
    "models.nerf_model": "object_nerf_b200.nerf_model",
    "models.embedding_helper": "object_nerf_b200.embedding_helper",
    "models.code_library": "object_nerf_b200.code_library",
    "render_tools.multi_rendering": "object_nerf_b200.multi_rendering",
    "models.losses": "object_nerf_b200.losses",
}


def install(reference_root=None):
    """Alias the hot-path modules.  reference_root (optional) is put on sys.path so that the remaining
    reference packages (`utils`, `datasets`, `render_tools.editable_renderer`) import."""
    if reference_root and reference_root not in sys.path:
        sys.path.insert(0, reference_root)
    for pkg in ("models", "render_tools"):
        if pkg not in sys.modules:
            try:
                importlib.import_module(pkg)          # the reference's package, if importable
            except Exception:
                m = types.ModuleType(pkg)
                m.__path__ = []
                sys.modules[pkg] = m
    for alias, target in ALIASES.items():
        mod = importlib.import_module(target)
        sys.modules[alias] = mod
        parent, _, leaf = alias.rpartition(".")
        setattr(sys.modules[parent], leaf, mod)
    return ALIASES
