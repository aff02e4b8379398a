"""object_nerf_b200 — H100-native (sm_90a) per-ray render path of zju3dv/object_nerf behind the
reference's own call surface.  See DESIGN.md and INTEGRATION.md."""
from .rendering import render_rays, inference_model, query_sigma  # noqa: F401
from .nerf_model import ObjectNeRF  # noqa: F401
from .embedding_helper import Embedding, EmbeddingVoxel  # noqa: F401
from .code_library import CodeLibrary  # noqa: F401
from .batches import RaySampler  # noqa: F401
from .frames import FrameSet  # noqa: F401
