"""CPU checks of the many-object editing entries: the exports of include/onerf_ext.h, their argument checks without a
device, and the workspace arithmetic of the rank-merge sort and the box culling."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from object_nerf_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        _lib.build()
    return _lib.load()


def test_ext_header_matches_the_exports(lib):
    from object_nerf_b200 import _lib
    src = open(os.path.join(ROOT, "include", "onerf_ext.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    names = sorted(set(re.findall(r"\b(onerf_[a-z0-9_]+)\s*\(", src)))
    assert names == sorted(_lib.EXPORTS_EXT)
    assert not set(names) & set(_lib.EXPORTS)
    for n in names:
        assert hasattr(lib, n), n


def test_new_entries_reject_a_null_context(lib):
    z = ctypes.c_void_p(0)
    for name in ("onerf_composite_multi_ws", "onerf_composite_multi_merge"):
        rc = getattr(lib, name)(None, z, z, 4, 30, 192, 0, z, z, z, z, z, z, z, z, 0, z)
        assert rc == -1, name
        assert b"null" in lib.onerf_last_error()


def test_composite_workspace_bytes(lib):
    f = lib.onerf_composite_multi_workspace_bytes
    assert f(-1, 2, 8) == 0 and f(4, 0, 8) == 0 and f(4, 2, 0) == 0
    assert f(0, 3, 64) == 0
    for n, no, s in ((1, 1, 2), (37, 3, 64), (4096, 25, 192), (4096, 41, 128)):
        t = n * no * s
        # 4-byte sorted key and 2-byte in-set index per sample, the keys padded to 256 bytes
        assert f(n, no, s) == ((t * 4 + 255) // 256) * 256 + t * 2


def test_render_multi_workspace_grows_by_the_culling_and_sort_scratch(lib):
    a256 = lambda x: (x + 255) // 256 * 256
    for n, no, s, si in ((40, 3, 64, 64), (4096, 3, 64, 64), (4096, 25, 64, 128), (77, 2, 32, 0)):
        sf = s + si
        old = (a256(n * 448 * 4) + a256(no * n * s * 4) + a256(no * n * sf * 4) + a256(no * n * sf * 16) +
               a256(no * n * s * 4))
        cull = a256(n * 4) * 2 + a256(4) + a256(n * 32) + a256(n * sf * 4) + a256(n * sf * 16)
        sort = a256(lib.onerf_composite_multi_workspace_bytes(n, no, sf))
        assert lib.onerf_render_multi_workspace_bytes(n, no, s, si) == old + cull + sort
    # 41 ray sets at 64 + 128 samples: refused before (T > 4096), sized now
    assert lib.onerf_render_multi_workspace_bytes(4096, 41, 64, 128) > 0
