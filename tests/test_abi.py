"""CPU test: libc3d.so loads and exports every symbol include/c3d.h declares (no compute calls)."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    names = set()
    for f in os.listdir(os.path.join(ROOT, "include")):
        if f.endswith(".h"):
            src = open(os.path.join(ROOT, "include", f)).read()
            src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
            names |= set(re.findall(r"\b(c3d_[a-z0-9_]+)\s*\(", src))
    return sorted(names)


def test_library_exports_every_declared_symbol():
    from omni3d_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    L = ctypes.CDLL(_lib.LIB_PATH)
    decl = _declared()
    assert len(decl) >= 6
    for name in decl:
        assert hasattr(L, name), f"{name} declared in include/*.h but not exported"
    assert sorted(_lib.EXPORTS) == decl, "omni3d_b200/_lib.py EXPORTS out of sync with include/c3d.h"
    L.c3d_abi_version.restype = ctypes.c_int32
    assert L.c3d_abi_version() >= 1


def test_product_fails_loudly_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from omni3d_b200 import box3d, _lib
    with pytest.raises(_lib.C3DError):
        box3d.box3d_overlap(torch.zeros(1, 8, 3), torch.zeros(1, 8, 3))


def test_product_never_imports_oracle():
    bad = []
    for dp, _, fs in os.walk(os.path.join(ROOT, "omni3d_b200")):
        for f in fs:
            if f.endswith((".py", ".cu", ".cuh", ".cpp", ".h")):
                s = open(os.path.join(dp, f), errors="ignore").read()
                if re.search(r"^\s*(from|import)\s+oracle\b|#include\s+\".*oracle", s, flags=re.M):
                    bad.append(f)
    assert not bad, bad


def test_host_side_entry_points_without_gpu():
    """entry points that do host arithmetic or argument checking only: tile query (incl. the rolling-halo path's
    one-row-per-CTA statistics layout), workspace sizes, EINVAL + c3d_last_error on bad arguments (no CUDA call)."""
    from omni3d_b200 import _lib, conv
    L = conv._bind()
    d = conv.ConvDesc(32, 640, 640, 16, 16, 3, 3, 1, 1, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0)       # DLA level0: halo path
    t, th, tw = conv.num_tiles(d)
    if os.environ.get("C3D_CONV_NO_HALO"):
        assert t == 32 * 640 * 640 // (th * tw)
    else:
        assert (t, th, tw) == (132 * 3, 1, 128)
    d = conv.ConvDesc(32, 160, 160, 256, 256, 3, 3, 1, 1, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0)     # FPN output conv
    t, th, tw = conv.num_tiles(d)
    assert th * tw <= 128 and t == 32 * -(-160 // th) * -(-160 // tw)
    L.c3d_nms_workspace_bytes.restype = ctypes.c_size_t
    L.c3d_nms_workspace_bytes.argtypes = [ctypes.c_int32, ctypes.c_int32]
    assert L.c3d_nms_workspace_bytes(32, 8192) > L.c3d_nms_workspace_bytes(32, 4096) > 32 * 4096 * 64 * 8
    L.c3d_anchor_match.restype = ctypes.c_int32
    L.c3d_last_error.restype = ctypes.c_char_p
    null = ctypes.c_void_p(None)
    L.c3d_anchor_match.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                   ctypes.c_int32, ctypes.c_int32, ctypes.c_float] + [ctypes.c_void_p] * 7
    rc = L.c3d_anchor_match(null, 10, null, null, null, 1, 1, 0.7, null, null, null, null, null, null, null)
    assert rc != 0 and b"anchor_match" in L.c3d_last_error()
    with pytest.raises(_lib.C3DError):
        _lib.check(rc)


def test_conv_descriptor_argument_checks_without_gpu():
    """c3d_conv2d_fwd validates the descriptor before any CUDA call: odd outputs have no nearest-x2 addend, the in-place
    accumulate needs a bf16 output, the split channel placement needs a multiple of 16 and excludes addend / statistics."""
    from omni3d_b200 import _lib, conv
    L = conv._bind()
    L.c3d_last_error.restype = ctypes.c_char_p
    p = ctypes.c_void_p(256)                       # non-null dummies: every case below is rejected before they are used

    def call(d, addend=p, stats=None):
        return L.c3d_conv2d_fwd(ctypes.byref(d), p, p, None, addend, p, stats, None)

    d = conv.ConvDesc(2, 9, 11, 64, 64, 3, 3, 1, 1, 0, 0, 2, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0)           # up2 addend, 9 x 11 output
    assert call(d) == _lib.C3D_EINVAL and b"even output" in L.c3d_last_error()
    d = conv.ConvDesc(2, 8, 8, 64, 64, 3, 3, 1, 1, 0, 0, 1, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0)             # addend mode without addend
    assert call(d, addend=None) == _lib.C3D_EINVAL and b"addend missing" in L.c3d_last_error()
    d = conv.ConvDesc(2, 8, 8, 64, 64, 3, 3, 1, 1, 0, 1, 3, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0)             # accumulate into fp32
    assert call(d) == _lib.C3D_EINVAL and b"bf16 output" in L.c3d_last_error()
    d = conv.ConvDesc(2, 8, 8, 64, 64, 2, 2, 1, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 8, 8, 0, 24, 0, 100)           # split not a multiple of 16
    assert call(d, addend=None) == _lib.C3D_EINVAL and b"y_split_c" in L.c3d_last_error()
    d = conv.ConvDesc(2, 8, 8, 64, 64, 3, 3, 3, 1, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0)             # stride 3
    assert call(d, addend=None) == _lib.C3D_EINVAL and b"stride" in L.c3d_last_error()
    with pytest.raises(_lib.C3DError):
        _lib.check(_lib.C3D_EINVAL)
