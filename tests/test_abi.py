"""CPU tests of the C ABI: include/c3d.h against libc3d.so and the ctypes declarations of omni3d_b200/_lib.py (prototypes,
struct layouts), plus the entry points that only do host arithmetic or argument checking (no compute calls)."""
import ctypes
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "c3d.h")

# by-value C types of the ABI and the ctypes type each must be bound as
_SCALARS = {"int32_t": ctypes.c_int32, "int64_t": ctypes.c_int64, "size_t": ctypes.c_size_t, "float": ctypes.c_float,
            "double": ctypes.c_double}


def _header_source():
    src = open(HEADER).read()
    src = re.sub(r"/\*.*?\*/", " ", src, flags=re.S)
    src = re.sub(r"//[^\n]*", " ", src)
    return re.sub(r"^\s*#[^\n]*", " ", src, flags=re.M)


def _c_type(decl, named=False):
    """'const float* boxes' -> ('float', 1); named: the declaration ends in a parameter name."""
    toks = [t for t in re.findall(r"\w+|\*", decl) if t != "const"]
    if named:
        assert len(toks) >= 2 and toks[-1] != "*", f"unnamed parameter {decl!r}"
        toks = toks[:-1]
    assert toks and toks[0] != "*" and all(t == "*" for t in toks[1:]), f"unparsed type {decl!r}"
    return toks[0], len(toks) - 1


def _prototypes():
    """{name: (return type, [parameter types])} of every c3d_* function c3d.h declares."""
    src = _header_source()
    protos = {}
    for stmt in re.split(r"[;{}]", src):
        m = re.fullmatch(r"\s*([\w\s*]+?)\s*\b(c3d_\w+)\s*\(([^()]*)\)\s*", stmt)
        if m:
            ret, name, params = m.groups()
            params = [] if params.strip() == "void" else [_c_type(p, named=True) for p in params.split(",")]
            protos[name] = (_c_type(ret), params)
    # a declaration this parser missed would drop out of every check below
    assert set(protos) == set(re.findall(r"\b(c3d_\w+)\s*\(", src)), "c3d.h declaration the prototype parser missed"
    return protos


def _expected_ctype(base, depth):
    from omni3d_b200 import _lib
    if depth == 0:
        assert base in _SCALARS, f"by-value {base} has no ctypes mapping"
        return _SCALARS[base]
    if base == "char":
        return ctypes.c_char_p
    if base in _lib.STRUCTS:
        assert depth == 1, f"{base} passed through {depth} pointer levels"
        return ctypes.POINTER(_lib.STRUCTS[base])
    return ctypes.c_void_p


def _lib_path():
    from omni3d_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    return _lib.LIB_PATH


def test_bindings_match_header_prototypes():
    """every c3d.h prototype is exported by the library and bound in _lib.SIGNATURES with the same arity, argument types
    and return type; nothing else is bound."""
    from omni3d_b200 import _lib
    protos = _prototypes()
    assert len(protos) >= 6
    unbound, undeclared = sorted(set(protos) - set(_lib.SIGNATURES)), sorted(set(_lib.SIGNATURES) - set(protos))
    assert not unbound and not undeclared, \
        f"declared in include/c3d.h but not in _lib.SIGNATURES: {unbound}; in _lib.SIGNATURES but not declared: {undeclared}"
    so = ctypes.CDLL(_lib_path())
    missing = [name for name in protos if not hasattr(so, name)]
    assert not missing, f"declared in include/c3d.h but not exported by libc3d.so: {missing}"
    bad = []
    for name, (ret, params) in protos.items():
        bound_ret, bound_params = _lib.SIGNATURES[name]
        if bound_ret is not _expected_ctype(*ret):
            bad.append(f"{name}: returns {ret}, bound as {bound_ret.__name__}")
        if len(bound_params) != len(params):
            bad.append(f"{name}: {len(params)} parameters, bound with {len(bound_params)}")
            continue
        for i, (p, t) in enumerate(zip(params, bound_params)):
            if t is not _expected_ctype(*p):
                bad.append(f"{name} parameter {i}: {p}, bound as {t.__name__}")
    assert not bad, "\n".join(bad)
    assert _lib.lib().c3d_abi_version() >= 1


def test_struct_mirrors_match_header_layout(tmp_path):
    """sizeof and every field's offset / size of the ctypes mirrors equal what the C compiler makes of c3d.h."""
    from omni3d_b200 import _lib
    cc = shutil.which("cc")
    assert cc, "no host C compiler `cc` on PATH"
    body = []
    for cname, mirror in _lib.STRUCTS.items():
        body.append(f'  printf("{cname} sizeof %zu\\n", sizeof({cname}));')
        for f, _ in mirror._fields_:
            body.append(f'  printf("{cname} {f} %zu %zu\\n", offsetof({cname}, {f}), sizeof((({cname}*)0)->{f}));')
    src, exe = tmp_path / "layout.c", tmp_path / "layout"
    src.write_text("#include <stddef.h>\n#include <stdio.h>\n#include \"c3d.h\"\nint main(void) {\n" + "\n".join(body)
                   + "\n  return 0;\n}\n")
    r = subprocess.run([cc, "-std=c99", "-I", os.path.dirname(HEADER), str(src), "-o", str(exe)], capture_output=True,
                       text=True)
    assert r.returncode == 0, f"layout probe does not compile against c3d.h:\n{r.stderr}"
    layout = {}
    for line in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines():
        cname, field, *vals = line.split()
        layout[cname, field] = tuple(int(v) for v in vals)
    bad = []
    for cname, mirror in _lib.STRUCTS.items():
        if (ctypes.sizeof(mirror),) != layout[cname, "sizeof"]:
            bad.append(f"sizeof({cname}) = {layout[cname, 'sizeof'][0]}, {mirror.__name__} has {ctypes.sizeof(mirror)}")
        for f, _ in mirror._fields_:
            got = (getattr(mirror, f).offset, getattr(mirror, f).size)
            if got != layout[cname, f]:
                bad.append(f"{cname}.{f} at (offset, size) {layout[cname, f]}, {mirror.__name__}.{f} at {got}")
    assert not bad, "\n".join(bad)


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
    L = _lib.lib()
    d = _lib.ConvDesc(N=32, H=640, W=640, Cin=16, Cout=16, KH=3, KW=3, stride=1, pad=1)       # DLA level0: halo path
    assert conv.num_tiles(d) == (132 * 3, 1, 128)
    d = _lib.ConvDesc(N=32, H=160, W=160, Cin=256, Cout=256, KH=3, KW=3, stride=1, pad=1)     # FPN output conv
    t, th, tw = conv.num_tiles(d)
    assert th * tw <= 128 and t == 32 * -(-160 // th) * -(-160 // tw)
    assert L.c3d_nms_workspace_bytes(32, 8192) > L.c3d_nms_workspace_bytes(32, 4096) > 32 * 4096 * 64 * 8
    null = ctypes.c_void_p(None)
    rc = L.c3d_anchor_match(null, 10, null, null, null, 1, 1, 0.7, null, null, null, null, null, null, null)
    assert rc != 0 and b"anchor_match" in L.c3d_last_error()
    with pytest.raises(_lib.C3DError):
        _lib.check(rc)
    # c3d_pack_conv_weight: null source, no output, stride-2 phase outputs for a weight that is not 3x3
    p = [ctypes.c_void_p(256 * k) for k in range(1, 8)]   # non-null dummies: every case is rejected before they are used
    pack = lambda **kw: L.c3d_pack_conv_weight(ctypes.byref(_lib.PackDesc(**{**dict(Cout=16, Cin=16, KH=3, KW=3), **kw})), None)
    assert pack(fwd=p[1], dgrad=p[2]) == _lib.C3D_EINVAL and b"null source" in L.c3d_last_error()
    assert pack(src=p[0]) == _lib.C3D_EINVAL and b"no output" in L.c3d_last_error()
    assert pack(src=p[0], fwd=p[1], phase=(ctypes.c_void_p * 4)(*p[3:7]), KH=1, KW=1) == _lib.C3D_EINVAL \
        and b"3x3" in L.c3d_last_error()


def test_conv_descriptor_argument_checks_without_gpu():
    """c3d_conv2d_fwd validates the descriptor before any CUDA call: odd outputs have no nearest-x2 addend, the in-place
    accumulate needs a bf16 output, the split channel placement needs a multiple of 16 and excludes addend / statistics."""
    from omni3d_b200 import _lib
    L = _lib.lib()
    p = ctypes.c_void_p(256)                       # non-null dummies: every case below is rejected before they are used

    def call(d, addend=p, stats=None):
        return L.c3d_conv2d_fwd(ctypes.byref(d), p, p, None, addend, p, stats, None)

    def desc(**kw):                                # a 3x3 conv of 2 x 8 x 8 x 64 unless kw says otherwise
        return _lib.ConvDesc(**{**dict(N=2, H=8, W=8, Cin=64, Cout=64, KH=3, KW=3, stride=1, pad=1), **kw})

    assert call(desc(H=9, W=11, add_mode=2)) == _lib.C3D_EINVAL and b"even output" in L.c3d_last_error()   # up2, 9 x 11 output
    assert call(desc(add_mode=1), addend=None) == _lib.C3D_EINVAL and b"addend missing" in L.c3d_last_error()
    assert call(desc(out_fp32=1, add_mode=3)) == _lib.C3D_EINVAL and b"bf16 output" in L.c3d_last_error()  # accumulate into fp32
    d = desc(KH=2, KW=2, pad=0, out_h=8, out_w=8, y_split_c=24, y_split_off=100)                     # split not a multiple of 16
    assert call(d, addend=None) == _lib.C3D_EINVAL and b"y_split_c" in L.c3d_last_error()
    assert call(desc(stride=3), addend=None) == _lib.C3D_EINVAL and b"stride" in L.c3d_last_error()
    with pytest.raises(_lib.C3DError):
        _lib.check(_lib.C3D_EINVAL)


def test_entry_point_argument_checks_without_gpu():
    """the linear, weight-gradient, SGD, max-pool backward, linear-weight pack and ROIAlign entry points reject bad
    arguments with C3D_EINVAL and a message before any CUDA call; an empty linear layer is a no-op."""
    from omni3d_b200 import _lib
    L = _lib.lib()
    p = ctypes.c_void_p(256)                       # non-null dummies: every case below is rejected before they are used

    def einval(rc, msg):
        return rc == _lib.C3D_EINVAL and msg in L.c3d_last_error()

    # linear layers: (nseg, seg_rows, seg_stride) row blocks
    assert einval(L.c3d_linear_fwd(p, p, None, p, 2, 64, 32, 64, 64, 0, 0, None), b"seg_stride < seg_rows")
    assert einval(L.c3d_linear_dgrad(p, p, p, 2, 64, 63, 64, 64, 1, None), b"seg_stride < seg_rows")
    assert einval(L.c3d_linear_wgrad(p, p, p, 1, 2**31, 2**31, 64, 64, 0, 0, None), b"INT32_MAX")   # no silent truncation
    assert einval(L.c3d_linear_fwd(p, p, None, p, 1, 2**31, 2**31, 64, 64, 0, 0, None), b"INT32_MAX")
    assert L.c3d_linear_fwd(p, p, None, p, 0, 64, 64, 64, 64, 0, 0, None) == _lib.C3D_OK                # nothing to do
    assert L.c3d_linear_dgrad(p, p, p, 4, 0, 0, 64, 64, 0, None) == _lib.C3D_OK
    d = _lib.ConvDesc(N=2, H=8, W=8, Cin=64, Cout=64, KH=3, KW=3, stride=1, pad=1)
    assert einval(L.c3d_conv2d_wgrad(ctypes.byref(d), p, p, None, 1, None), b"wgrad: null pointer")
    assert einval(L.c3d_sgd_momentum(None, p, p, 1024, 0.1, None, 0.9, 1e-4, 1.0, None, None), b"sgd")
    assert einval(L.c3d_maxpool2_bwd(p, p, p, 2, 8, 8, 12, 0, 0, 1, None), b"maxpool2_bwd")             # C % 8 != 0
    assert einval(L.c3d_pack_linear_weight(p, 64, 64, 0, 0, p, None, None), b"pack_linear_weight")      # no transpose
    lv = _lib.RoiLevels(num_levels=1, num_images=0)
    lv.feat[0], lv.H[0], lv.W[0], lv.scale[0] = 256, 8, 8, 0.25
    assert einval(L.c3d_roi_align_fwd(ctypes.byref(lv), p, 4, 64, 7, 7, p, None), b"num_images")
    assert einval(L.c3d_roi_align_bwd(ctypes.byref(lv), p, 4, 64, 7, 7, p, None), b"num_images")
