"""The C-ABI library loads without a GPU and exports exactly what include/frosting_b200.h declares."""
import ctypes as C
import os
import re

import pytest

from frosting_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_source():
    src = open(os.path.join(ROOT, "include", "frosting_b200.h")).read()
    return re.sub(r"/\*.*?\*/", "", src, flags=re.S)


def header_functions():
    return sorted(set(re.findall(r"\b(fb200_[a-z_0-9]+)\s*\(", header_source())))


def header_prototypes():
    """name -> (return type, [parameter types]) of every function the header declares; a type is (base, pointer depth)
    with `const` dropped, e.g. `const float* d_x` -> ("float", 1); `(void)` -> []."""
    src = re.sub(r"^\s*#.*$", "", header_source(), flags=re.M)

    def ctype(decl):
        words = decl.replace("*", " ").split()
        if len(words) > 1 and not decl.rstrip().endswith("*"):
            words = words[:-1]                                   # the parameter's name
        return " ".join(w for w in words if w != "const"), decl.count("*")

    out = {}
    for ret, name, params in re.findall(r"([\w\s*]+?)\b(fb200_\w+)\s*\(([^;{}()]*)\)\s*;", src):
        params = [] if params.strip() == "void" else [ctype(p) for p in params.split(",")]
        out[name] = (ctype(ret + " _"), params)
    return out


def test_declared_symbols_are_exported_at_the_header_abi_version():
    """ABI 9: fb200_layout carries the hit lists (img_last_entry, bin_sub_hits).  The library, the binding and the
    header's FB200_ABI_VERSION agree."""
    L = _lib.lib()
    names = header_functions()
    assert len(names) >= 14
    for n in names:
        assert hasattr(L, n), f"{n} declared in the header but not exported"
    assert sorted(_lib.EXPORTED) == names, "frosting_b200/_lib.py:EXPORTED out of sync with the header"
    version = re.search(r"#define FB200_ABI_VERSION (\d+)", header_source())
    assert L.fb200_abi_version() == _lib.ABI_VERSION == int(version.group(1)) == 9
    count = re.search(r"#define FB200_ABI_STRUCTS (\d+)", header_source())
    assert int(count.group(1)) == len(_lib.ABI_STRUCTS)


SCALARS = {"int": C.c_int, "int32_t": C.c_int32, "int64_t": C.c_int64, "size_t": C.c_size_t, "float": C.c_float}


def test_binding_matches_every_prototype():
    """restype and argtypes of each bound function against the header: scalars at their exact ctypes type, fb200_*
    struct pointers as POINTER(<the struct's mirror>), every other pointer as some pointer type."""
    L = _lib.lib()
    mirrors = dict(_lib.ABI_STRUCTS)
    protos = header_prototypes()
    assert sorted(protos) == header_functions()

    def mismatch(t, decl):
        base, depth = decl
        if depth == 0:
            return t is not SCALARS[base]
        if depth == 1 and base in mirrors:
            return t is not C.POINTER(mirrors[base])
        return not (isinstance(t, type) and issubclass(t, (C.c_void_p, C.c_char_p, C._Pointer)))

    bad = []
    for name, (ret, params) in protos.items():
        fn = getattr(L, name)
        if mismatch(fn.restype, ret):
            bad.append(f"{name}: restype {fn.restype} for {ret}")
        if fn.argtypes is None or len(fn.argtypes) != len(params):
            bad.append(f"{name}: argtypes {fn.argtypes} for {len(params)} parameters")
            continue
        bad += [f"{name}: argument {i} {t} for {p}" for i, (t, p) in enumerate(zip(fn.argtypes, params))
                if mismatch(t, p)]
    assert not bad, "\n".join(bad)


def test_workspace_size_queries_are_host_only_and_monotonic():
    L = _lib.lib()
    assert L.fb200_geom_bytes(0) >= 128
    g1, g2 = L.fb200_geom_bytes(1000), L.fb200_geom_bytes(2000)
    assert g2 > g1 >= 1000 * 109
    i1 = L.fb200_image_bytes(1920, 1080)
    assert i1 >= 1920 * 1080 * 12 + 8160 * 8
    assert L.fb200_image_bytes(1921, 1080) > i1
    b = L.fb200_binning_bytes(10_000)
    assert 10_000 * 52 <= b <= 10_000 * 52 + 1024      # 20 B of keys + 8 sub-tile hit lists of 4 B per instance


def test_layout_offsets_are_aligned_and_ordered():
    L = _lib.lib()
    lay = _lib.Layout()
    assert L.fb200_get_layout(1000, 256, 128, 5000, C.byref(lay)) == 0
    offs = [getattr(lay, n) for n, _ in _lib.Layout._fields_]
    assert all(o % 128 == 0 for o in offs)
    assert lay.geom_rec < lay.geom_depth < lay.geom_rect < lay.geom_clamped < lay.geom_acc
    assert lay.img_final_T < lay.img_n_contrib < lay.img_last_entry < lay.img_ranges < lay.img_tile_count
    assert lay.bin_point_list < lay.bin_keys < lay.bin_sub_hits
    # the two hit-list arrays: one u32 per pixel, eight u32 per instance, both inside their workspaces
    assert lay.img_ranges - lay.img_last_entry >= 4 * 256 * 128
    assert lay.bin_sub_hits + 4 * 8 * 5000 <= L.fb200_binning_bytes(5000)


def test_workspace_views_start_at_the_aligned_base():
    """_lib.workspace_views reads each sub-array where the library carves it: at its fb200_layout offset from the
    buffer's first 128-byte aligned byte, whatever the buffer's own alignment."""
    import torch
    P, W, H, cap, R = 1000, 250, 130, 5000, 4000
    L = _lib.lib()
    lay = _lib.Layout()
    assert L.fb200_get_layout(P, W, H, cap, C.byref(lay)) == 0
    sizes = (L.fb200_geom_bytes(P), L.fb200_image_bytes(W, H), L.fb200_binning_bytes(cap))
    bufs = [torch.zeros(n + 128, dtype=torch.uint8)[40:40 + n] for n in sizes]      # 8 bytes past a 64-byte boundary
    assert all(b.data_ptr() % 128 for b in bufs)
    g, im, bn = ((b.data_ptr() + 127) // 128 * 128 for b in bufs)
    v = _lib.workspace_views(*bufs, P, W, H, cap, R)
    T = 16 * 9
    expect = dict(rec=(g + lay.geom_rec, (P, 12)), clamped=(g + lay.geom_clamped, (P,)), acc=(g + lay.geom_acc, (P, 12)),
                  final_T=(im + lay.img_final_T, (H, W)), ranges=(im + lay.img_ranges, (T, 2)),
                  tile_count=(im + lay.img_tile_count, (T,)), keys=(bn + lay.bin_keys, (R,)),
                  sub_hits=(bn + lay.bin_sub_hits, (8 * R,)))
    assert {k: (v[k].data_ptr(), tuple(v[k].shape)) for k in expect} == expect
    assert v.keys() == {"rec", "depth", "rect", "clamped", "acc", "final_T", "n_contrib", "last_entry", "ranges",
                        "tile_count", "point_list", "keys", "sub_hits"}
    assert _lib.workspace_views(None, bufs[1], None, P, W, H, 0, 0).keys() == \
        {"final_T", "n_contrib", "last_entry", "ranges", "tile_count"}


def test_argument_errors_are_reported_without_touching_cuda():
    L = _lib.lib()
    lay = _lib.Layout()
    assert L.fb200_get_layout(-1, 256, 128, 0, C.byref(lay)) == -1
    assert b"layout" in L.fb200_last_error()
    prm = _lib.Params(P=10, sh_degree=0, sh_coeffs=0, image_width=64, image_height=64, tanfovx=0.5, tanfovy=0.5,
                      scale_modifier=1.0, prefiltered=0, debug=0)
    inp = _lib.Inputs()      # all NULL
    ws = _lib.Workspace()
    rc = L.fb200_forward(C.byref(prm), C.byref(inp), C.byref(ws), None, None, None)
    assert rc == -1 and b"missing" in L.fb200_last_error()
    # exactly-one-of checks carry the reference's messages (DGR/diff_gaussian_rasterization/__init__.py:191-195)
    dummy = C.c_void_p(0x1000)
    inp = _lib.Inputs(d_background=dummy, d_means3D=dummy, d_opacities=dummy, d_viewmatrix=dummy,
                      d_projmatrix=dummy, d_campos=dummy)
    rc = L.fb200_forward(C.byref(prm), C.byref(inp), C.byref(ws), None, None, None)
    assert rc == -1 and b"excatly one of either SHs or precomputed colors" in L.fb200_last_error()
    inp.d_colors_precomp = dummy
    rc = L.fb200_forward(C.byref(prm), C.byref(inp), C.byref(ws), None, None, None)
    assert rc == -1 and b"exactly one of either scale/rotation pair" in L.fb200_last_error()
    with pytest.raises(_lib.Fb200Error):
        _lib.check(rc)
    # debug has two defined bits (sync, no sub-tile culling); any other bit is an error, not the default kernels
    prm.debug = 8
    rc = L.fb200_forward(C.byref(prm), C.byref(inp), C.byref(ws), None, None, None)
    assert rc == -1 and b"debug" in L.fb200_last_error()
    prm.debug = 0
    # frosting mode: the parameter block replaces the attribute pointers, it does not coexist with them
    d = dummy
    fp = _lib.FrostingParams(P=10, n_verts=4, n_faces=2, sh_rest=15, d_bary_logits=d, d_cells=d, d_faces=d, d_inner_verts=d,
                             d_outer_verts=d, d_opacity_logits=d, d_log_scales=d, d_quats=d, d_sh_dc=d, d_sh_rest=d)
    prm.sh_degree, prm.sh_coeffs = 3, 16
    inp = _lib.Inputs(d_background=d, d_means3D=d, d_viewmatrix=d, d_projmatrix=d, d_campos=d, frosting=C.addressof(fp))
    rc = L.fb200_forward(C.byref(prm), C.byref(inp), C.byref(ws), None, None, None)
    assert rc == -1 and b"frosting mode: the attribute / mask pointers" in L.fb200_last_error()
    inp.d_means3D = None
    prm.sh_coeffs = 9
    rc = L.fb200_forward(C.byref(prm), C.byref(inp), C.byref(ws), None, None, None)
    assert rc == -1 and b"do not match the parameter block" in L.fb200_last_error()
    prm.sh_coeffs = 16
    rc = L.fb200_forward(C.byref(prm), C.byref(inp), C.byref(ws), None, None, None)
    assert rc == -1 and b"workspace pointers missing" in L.fb200_last_error()      # got past the frosting checks


def test_profile_and_launch_counter_entry_points():
    assert _lib.kernel_launches() >= 0
    _lib.profile_enable(True)
    t = _lib.profile_read()
    assert set(t) == set(_lib.STAGES) and all(v == -1.0 for v in t.values())   # nothing recorded without a GPU
    _lib.profile_enable(False)
