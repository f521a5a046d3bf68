"""CPU-side checks of the drop-in boundary: libtfl.so loads and exports every symbol
include/tfl.h declares; without a CUDA device the product refuses to run (no fallback)."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    txt = open(os.path.join(ROOT, "include", "tfl.h")).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(tfl_[a-z0-9_]+)\s*\(", txt)))


def test_header_and_binding_agree():
    from fluidnet_b200 import _lib
    assert sorted(_lib.SYMBOLS) == header_symbols()


def test_library_exports_every_symbol():
    from fluidnet_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for s in header_symbols():
        assert hasattr(lib, s), "libtfl.so does not export " + s
    lib.tfl_version.restype = ctypes.c_char_p
    assert b"sm_90a" in lib.tfl_version()
    assert lib.tfl_advect_method_from_string(b"maccormackOurs") == 5
    assert lib.tfl_advect_method_from_string(b"bogus") == -1


def test_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from fluidnet_b200 import tfluids
    from fluidnet_b200._lib import TflError
    t = torch.zeros(1, 1, 4, 4, 4)
    with pytest.raises(TflError):
        tfluids.emptyDomain(t, True, 1)
    h = ctypes.c_void_p()
    from fluidnet_b200 import _lib
    assert _lib.load().tfl_create(ctypes.byref(h), 0) != 0


def test_product_never_imports_oracle():
    """The oracle is test infrastructure: nothing under fluidnet_b200/ may reference it."""
    pkg = os.path.join(ROOT, "fluidnet_b200")
    for dirpath, _, files in os.walk(pkg):
        if "build" in dirpath:
            continue
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp", ".lua")):
                txt = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(import|from)\s+oracle", txt, flags=re.M), f
                assert "liboracle" not in txt and "libtfluids_ref" not in txt, f


def test_lua_shim_is_consistent_with_the_header():
    """fluidnet_b200/lua/tfluids_ffi.lua cannot be executed here (no LuaJIT), so it is checked statically:
    every function its ffi.cdef declares exists in include/tfl.h with the same number of parameters, every
    lib.tfl_* it calls is declared, and it defines every tfluids.* function of the reference's init.lua that
    the library implements."""
    import os
    import re
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

    def decls(text):
        text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
        text = re.sub(r"//[^\n]*", "", text)
        out = {}
        for m in re.finditer(r"\b(tfl_[a-z0-9_]+)\s*\(([^;{}]*?)\)\s*;", text, flags=re.S):
            args = m.group(2).strip()
            out[m.group(1)] = 0 if args in ("", "void") else len(args.split(","))
        return out

    header = decls(open(os.path.join(root, "include", "tfl.h")).read())
    lua = open(os.path.join(root, "fluidnet_b200", "lua", "tfluids_ffi.lua")).read()
    start = lua.index("ffi.cdef[[")
    cdef = decls(lua[start:lua.index("]]", start)])
    assert len(cdef) >= 30
    assert not set(cdef) - set(header), sorted(set(cdef) - set(header))
    assert not [(k, header[k], cdef[k]) for k in cdef if header[k] != cdef[k]]
    assert not set(re.findall(r"lib\.(tfl_[a-z0-9_]+)", lua)) - set(cdef)
    defined = set(re.findall(r"^function tfluids\.([A-Za-z]+)", lua, flags=re.M))
    for name in ("advectScalar", "advectVel", "setWallBcsForward", "velocityDivergenceForward", "velocityUpdateForward",
                 "addBuoyancy", "addGravity", "vorticityConfinement", "solveLinearSystemJacobi", "solveLinearSystemPCG",
                 "emptyDomain", "flagsToOccupancy", "normalizePressureMean", "rectangularBlur", "signedDistanceField",
                 "volumetricUpSamplingNearestForward", "volumetricUpSamplingNearestBackward",
                 "velocityDivergenceBackward", "velocityUpdateBackward"):
        assert name in defined, name


def test_header_is_plain_c_and_a_c_host_links_against_the_abi(tmp_path):
    """include/tfl.h must be consumable from C (LuaJIT's ffi.cdef, cgo, a C host): examples/c_host.c -- one step
    through the ABI from plain C99, the library dlopen'ed -- compiles, and without a GPU fails cleanly in
    tfl_create (exit code 1, a message, no crash)."""
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = os.path.join(root, "examples", "c_host.c")
    exe = str(tmp_path / "c_host")
    r = subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I" + os.path.join(root, "include"), src, "-o", exe, "-ldl"],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe, os.path.join(root, "fluidnet_b200", "libtfl.so")], capture_output=True, text=True, timeout=120)
    assert r.returncode in (0, 1), (r.returncode, r.stderr)
    if r.returncode == 1:
        assert "tfl_create failed" in r.stderr or "libtfl:" in r.stderr
    else:
        assert "step done" in r.stdout
