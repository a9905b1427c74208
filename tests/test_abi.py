"""The C-ABI libraries load and export every symbol include/*.h declare (no compute calls: runs without a GPU), and the
product package refuses to run on anything but the CUDA build."""
import ctypes as C, os, pytest
from kajiya_b200._abi import declared_symbols, KjbLib, MeshMaterial, WorldDesc, WorldFrame
import conftest

INCLUDE = os.path.join(conftest.ROOT, "include")


def _exports(path):
    dll = C.CDLL(path)
    return [s for s in declared_symbols(INCLUDE) if not hasattr(dll, s)]


def test_cuda_library_exports_every_declared_symbol():
    assert os.path.exists(conftest.CUDA_SO), "kajiya_b200/csrc/libkjb.so missing: run __graft_entry__.build()"
    assert _exports(conftest.CUDA_SO) == []
    assert KjbLib(conftest.CUDA_SO).backend == "cuda-sm90a"


def test_oracle_and_emulator_export_the_same_abi(oracle_lib, emu_lib):
    assert _exports(conftest.ORACLE_SO) == [] and _exports(conftest.EMU_SO) == []
    assert oracle_lib.backend == "oracle-cpu" and emu_lib.backend == "emu-cpu"


def test_struct_layouts():
    assert C.sizeof(MeshMaterial) == 152          # inc/mesh.hlsl:52-61
    src = open(os.path.join(INCLUDE, "kjb.h")).read()
    assert "1216 bytes" in src
    # compile-time check of the FrameConstants layout against the Rust repr(C) sizes (frame_constants.rs:13-37)
    import subprocess, tempfile
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "t.c"), "w").write('#include "kjb.h"\n#include "kjb_world.h"\n_Static_assert(sizeof(kjb_frame_constants) == 1216, "fc");\n'
                                                 '_Static_assert(sizeof(kjb_view_constants) == 720, "vc");\n_Static_assert(sizeof(kjb_mesh_material) == 152, "mm");\n'
                                                 '_Static_assert(sizeof(kjb_triangle_light) == 48, "tl");\nint main(void){return 0;}\n')
        subprocess.check_call(["gcc", "-I", INCLUDE, "-c", os.path.join(d, "t.c"), "-o", os.path.join(d, "t.o")])


def test_product_fails_loudly_without_a_gpu():
    """kjb_create on the CUDA library must error (not fall back) when no device is usable."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    lib = KjbLib(conftest.CUDA_SO)
    ctx = C.c_void_p()
    assert lib.dll.kjb_create(0, C.byref(ctx)) != 0
    assert b"no CUDA device" in lib.dll.kjb_last_error(None)


def test_product_package_never_reaches_the_oracle():
    """nothing under kajiya_b200/ references oracle/ or the emulator (the oracle is test infrastructure only)"""
    pkg = os.path.join(conftest.ROOT, "kajiya_b200")
    for base, _, files in os.walk(pkg):
        if "_obj" in base:
            continue
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp")):
                txt = open(os.path.join(base, f), errors="ignore").read()
                assert "kj_oracle" not in txt and "oracle/_build" not in txt and "libkjb_emu" not in txt, f
