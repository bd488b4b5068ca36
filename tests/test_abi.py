"""CPU: the C-ABI library loads and exports every symbol include/rwgpu.h declares (no compute calls)."""
import ctypes
import os
import re

from risingwave_b200 import abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_symbols():
    src = open(os.path.join(ROOT, "include", "rwgpu.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(rwgpu_\w+)\s*\(", src)))


def test_header_and_python_symbol_lists_agree():
    assert _header_symbols() == sorted(abi.ABI_SYMBOLS)


def test_library_exports_every_symbol():
    lib = abi.load_library()  # raises if librwgpu.so is not built -- there is no fallback
    for sym in _header_symbols():
        assert hasattr(lib, sym), sym


def test_type_width_and_version():
    lib = abi.load_library()
    lib.rwgpu_type_width.restype = ctypes.c_int32
    for t, w in abi.TYPE_WIDTH.items():
        assert lib.rwgpu_type_width(t) == w
    lib.rwgpu_version.restype = ctypes.c_char_p
    assert b"sm_90a" in lib.rwgpu_version()


def test_struct_sizes_match_header():
    # x86-64 SysV layout of the structs in include/rwgpu.h
    assert ctypes.sizeof(abi.RwColumn) == 32
    assert ctypes.sizeof(abi.RwChunk) == 40
    assert ctypes.sizeof(abi.RwAggCall) == 16
    assert ctypes.sizeof(abi.RwAggDesc) == 72
    assert ctypes.sizeof(abi.RwJoinSideDesc) == 72
    assert ctypes.sizeof(abi.RwJoinDesc) == 208
    assert ctypes.sizeof(abi.RwFilterTerm) == 24


def test_product_does_not_reference_oracle():
    """The product path must never import / link the oracle (it is test infrastructure)."""
    pkg = os.path.join(ROOT, "risingwave_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cc")):
                txt = open(os.path.join(dirpath, f)).read()
                assert "liboracle" not in txt and "rwo_" not in txt and "oracle/" not in txt, f


def test_cpp_host_mirror_watermark_buffers():
    """include/rwgpu_executor.hpp BufferedWatermarks (CPU-only binary built by __graft_entry__.build()): the traces of the
    reference's test_streaming_hash_join_watermark and a three-upstream case"""
    import subprocess
    exe = os.path.join(ROOT, "build", "test_watermarks")
    if not os.path.exists(exe):
        import __graft_entry__
        __graft_entry__.build()
    r = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0 and "watermarks: ok" in r.stdout, r.stdout + r.stderr


def test_flat_exchange_layout_host_side():
    """rwgpu_shuffle_flat_layout (host arithmetic only): header of 64 x 64 int64 counts, then ops and the columns, every part
    256-byte aligned and large enough for cap rows; varlen columns are refused"""
    lib = abi.load_library()
    lib.rwgpu_shuffle_flat_layout.restype = ctypes.c_int32
    lib.rwgpu_shuffle_flat_layout.argtypes = [ctypes.POINTER(ctypes.c_int32), ctypes.c_int32, ctypes.c_int64, ctypes.POINTER(ctypes.c_int64),
                                              ctypes.POINTER(ctypes.c_int64), ctypes.POINTER(ctypes.c_int64)]
    for types, cap in (([abi.T_INT64] * 4, 1 << 20), ([abi.T_INT64, abi.T_INT32, abi.T_INT16, abi.T_DECIMAL], 1000), ([abi.T_BOOL], 7)):
        t = (ctypes.c_int32 * len(types))(*types)
        total, ops_off = ctypes.c_int64(), ctypes.c_int64()
        col_off = (ctypes.c_int64 * len(types))()
        assert lib.rwgpu_shuffle_flat_layout(t, len(types), cap, ctypes.byref(total), ctypes.byref(ops_off), col_off) == abi.RW_OK
        assert ops_off.value == 64 * 64 * 8
        prev_end = ops_off.value + cap
        for k, ty in enumerate(types):
            assert col_off[k] % 256 == 0 and col_off[k] >= prev_end
            prev_end = col_off[k] + cap * abi.TYPE_WIDTH[ty]
        assert total.value >= prev_end and total.value % 256 == 0
    t = (ctypes.c_int32 * 1)(abi.T_VARCHAR)
    total, ops_off = ctypes.c_int64(), ctypes.c_int64()
    col_off = (ctypes.c_int64 * 1)()
    assert lib.rwgpu_shuffle_flat_layout(t, 1, 10, ctypes.byref(total), ctypes.byref(ops_off), col_off) != abi.RW_OK
