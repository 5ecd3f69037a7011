"""CPU-side checks of the drop-in boundary: the C-ABI shared library builds for sm_90a, loads, exports
every symbol include/sr_gpu_ops.h declares, agrees with the ctypes struct layouts, and fails LOUDLY
(no CPU fallback) when no CUDA device is present.  No compute calls here."""
import ctypes as C
import os
import re

import pytest

from starrocks_b200 import abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_functions():
    src = open(os.path.join(ROOT, "include", "sr_gpu_ops.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(sr_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol(gpu):
    L = gpu.lib()
    declared = _declared_functions()
    assert len(declared) >= 40
    for name in declared:
        assert hasattr(L, name), f"libsr_gpu.so does not export {name}"
    assert sorted(gpu.EXPORTED_SYMBOLS) == declared


def test_ctypes_layouts_match_the_compiled_structs(gpu):
    L = gpu.lib()
    structs = [abi.sr_col_view, abi.sr_chunk_view, abi.sr_chunk_out, abi.sr_pred, abi.sr_expr, abi.sr_scan_desc,
               abi.sr_join_desc, abi.sr_join_info, abi.sr_agg_fn, abi.sr_agg_desc, abi.sr_frag_join,
               abi.sr_fragment_desc, abi.sr_part_desc, abi.sr_agg_state_array, abi.sr_fragment_plan,
               abi.sr_rf_info]
    for k, st in enumerate(structs):
        assert L.sr_abi_sizeof(k) == C.sizeof(st), st.__name__
    assert L.sr_abi_sizeof(99) == -1
    assert L.sr_abi_version() == abi.SR_ABI_VERSION
    for t, w in abi.TYPE_WIDTH.items():
        assert L.sr_type_width(t) == w
    assert L.sr_type_width(0) == 0


def test_oracle_and_product_are_separate_libraries(gpu):
    # the product never links the oracle: no orc_* symbol in libsr_gpu.so
    import subprocess
    out = subprocess.run(["nm", "-D", gpu.LIB_PATH], capture_output=True, text=True).stdout
    assert "orc_" not in out
    assert "sr_fragment_push" in out


def test_no_device_is_a_loud_error(gpu):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    with pytest.raises(gpu.GpuError) as ei:
        gpu.Context(0)
    assert ei.value.code == abi.SR_ERR_NO_DEVICE
    assert "no CPU fallback" in str(ei.value)
