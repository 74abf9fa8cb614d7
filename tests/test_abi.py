"""CPU: libgpr.so loads, exports every symbol include/gpr.h declares, the ctypes mirror matches
the header's struct layout, and the product path fails loudly without a CUDA device (no CPU
fallback).  No compute is attempted here."""
import ctypes as C
import os
import re
import subprocess
import sys
import textwrap

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "gpr.h")


def _declared_symbols():
    src = open(HEADER).read()
    return sorted(set(re.findall(r"^GPR_API\s+[\w\s\*]+?\b(gpr_\w+)\s*\(", src, flags=re.M)))


def test_header_declares_expected_entry_points():
    syms = _declared_symbols()
    for must in ("gpr_create", "gpr_decide", "gpr_decide_async", "gpr_sync", "gpr_append",
                 "gpr_decide_resident", "gpr_comm_init", "gpr_last_error", "gpr_destroy", "gpr_version"):
        assert must in syms
    assert len(syms) >= 26


def test_library_exports_every_declared_symbol():
    from gpu_pruner_b200 import ffi
    lib = ffi.load()
    for s in _declared_symbols():
        assert hasattr(lib, s), f"libgpr.so does not export {s}"
        assert s in ffi.PROTOTYPES, f"ffi.py has no prototype for {s}"
    assert set(ffi.PROTOTYPES) == set(_declared_symbols())
    assert lib.gpr_version() == 200


def test_struct_layout_matches_a_c_compiler(tmp_path):
    """sizeof/offsetof as gcc sees include/gpr.h == the ctypes mirror."""
    from gpu_pruner_b200 import ffi
    prog = tmp_path / "layout.c"
    prog.write_text(textwrap.dedent(r'''
        #include <stdio.h>
        #include <stddef.h>
        #include "gpr.h"
        int main(void) {
          printf("%zu %zu %zu %zu\n", sizeof(gpr_config), sizeof(gpr_window), sizeof(gpr_result), sizeof(gpr_device_info));
          printf("%zu %zu %zu\n", offsetof(gpr_config, stream), offsetof(gpr_window, power_threshold), offsetof(gpr_result, kernel_ms));
          printf("%zu %zu\n", offsetof(gpr_window, n_pods), offsetof(gpr_window, row_stride));
          return 0; }'''))
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)])
    out = subprocess.check_output([str(exe)]).decode().split()
    got = list(map(int, out))
    want = [C.sizeof(ffi.gpr_config), C.sizeof(ffi.gpr_window), C.sizeof(ffi.gpr_result),
            C.sizeof(ffi.gpr_device_info), ffi.gpr_config.stream.offset,
            ffi.gpr_window.power_threshold.offset, ffi.gpr_result.kernel_ms.offset,
            ffi.gpr_window.n_pods.offset, ffi.gpr_window.row_stride.offset]
    assert got == want


def test_every_struct_field_matches_the_ctypes_mirror(tmp_path):
    """all six structs of include/gpr.h: sizeof and the offset of every field, gcc vs gpu_pruner_b200/ffi.py"""
    import abi_parse
    from gpu_pruner_b200 import ffi
    structs = abi_parse.structs()
    assert set(structs) == {"gpr_config", "gpr_window", "gpr_result", "gpr_device_info", "gpr_text_span", "gpr_text_grid"}
    lines = []
    for name, fields in structs.items():
        lines.append(f'printf("{name} %zu\\n", sizeof({name}));')
        for _, _, f, _ in fields:
            lines.append(f'printf("{name}.{f} %zu\\n", offsetof({name}, {f}));')
    prog = tmp_path / "fields.c"
    prog.write_text("#include <stdio.h>\n#include <stddef.h>\n#include \"gpr.h\"\nint main(void) {\n" + "\n".join(lines) + "\nreturn 0; }\n")
    exe = tmp_path / "fields"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)])
    got = dict(l.split() for l in subprocess.check_output([str(exe)]).decode().splitlines())
    for name, fields in structs.items():
        mirror = getattr(ffi, name)
        assert int(got[name]) == C.sizeof(mirror), name
        assert [f for _, _, f, _ in fields] == [f[0] for f in mirror._fields_], name
        for _, _, f, _ in fields:
            assert int(got[f"{name}.{f}"]) == getattr(mirror, f).offset, (name, f)
    # the power threshold travels at the END of gpr_text_grid (power samples are snapped to it at parse time)
    assert [f for _, _, f, _ in structs["gpr_text_grid"]][-1] == "power_threshold"
    assert (int(got["gpr_text_grid"]), int(got["gpr_text_grid.power_threshold"])) == (48, 40)


def test_header_is_plain_c():
    subprocess.check_call(["gcc", "-std=c99", "-pedantic", "-Wall", "-Werror", "-fsyntax-only", "-x", "c", HEADER])


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


@pytest.mark.skipif(_has_gpu(), reason="checks the no-GPU failure mode")
def test_no_cpu_fallback_without_a_device():
    import gpu_pruner_b200 as g
    with pytest.raises(g.GprError) as ei:
        g.IdleEngine(device=0)
    assert ei.value.code == g.ffi.GPR_E_CUDA
    assert "no CPU fallback" in str(ei.value)


def test_bad_config_is_an_error_code_not_a_crash():
    from gpu_pruner_b200 import ffi
    lib = ffi.load()
    h = C.c_void_p()
    cfg = ffi.gpr_config()
    cfg.struct_size = 3
    assert lib.gpr_create(C.byref(cfg), C.byref(h)) == ffi.GPR_E_INVALID
    assert b"struct_size" in lib.gpr_last_error(None)
    assert lib.gpr_create(None, C.byref(h)) == ffi.GPR_E_INVALID
    assert lib.gpr_sync(None) == ffi.GPR_E_INVALID
    lib.gpr_destroy(None)  # no-op


def test_product_package_never_imports_the_oracle():
    """no import / include / link / call of anything under oracle/ from the product tree"""
    pkg = os.path.join(ROOT, "gpu-pruner_b200")
    bad = re.compile(r"(^\s*(from|import)\s+oracle\b)|(#include\s*[\"<][^\">]*oracle)|libgpr_oracle|\bgpo_\w+|oracle_np|oracle_c\b",
                     re.M)
    for dp, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".cpp", ".cc", ".h", ".hpp", "Makefile")):
                txt = open(os.path.join(dp, f), errors="replace").read()
                m = bad.search(txt)
                assert m is None, f"{os.path.join(dp, f)} uses the oracle: {m.group(0)!r}"
    out = subprocess.run(["ldd", os.path.join(pkg, "libgpr.so")], capture_output=True, text=True).stdout
    assert "oracle" not in out


def test_biased_u8_helpers_round_trip():
    """GPR_FMT_U8B: 0 = no sample, b = value + 1; only integer samples 0..254 are representable"""
    import gpu_pruner_b200 as g
    u = np.array([[[0, np.nan, 100, 254, 1]]], np.float32)
    b = g.to_biased_u8(u)
    assert b.dtype == np.uint8 and b.tolist() == [[[1, 0, 101, 255, 2]]]
    back = g.from_biased_u8(b)
    assert np.array_equal(np.isnan(back), np.isnan(u)) and np.array_equal(np.nan_to_num(back), np.nan_to_num(u))
    for bad in (0.5, -1.0, 255.0, np.inf):
        with pytest.raises(ValueError):
            g.to_biased_u8(np.array([bad], np.float32))
    assert (g.ffi.GPR_FMT_F32, g.ffi.GPR_FMT_U8B) == (0, 1)
