"""CPU: the struct of gpr_resident_export (include/gpr.h), gpr_chunk_export, as gcc lays it out equals the ctypes mirror
of gpu_pruner_b200/ffi.py field by field, and the #[repr(C)] transcription in INTEGRATION.md §5 has the header's
fields in the header's order with the matching Rust types."""
import ctypes as C
import os
import re
import subprocess

import abi_parse as A
from test_samples_abi import RUST, _fields

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RUST_TYPES = {**RUST, ("uint64_t", 1): "*mut u64", ("uint32_t", 1): "*mut u32", ("uint8_t", 1): "*mut u8"}
NAME = "gpr_chunk_export"


def test_layout_matches_the_ctypes_mirror(tmp_path):
    from gpu_pruner_b200 import ffi
    lines = [f'printf("{NAME} %zu\\n", sizeof({NAME}));']
    lines += [f'printf("{NAME}.{f} %zu\\n", offsetof({NAME}, {f}));' for _, _, f in _fields(NAME)]
    prog = tmp_path / "fields.c"
    prog.write_text("#include <stdio.h>\n#include <stddef.h>\n#include \"gpr.h\"\nint main(void) {\n" + "\n".join(lines) +
                    "\nreturn 0; }\n")
    exe = tmp_path / "fields"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(prog), "-o",
                           str(exe)])
    got = dict(l.split() for l in subprocess.check_output([str(exe)]).decode().splitlines())
    mirror = ffi.gpr_chunk_export
    assert int(got[NAME]) == C.sizeof(mirror) == 96
    assert [f for _, _, f in _fields(NAME)] == [f[0] for f in mirror._fields_]
    for _, _, f in _fields(NAME):
        assert int(got[f"{NAME}.{f}"]) == getattr(mirror, f).offset, f


def test_rust_struct_matches_the_header():
    doc = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    sec = doc[doc.index("## 5."):doc.index("## 6.")]
    found = {m.group(1): [(f, " ".join(t.split())) for f, t in re.findall(r"pub (\w+):\s*([^,]+),", m.group(2))]
             for m in re.finditer(r"#\[repr\(C\)\]\s*pub struct (\w+) \{(.*?)\}", sec, flags=re.S)}
    assert found.get("GprChunkExport") == [(f, RUST_TYPES[(b, s)]) for b, s, f in _fields(NAME)]


def test_entry_point_takes_the_struct():
    ret, params = A.functions()["gpr_resident_export"]
    assert ret == ("int", 0)
    assert [(b, s) for b, s, _ in params] == [("gpr_ctx", 1), ("const gpr_text_grid", 1), ("int32_t", 0),
                                              ("uint32_t", 0), ("gpr_chunk_export", 1)]
