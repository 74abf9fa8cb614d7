"""CPU: the two structs of gpr_samples_scatter (include/gpr.h) — gpr_sample_batch and gpr_sample_stats — as gcc lays
them out equal the ctypes mirror of gpu_pruner_b200/ffi.py field by field, and the #[repr(C)] transcription in
INTEGRATION.md §7b has the header's fields in the header's order with the matching Rust types."""
import ctypes as C
import os
import re
import subprocess

import abi_parse as A

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ("gpr_sample_batch", "gpr_sample_stats")
RUST = {("uint32_t", 0): "u32", ("int32_t", 0): "i32", ("uint64_t", 0): "u64", ("const uint64_t", 1): "*const u64",
        ("const uint32_t", 1): "*const u32", ("const int64_t", 1): "*const i64", ("const double", 1): "*const f64"}


def _fields(name):
    src = A._strip_comments(open(A.HEADER).read())
    body = re.search(r"struct %s \{(.*?)\};" % name, src, flags=re.S).group(1)
    assert re.search(r"typedef struct %s %s;" % (name, name), src)
    out = []
    for stmt in body.split(";"):
        if stmt.strip():
            (base, stars), f, _ = A._decl(stmt.strip())
            out.append((base, stars, f))
    return out


def test_layout_matches_the_ctypes_mirror(tmp_path):
    from gpu_pruner_b200 import ffi
    lines = []
    for name in NAMES:
        lines.append(f'printf("{name} %zu\\n", sizeof({name}));')
        for _, _, f in _fields(name):
            lines.append(f'printf("{name}.{f} %zu\\n", offsetof({name}, {f}));')
    prog = tmp_path / "fields.c"
    prog.write_text("#include <stdio.h>\n#include <stddef.h>\n#include \"gpr.h\"\nint main(void) {\n" + "\n".join(lines) +
                    "\nreturn 0; }\n")
    exe = tmp_path / "fields"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(prog), "-o",
                           str(exe)])
    got = dict(l.split() for l in subprocess.check_output([str(exe)]).decode().splitlines())
    for name in NAMES:
        mirror = getattr(ffi, name)
        assert int(got[name]) == C.sizeof(mirror), name
        assert [f for _, _, f in _fields(name)] == [f[0] for f in mirror._fields_], name
        for _, _, f in _fields(name):
            assert int(got[f"{name}.{f}"]) == getattr(mirror, f).offset, (name, f)
    assert (int(got["gpr_sample_batch"]), int(got["gpr_sample_stats"])) == (48, 24)


def test_rust_structs_match_the_header():
    doc = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    sec = doc[doc.index("## 7b."):doc.index("## 8.")]
    found = {m.group(1): [(f, " ".join(t.split())) for f, t in re.findall(r"pub (\w+):\s*([^,]+),", m.group(2))]
             for m in re.finditer(r"#\[repr\(C\)\]\s*pub struct (\w+) \{(.*?)\}", sec, flags=re.S)}
    for name in NAMES:
        camel = "".join(p.capitalize() for p in name.split("_"))
        assert found.get(camel) == [(f, RUST[(b, s)]) for b, s, f in _fields(name)], name


def test_entry_point_takes_the_structs():
    ret, params = A.functions()["gpr_samples_scatter"]
    assert ret == ("int", 0)
    assert [(b, s) for b, s, _ in params] == [("gpr_ctx", 1), ("const gpr_sample_batch", 1), ("const gpr_text_grid", 1),
                                              ("int32_t", 0), ("gpr_sample_stats", 1)]
