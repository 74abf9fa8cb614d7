"""The C ABI's context owns its memory through member types (gpu-pruner_b200/csrc/gpr_api.cu): every device and pinned
buffer, event and stream of gpr_ctx releases itself, and gpr_destroy only stops what could still use them.  Read from
the source, so a buffer added later with a hand-written release, or a release moved ahead of the scan's shutdown,
fails here on any machine."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "gpu-pruner_b200", "csrc", "gpr_api.cu")

OWNERS = {"Buf", "Handle"}
RELEASES = ("cudaFree", "cudaFreeHost", "cudaEventDestroy", "cudaStreamDestroy", "cudaIpcCloseMemHandle", "CommDestroy")
# the releases outside the owner types: caller memory, peer mappings, the communicator and a stream the context made
OUTSIDE = {("gpr_host_free", "cudaFreeHost"), ("gpr_device_free", "cudaFree"),
           ("gpr_destroy", "cudaIpcCloseMemHandle"), ("gpr_destroy", "CommDestroy"), ("gpr_comm_destroy", "CommDestroy"),
           ("gpr_destroy", "cudaStreamDestroy")}


def _code():
    """the source with comments, string and character literals blanked (line breaks kept)"""
    src = open(SRC).read()
    out, i, n = [], 0, len(src)
    while i < n:
        if src.startswith("//", i):
            j = src.find("\n", i)
            i = n if j < 0 else j
        elif src.startswith("/*", i):
            j = src.index("*/", i) + 2
            out.append("\n" * src.count("\n", i, j))
            i = j
        elif src[i] in "\"'":
            q, j = src[i], i + 1
            while src[j] != q:
                j += 2 if src[j] == "\\" else 1
            out.append(q + q)
            i = j + 1
        else:
            out.append(src[i])
            i += 1
    return "".join(out)


def _definition(lines, at):
    """the top-level struct or function whose text holds line `at`: the nearest line above that starts in column 0
    and opens one"""
    for line in reversed(lines[:at + 1]):
        m = re.match(r"(?:struct|class)\s+(\w+)", line)
        if m:
            return m.group(1)
        if re.match(r"[A-Za-z_]", line) and "(" in line and not line.startswith(("template", "using")):
            return re.findall(r"(\w+)\s*\(", line)[0]
    return None


def _body(code, head):
    """the braces of the definition that starts with `head`"""
    i = code.index(head)
    j = code.index("{", i)
    depth = 0
    for k in range(j, len(code)):
        depth += {"{": 1, "}": -1}.get(code[k], 0)
        if depth == 0:
            return code[j:k + 1]
    raise AssertionError(head)


def test_only_the_owner_types_release_context_memory():
    lines = _code().split("\n")
    found = set()
    for at, line in enumerate(lines):
        for m in re.finditer(r"\b(%s)\s*\(" % "|".join(RELEASES), line):
            found.add((_definition(lines, at), m.group(1)))
    inside = {f for f in found if f[0] in OWNERS}
    assert found - inside == OUTSIDE, sorted(found - inside)
    assert inside == {("Buf", "cudaFree"), ("Buf", "cudaFreeHost")}, inside


def test_the_context_keeps_no_capacity_or_handle_by_hand():
    ctx = _body(_code(), "struct gpr_ctx {")
    assert not re.findall(r"\b\w+_cap\b", ctx), re.findall(r"\b\w+_cap\b", ctx)
    assert not re.search(r"\bcudaEvent_t\b", ctx)
    # the one raw stream: the caller's, which the context must never destroy, unless own_stream
    assert re.findall(r"\bcudaStream_t\s+(\w+)", ctx) == ["stream"]
    assert re.search(r"\bown_stream\b", ctx)


def test_destroy_stops_the_scan_before_anything_is_released():
    body = _body(_code(), "void gpr_destroy(gpr_ctx* ctx) {")
    first = {k: body.find(k) for k in ("scan_pipe_abort(", "cudaStreamSynchronize(", "CommDestroy(",
                                       "cudaIpcCloseMemHandle(", "cudaStreamDestroy(", "delete ctx")}
    assert all(v >= 0 for v in first.values()), first
    order = sorted(first, key=first.get)
    assert order == ["scan_pipe_abort(", "cudaStreamSynchronize(", "CommDestroy(", "cudaIpcCloseMemHandle(",
                     "cudaStreamDestroy(", "delete ctx"], order
