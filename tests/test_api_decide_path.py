"""The decision path of the C ABI (gpu-pruner_b200/csrc/gpr_api.cu).  read_window reads and checks the window before
anything is enqueued.  decide_impl then enqueues every decision through one sequence: a device window is one piece read
in place and a host window a list of staged pieces, and one loop launches the reduce over either, after the one
k_group_rows and before the one k_group_sum and the one fold.  The outputs leave through one copy, and a failed
decision marks the scratch dirty in one place.  Read from the source like tests/test_api_launch_path.py, so a second
launch or copy site, a check after the first enqueue, or a caller with its own failure rule fails here on any machine.
What the path computes is checked on the H100 by the parity, session, geometry, groups and resident suites."""
import re

from test_context_ownership import _body, _code, _definition


def _sites(pattern):
    """the definitions that hold a match of `pattern`, one entry per match"""
    lines = _code().split("\n")
    return [_definition(lines, at) for at, line in enumerate(lines) for _ in re.finditer(pattern, line)]


def _fn(name):
    """the body of the function `name`"""
    code = _code()
    return _body(code, re.search(r"^int %s\(" % name, code, re.M).group(0))


def _statements(name):
    return [s.strip() for s in _fn(name).split(";") if s.strip()]


def test_the_window_is_read_and_checked_before_the_decision():
    assert "fail(" in _fn("read_window")
    assert "fail(" not in _fn("decide_impl")
    assert _sites(r"\bread_window\s*\(") == ["read_window", "decide_impl"]


def test_one_reduce_launch_site():
    assert _sites(r"\blaunch_reduce\s*\(") == ["launch_reduce", "decide_impl"]


def test_one_enqueue_for_every_window():
    body, statements = _fn("decide_impl"), _statements("decide_impl")
    assert not re.search(r"\[[&=]?\]\s*\(", body), "a lambda stands in for a launch site"
    launches = [s for s in statements if re.search(r"\blaunch(?:_reduce)?\s*\(", s)]
    assert len(launches) == 4, launches   # k_group_rows, the reduce, k_group_sum, the fold
    for kernel in ("k_group_rows", "k_group_sum"):
        assert sum(kernel in s for s in launches) == 1, kernel
    assert sum("k_fold" in s for s in statements) == 1
    assert sum("fold_grid" in s for s in launches) == 1


def test_one_copy_delivers_the_outputs():
    """every copy of the decision stages an input, but one: the loop that copies the bitmaps, veto bits, series_max
    and idle_slots out"""
    dests = []
    for s in _statements("decide_impl"):
        dests += re.findall(r"\bcudaMemcpy(?:2D)?Async\(\s*([^,]+),", s)
        dests += re.findall(r"\bcopy_rows\(\s*ctx,\s*([^,]+),", s)
    assert sorted(dests) == sorted(["ctx->d_elig_stage", "ctx->d_created_stage", "ctx->d_gtable", "du", "dp",
                                    "o.dst"]), dests


def test_one_failure_rule_marks_the_scratch_dirty():
    assert sorted(_sites(r"\bmasks_dirty\s*=\s*true\b")) == ["decide", "sync_impl", "sync_impl", "sync_impl"]
    assert _sites(r"\bdecide_impl\s*\(") == ["decide_impl", "decide"]
