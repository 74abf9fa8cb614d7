"""`gpu-pruner --late-seconds L` on the command line: it needs -d, L is a whole number below the window, and the help
text lists it.  (What the flag does is checked on the H100 by tests/test_gpu_late_ticks.py.)"""
import subprocess

import pytest

import hostlib as H


def _run(*args):
    p = subprocess.run([H.BIN, *args], capture_output=True, text=True, timeout=60)
    return p.returncode, p.stdout + p.stderr


@pytest.mark.parametrize("args,why", [
    (("--late-seconds", "30"), "can only be used with '--daemon-mode'"),
    (("--late-seconds", "0"), "can only be used with '--daemon-mode'"),
    (("-d", "--late-seconds", "1800"), "must be less than the window"),
    (("-d", "-t", "2", "--late-seconds", "120"), "must be less than the window"),
    (("-d", "--late-seconds", "-5"), "invalid digit"),
    (("-d", "--late-seconds", "1.5"), "invalid digit"),
    (("-d", "--late-seconds", "x"), "invalid digit"),
])
def test_bad_values_exit_2(args, why):
    rc, out = _run(*args, "--prometheus-url", "file:///nonexistent")
    assert rc == 2 and out.startswith("error: ") and why in out, out


def test_a_missing_value_exits_2():
    rc, out = _run("-d", "--prometheus-url", "file:///nonexistent", "--late-seconds")
    assert rc == 2 and "a value is required for '--late-seconds'" in out, out


@pytest.mark.parametrize("L", ["0", "45", "119"])
def test_good_values_parse(L):
    rc, out = _run("-d", "-t", "2", "--late-seconds", L, "--print-query")
    assert rc == 0 and "max_over_time" in out, out


def test_help_lists_the_flag():
    rc, out = _run("--help")
    assert rc == 0
    line = [l for l in out.splitlines() if "--late-seconds" in l]
    assert len(line) == 1 and "with -d" in line[0] and "[default: 0 = off]" in line[0], line
