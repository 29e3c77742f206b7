"""The CPU oracle stays defined at the int16 rails.

The device kernels are checked against the oracle bit for bit, so wherever the oracle's C++ overflows a signed integer its answer is
whatever the compiler chose to emit, and agreement with the device means nothing.  The oracle is built here with a trapping signed-
overflow check (-fsanitize=signed-integer-overflow -fsanitize-trap=all: no runtime library needed) and every rail capture of
rail_inputs.py goes through its receive entry points in a subprocess; a trap kills the subprocess with SIGILL."""
import os, re, shlex, subprocess, sys
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE = os.path.join(ROOT, "oracle")


def _make_var(name):
    """A variable of oracle/Makefile (`NAME = ...` or `NAME ?= ...`), so this build uses the same sources and flags."""
    with open(os.path.join(ORACLE, "Makefile")) as f:
        for line in f:
            m = re.match(r"\s*%s\s*\??=\s*(.*)$" % name, line)
            if m: return shlex.split(m.group(1))
    raise KeyError(name)


def test_oracle_has_no_signed_overflow_at_the_rails(tmp_path):
    so = str(tmp_path / "libsora_oracle_trapv.so")
    cxx = os.environ.get("CXX", "g++")
    flags = [f for f in _make_var("CXXFLAGS") if not f.startswith("-W")] + ["-w", "-fsanitize=signed-integer-overflow", "-fsanitize-trap=all"]
    subprocess.run([cxx] + flags + ["-shared", "-o", so] + _make_var("SRC"), cwd=ORACLE, check=True, capture_output=True, timeout=600)
    p = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "rail_inputs.py"), so], capture_output=True, text=True, timeout=600)
    lines = p.stdout.splitlines()
    assert p.returncode == 0 and lines[-1:] == ["done"], \
        f"oracle stopped (exit {p.returncode}) in case {lines[-1] if lines else '?'!r}; stderr: {p.stderr[-400:]}"
