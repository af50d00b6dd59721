"""gnss_sdr_b200.build redoes a build exactly when its inputs change: the bytes of csrc/ and the header, and the nvcc flags.
File times play no part.  No GPU and no real nvcc: build.NVCC is a stub that logs each call and writes the output file."""
import os
import stat

import pytest

from gnss_sdr_b200 import build as b

STUB = """#!/bin/sh
echo "$@" >> "{log}"
while [ $# -gt 0 ]; do
    if [ "$1" = "-o" ]; then echo stub > "$2"; fi
    shift
done
"""


@pytest.fixture
def tree(tmp_path, monkeypatch):
    """a csrc/ and header of their own, the stub compiler; -> (output path, function counting the stub's calls)"""
    csrc = tmp_path / "csrc"
    csrc.mkdir()
    for name in ("a.cu", "b_nofma.cu", "c.cuh"):
        (csrc / name).write_text(f"// {name}\n")
    header = tmp_path / "b200gnss.h"
    header.write_text("/* header */\n")
    log = tmp_path / "nvcc.log"
    log.write_text("")
    nvcc = tmp_path / "nvcc"
    nvcc.write_text(STUB.format(log=log))
    nvcc.chmod(nvcc.stat().st_mode | stat.S_IXUSR)
    monkeypatch.setattr(b, "NVCC", str(nvcc))
    monkeypatch.setattr(b, "CSRC", str(csrc))
    monkeypatch.setattr(b, "HEADER", str(header))
    monkeypatch.setattr(b, "OBJ_DIR", str(tmp_path / "obj"))
    return str(tmp_path / "lib.so"), lambda: len(log.read_text().splitlines())


def test_touching_every_source_does_not_rebuild(tree):
    out, calls = tree
    b.build(out=out)
    n = calls()
    assert n == 3                                   # two compiles and the link
    later = os.path.getmtime(out) + 100
    for p in [os.path.join(b.CSRC, f) for f in os.listdir(b.CSRC)] + [b.HEADER]:
        os.utime(p, (later, later))
    b.build(out=out)
    assert calls() == n


def test_one_changed_byte_rebuilds(tree):
    out, calls = tree
    b.build(out=out)
    n = calls()
    for path in (os.path.join(b.CSRC, "c.cuh"), b.HEADER):
        with open(path, "r+b") as fh:
            first = fh.read(1)
            fh.seek(0)
            fh.write(b"#" if first != b"#" else b"/")
        b.build(out=out)
        assert calls() == n + 3, path
        n = calls()
        b.build(out=out)
        assert calls() == n


def test_a_different_define_rebuilds(tree):
    out, calls = tree
    b.build(out=out, extra=["-DSH_STAGES=2"])
    n = calls()
    b.build(out=out, extra=["-DSH_STAGES=2"])
    assert calls() == n
    b.build(out=out, extra=["-DSH_STAGES=4"])
    assert calls() == n + 3
