"""Race detection for the reader/device/writer pipeline of fastmap, aln, samse, sampe and pemerge (bb_pipe_run, bb_util.c) and
for the single-slot mailbox it shares with `mem`: tests/pipe_check.c, built with bb_util.c under ThreadSanitizer, runs thousands
of items through the pipeline (groups cut into batches, batches dropped or cut again) and closes one mailbox on several
consumers.  It checks order, counts and busy times itself; no ThreadSanitizer report may appear."""
import os
import subprocess

import pytest

from conftest import ROOT

HOST = os.path.join(ROOT, "bwa_b200", "csrc", "host")


def _tsan_cc():
    """The Makefile's tsan target: a compiler whose installation ships libtsan"""
    return "/usr/bin/gcc" if os.access("/usr/bin/gcc", os.X_OK) else os.environ.get("CC", "gcc")


def test_pipeline_is_race_free(tmp_path):
    exe = str(tmp_path / "pipe_check")
    r = subprocess.run([_tsan_cc(), "-fsanitize=thread", "-O1", "-g", "-Wall", "-Iinclude", "-I" + HOST, "-pthread", "-o", exe,
                        os.path.join(ROOT, "tests", "pipe_check.c"), os.path.join(HOST, "bb_util.c"), "-lm", "-lpthread"],
                       cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    if r.returncode != 0:
        pytest.skip("ThreadSanitizer build not available: " + r.stdout.decode()[-300:])
    p = subprocess.run([exe], stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=300)
    err = p.stderr.decode()
    assert p.returncode == 0, err[-3000:]
    assert "ThreadSanitizer" not in err, err[-3000:]
    assert b"pipe: " in p.stdout and b"mbox: " in p.stdout
