"""The traceback of the checkpoint aligner (vsearch_b200/csrc/tb_ckpt.h: direction bits regenerated tile by tile
from the forward pass's H/E/F checkpoints) compiled for the HOST and checked against the oracle over checkpoints
in the device layout, written by a scalar model of nw_ckpt_kernel under its shifted scoring
(tools/ckpt_host_check.cpp).  CPU only: it pins the algorithm and the layout, the GPU tests pin the kernels."""
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    import checkers
    checkers.oracle()   # builds oracle/liboracle.so if needed
    path = str(tmp_path_factory.mktemp("ckpt") / "ckpt_host_check")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I", os.path.join(ROOT, "oracle"),
                           os.path.join(ROOT, "tools", "ckpt_host_check.cpp"), "-L", os.path.join(ROOT, "oracle"),
                           "-loracle", "-Wl,-rpath," + os.path.join(ROOT, "oracle"), "-o", path])
    return path


def run(exe, *args):
    """the tool's summary line as (pairs checked, longest target, lowest shifted score, highest score), after
    asserting that no pair differed from the oracle"""
    r = subprocess.run([exe] + [str(a) for a in args], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and " 0 mismatches" in r.stdout, r.stdout + r.stderr
    m = re.search(r"(\d+) pairs checked, 0 mismatches \(longest target (\d+), lowest shifted score (-?\d+), "
                  r"highest score (-?\d+)\)", r.stdout)
    assert m, r.stdout
    return tuple(int(x) for x in m.groups())


def test_host_device_checkpoint_traceback_matches_oracle(exe):
    checked, longest, _, _ = run(exe, 500)
    assert checked > 900 and longest <= 300


def test_checkpoint_traceback_on_long_targets(exe):
    """default penalties, targets up to the checkpoint kernels' bound (10 353 nt at 16 rows per lane, 10 833 at one):
    the query at the start, end or middle, so the walk crosses hundreds of regenerated tiles along an end gap"""
    checked, longest, low, _ = run(exe, 40, 65535, "long")
    assert checked >= 70 and longest > 10300 and low < -15000


def test_checkpoint_traceback_at_the_16bit_limits(exe):
    """harsh penalties and match 60 / 64 at Q = 32 R, both targets at the bound: the shifted scores approach the
    16-bit floor and the unshifted ones its ceiling"""
    checked, _, low, high = run(exe, 30, 65535, "limits")
    assert checked >= 50 and low < -25000 and high > 25000
