"""The C++ drop-in boundary: include/ORBextractor.h + include/ORBmatcher.h and the facades in
orb_slam_b200/host/ compile against a minimal cv::/Frame stub and link against liborbfe.so; the call
expressions of Frame.cc / Tracking.cc / MapPoint.cc are reproduced in tests/stubs/conformance.cc."""
import os
import subprocess

import pytest

import orb_slam_b200 as fe

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _build(tmp_path):
    """Links the conformance program into the test's temporary directory: the source tree may be read-only."""
    exe = str(tmp_path / "conformance.bin")
    srcs = [os.path.join(ROOT, "tests", "stubs", "conformance.cc"),
            os.path.join(ROOT, "orb_slam_b200", "host", "ORBextractor.cc"),
            os.path.join(ROOT, "orb_slam_b200", "host", "ORBmatcher.cc")]
    so_dir = os.path.dirname(fe.library_path())
    cmd = ["g++", "-std=c++11", "-O1", "-Wall", "-ffp-contract=off",
           "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "tests", "stubs"),
           "-I", os.path.join(ROOT, "tests", "stubs", "slam")] + srcs + \
          ["-L", so_dir, "-lorbfe", "-Wl,-rpath," + so_dir, "-o", exe]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    return exe


def test_facades_compile_and_link(tmp_path):
    exe = _build(tmp_path)
    r = subprocess.run([exe], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300)
    assert r.returncode == 0, r.stdout
    assert "conformance:" in r.stdout


@pytest.mark.gpu
def test_facades_run_on_gpu(gpu_required, tmp_path):
    exe = _build(tmp_path)
    r = subprocess.run([exe], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300)
    assert r.returncode == 0, r.stdout
    assert "conformance: run ok" in r.stdout
