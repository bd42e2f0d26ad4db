"""CPU tests of orbfe_vocabulary_load_text's argument and header checks (include/orbfe_bow.h): a missing file, a NULL path,
out == NULL and every out-of-range header field are rejected with ORBFE_ERR_ARG and a message, before any device is used, so
they hold on a machine without one."""
import ctypes as C

import pytest

import orb_slam_b200 as fe
from orb_slam_b200 import bow as B


def _load(path, out=True):
    L = B._bind()
    h = C.c_void_p(0x1234)
    rc = L.orbfe_vocabulary_load_text(0, None if path is None else str(path).encode(), C.byref(h) if out else None)
    return rc, h.value


def _last_error():
    return fe.lib().orbfe_last_error().decode()


def test_missing_file(tmp_path):
    rc, h = _load(tmp_path / "absent.txt")
    assert rc == fe.ORBFE_ERR_ARG and h is None
    assert "cannot open" in _last_error() and "absent.txt" in _last_error()


def test_null_path_and_null_out(tmp_path):
    rc, h = _load(None)
    assert rc == fe.ORBFE_ERR_ARG and h is None
    assert "NULL path" in _last_error()
    p = tmp_path / "v.txt"
    p.write_text("10 6 0 0\n")
    rc, _ = _load(p, out=False)
    assert rc == fe.ORBFE_ERR_ARG
    assert "out is NULL" in _last_error()


def test_directory_is_not_a_vocabulary(tmp_path):
    rc, _ = _load(tmp_path)
    assert rc == fe.ORBFE_ERR_ARG
    assert "regular file" in _last_error()


@pytest.mark.parametrize("header, field", [
    ("-1 6 0 0", "k = -1"), ("21 6 0 0", "k = 21"),
    ("10 0 0 0", "L = 0"), ("10 11 0 0", "L = 11"),
    ("10 6 -1 0", "scoring = -1"), ("10 6 6 0", "scoring = 6"),
    ("10 6 0 -1", "weighting = -1"), ("10 6 0 4", "weighting = 4"),
])
def test_out_of_range_header_field(tmp_path, header, field):
    p = tmp_path / "v.txt"
    p.write_text(header + "\n0 1 " + " ".join(["7"] * 32) + " 1.5\n")
    rc, h = _load(p)
    assert rc == fe.ORBFE_ERR_ARG and h is None
    assert "line 1" in _last_error() and field in _last_error()


@pytest.mark.parametrize("header", ["", "10 6 0", "10 6 zero 0", "10 6 0 0.5", "10 6 0 99999999999"])
def test_malformed_header(tmp_path, header):
    p = tmp_path / "v.txt"
    p.write_text(header + "\n")
    rc, h = _load(p)
    assert rc == fe.ORBFE_ERR_ARG and h is None
    assert "line 1" in _last_error() and "four integers" in _last_error()


def test_good_header_reaches_the_device_check(tmp_path):
    """Past the header the loader needs a device: without one the answer is ORBFE_ERR_NO_DEVICE."""
    if fe.lib().orbfe_device_count() > 0:
        pytest.skip("a device is present: the load itself is covered by tests/test_gpu_vocab_text.py")
    p = tmp_path / "v.txt"
    p.write_text("10 6 0 0\n0 1 " + " ".join(["7"] * 32) + " 1.5\n")
    rc, h = _load(p)
    assert rc == fe.ORBFE_ERR_NO_DEVICE and h is None
    assert "no CUDA device" in _last_error()
