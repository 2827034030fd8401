"""CPU tests of the device math harness (tests/devmath, used by tests/test_zz_devmath_gpu.py): it compiles for sm_90a with
the product's nvcc flags, and its host half -- glibc, the host-compiled restatements and the comparison -- reports no
mismatch where there is none and exactly the input where there is one."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT

DEVMATH = os.path.join(ROOT, "tests", "devmath")
EXPF, LOGF, SINF, COSF, ACOSF, ATANF, PHI_COS, PHI_SIN = range(8)
GLIBC, HOST = 0, 1


class Report(C.Structure):
    _fields_ = [("checked", C.c_uint64), ("mismatches", C.c_uint64), ("n_first", C.c_int32), ("pad", C.c_int32),
                ("input", C.c_uint64 * 16), ("got", C.c_uint64 * 16), ("want", C.c_uint64 * 16)]


@pytest.fixture(scope="module")
def built(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("devmath") / "libdevmath.so")
    r = subprocess.run(["make", "-C", DEVMATH, "OUT=" + out], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    return out


def test_harness_compiles_for_sm90a_with_the_product_flags(built):
    mk = open(os.path.join(ROOT, "pbrt-v3-distributed_b200", "csrc", "nvflags.mk")).read()
    assert "-fmad=false" in mk and "code=sm_90a" in mk and "use_fast_math" not in mk
    log = open(built + ".ptxas.log").read()
    assert "for 'sm_90a'" in log and "k_unary" in log and "k_composite" in log, log[-2000:]
    cuobjdump = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
    if os.path.exists(cuobjdump):
        r = subprocess.run([cuobjdump, "--list-elf", built], capture_output=True, text=True)
        assert "sm_90a" in r.stdout, r.stdout


@pytest.fixture(scope="module")
def dm(built):
    lib = C.CDLL(built)
    u64, vp = C.c_uint64, C.c_void_p
    lib.dm_host_unary.argtypes = [C.c_int, C.c_int, u64, u64, vp]
    lib.dm_compare.argtypes = [vp, vp, u64, C.c_int, u64, u64, C.POINTER(Report)]
    return lib


def host(dm, f, ref, start, n):
    out = np.zeros(n, np.uint64 if f in (PHI_COS, PHI_SIN) else np.uint32)
    assert dm.dm_host_unary(f, ref, start, n, out.ctypes.data) == 0
    return out


def compare(dm, got, want, start):
    rep = Report()
    dm.dm_compare(got.ctypes.data, want.ctypes.data, len(got), int(got.dtype == np.uint64), start, 1, C.byref(rep))
    return rep


CASES = [(EXPF, 0x42a00000), (LOGF, 0x00000000), (ATANF, 0x3ee00000), (SINF, 0x40800000), (COSF, 0xc0400000),
         (ACOSF, 0xbf000000), (PHI_COS, 0x3f000000), (PHI_SIN, 0x3e800000)]


@pytest.mark.parametrize("f,start", CASES, ids=["expf", "logf", "atanf", "sinf", "cosf", "acosf", "cos_phi", "sin_phi"])
def test_host_half_reports_nothing_for_equal_outputs_and_exactly_a_flipped_bit(dm, f, start):
    n = 1 << 20
    want = host(dm, f, GLIBC, start, n)
    got = host(dm, f, HOST, start, n)
    rep = compare(dm, got, want, start)
    assert (rep.checked, rep.mismatches, rep.n_first) == (n, 0, 0)
    k = 12345
    got[k] ^= 1
    rep = compare(dm, got, want, start)
    assert (rep.mismatches, rep.n_first) == (1, 1)
    assert (rep.input[0], rep.got[0], rep.want[0]) == (start + k, int(got[k]), int(want[k]))


def test_host_half_passes_nan_against_nan_only(dm):
    want = np.array([0x7fc00000, 0x7fc00000, 0x3f800000], np.uint32)
    got = np.array([0xffc00001, 0x3f800000, 0x3f800000], np.uint32)  # NaN payloads differ: passes; NaN vs 1.0: fails
    rep = compare(dm, got, want, 100)
    assert (rep.mismatches, rep.input[0]) == (1, 101)


def test_host_build_gives_the_tr_sample11_known_answers(dm):
    """The host build's slopes for the normal-incidence rows of tests/test_zz_devmath_gpu.py (TR11_KNOWN): glibc's."""
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from test_zz_devmath_gpu import TR11, TR11_KNOWN, WORDS
    fp = C.POINTER(C.c_float)
    dm.dm_host_composite.argtypes = [C.c_int, fp, fp, C.c_uint64, fp, C.c_uint64, C.c_uint64, C.c_void_p]
    for u1, u2, sx, sy in TR11_KNOWN:
        prm = np.zeros(8, np.float32)
        prm[0] = 1.0
        ax, ay = np.array([u1], np.uint32).view(np.float32), np.array([u2], np.uint32).view(np.float32)
        out = np.zeros(WORDS, np.uint32)
        assert dm.dm_host_composite(TR11, prm.ctypes.data_as(fp), ax.ctypes.data_as(fp), 1, ay.ctypes.data_as(fp), 0, 1,
                                    out.ctypes.data) == 0
        assert (int(out[0]), int(out[1])) == (sx, sy)
