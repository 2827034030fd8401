"""CPU test: the __sincostab of pt_sincos_dbl.cuh (glibc's table behind double sin / cos) regenerated with mpmath, and
compared byte for byte with the table in the host's libm.so.6."""
import os
import re
import struct

import pytest

from conftest import ROOT

HDR = os.path.join(ROOT, "pbrt-v3-distributed_b200", "csrc", "pt_sincos_dbl.cuh")


def table():
    src = open(HDR).read()
    body = src[src.index("#define PT_SINCOSTAB_DATA"):src.index("#ifdef __CUDACC__", src.index("#define PT_SINCOSTAB_DATA"))]
    vals = [float.fromhex(t) for t in re.findall(r"-?0x[0-9a-fA-F.]+p[-+]?\d+", body)]
    assert len(vals) == 440
    return vals


def test_table_is_sin_and_cos_of_i_over_128_with_their_remainders():
    mpmath = pytest.importorskip("mpmath")
    mpmath.mp.prec = 300
    tab = table()
    off = 0
    for i in range(110):
        x = mpmath.mpf(i) / 128
        for j, f in ((0, mpmath.sin), (2, mpmath.cos)):
            exact = f(x)
            hi, lo = tab[4 * i + j], tab[4 * i + j + 1]
            assert hi == float(exact), (i, j)  # the leading part is correctly rounded
            rem = exact - hi
            if lo != float(rem):
                off += 1
                assert abs(mpmath.mpf(lo) - rem) < mpmath.mpf(2) ** -106, (i, j)
    assert off == 18  # the remainders glibc's table has off the correctly rounded one (1 to 39 of its units)


def test_table_equals_the_host_libm_bytes():
    libm = next((p for p in ("/lib/x86_64-linux-gnu/libm.so.6", "/usr/lib/x86_64-linux-gnu/libm.so.6", "/lib64/libm.so.6")
                 if os.path.exists(p)), None)
    if libm is None:
        pytest.skip("no x86-64 glibc libm.so.6 on this host")
    data = open(libm, "rb").read()
    packed = struct.pack("<440d", *table())
    at = data.find(packed[32:96])  # entries 1 and 2 are unique in the library; entry 0 is (0, 0, 1, 0)
    assert at >= 32, "the table's entries 1..2 are not in %s" % libm
    assert data[at - 32:at - 32 + len(packed)] == packed
