"""GPU tests: the path's scalar math as nvcc compiles it for the H100 (tests/devmath/libdevmath.so, built by build() with
the product's flags) against the host's glibc -- what the reference calls -- or against the host-compiled build of the
same headers, bit for bit (both NaN also passes: NaN payloads differ between the device and x86).  Renders reach these
functions only 10^4..10^5 times per scene, far too rarely to show a last-bit difference in a sampled direction.

Also the device-only branches of the sample generators through the C ABI: Sobol' with its byte tables (and without,
B200PT_NO_SOBOL_TABLE) at indices that set every byte and bits >= 40, and Halton's __brev dimension at indices >= 2^32,
against the oracle."""
import ctypes as C
import os
import struct

import numpy as np
import pytest

from conftest import ROOT, bits

pytestmark = pytest.mark.gpu

# B200PT_DEVMATH_LIB: the same harness built against another copy of the headers (tests/devmath/Makefile CSRC=)
LIB = os.environ.get("B200PT_DEVMATH_LIB") or os.path.join(ROOT, "tests", "devmath", "libdevmath.so")
EXPF, LOGF, SINF, COSF, ACOSF, ATANF, PHI_COS, PHI_SIN = range(8)
GLIBC, HOST = 0, 1
DISK, HG, TR11, TR_WH, SPHDIR, SPH_AREA, SPH_CONE, DISCRETE, HALTON = range(9)
WORDS = 8


class Report(C.Structure):
    _fields_ = [("checked", C.c_uint64), ("mismatches", C.c_uint64), ("n_first", C.c_int32), ("pad", C.c_int32),
                ("input", C.c_uint64 * 16), ("got", C.c_uint64 * 16), ("want", C.c_uint64 * 16)]

    def describe(self, wide=False):
        w = 16 if wide else 8
        rows = ["input 0x%x: device 0x%0*x, expected 0x%0*x" % (self.input[i], w, self.got[i], w, self.want[i])
                for i in range(self.n_first)]
        return "%d of %d differ; first: %s" % (self.mismatches, self.checked, "; ".join(rows))


@pytest.fixture(scope="module")
def dm():
    assert os.path.exists(LIB), "%s is missing: build() compiles it (tests/devmath/Makefile)" % LIB
    lib = C.CDLL(LIB)
    u64, vp, fp = C.c_uint64, C.c_void_p, C.POINTER(C.c_float)
    lib.dm_check_unary.argtypes = [C.c_int, C.c_int, u64, u64, C.POINTER(Report)]
    lib.dm_check_atan2.argtypes = [C.c_int, fp, fp, u64, u64, C.POINTER(Report)]
    lib.dm_check_composite.argtypes = [C.c_int, fp, fp, u64, fp, u64, C.POINTER(Report), vp, u64]
    return lib


def f32bits(x):
    return struct.unpack("<I", struct.pack("<f", x))[0]


def fp(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def unary(dm, f, ref, *ranges):
    rep = Report()
    for lo, hi in ranges:
        assert dm.dm_check_unary(f, ref, lo, hi, C.byref(rep)) == 0
    return rep


NEG = 0x80000000


@pytest.mark.parametrize("f", [EXPF, LOGF, ATANF], ids=["expf", "logf", "atanf"])
def test_expf_logf_atanf_equal_glibc_on_every_float(dm, f):
    rep = unary(dm, f, GLIBC, (0, 1 << 32))
    assert rep.checked == 1 << 32
    assert rep.mismatches == 0, rep.describe()


@pytest.mark.parametrize("f", [SINF, COSF], ids=["sinf", "cosf"])
def test_sinf_cosf_equal_glibc_below_8(dm, f):
    """Every float with |x| < 8 (+-0 and subnormals included): the path passes |x| <= 2 pi."""
    b8 = f32bits(8.0)
    rep = unary(dm, f, GLIBC, (0, b8), (NEG, NEG + b8))
    assert rep.mismatches == 0, rep.describe()


@pytest.mark.parametrize("f", [SINF, COSF], ids=["sinf", "cosf"])
def test_sinf_cosf_equal_the_host_build_below_120(dm, f):
    b120 = f32bits(120.0)
    rep = unary(dm, f, HOST, (0, b120), (NEG, NEG + b120))
    assert rep.mismatches == 0, rep.describe()


def test_acosf_equals_glibc_on_minus_one_to_one(dm):
    one = f32bits(1.0)
    rep = unary(dm, ACOSF, GLIBC, (0, one + 1), (NEG, NEG + one + 1),  # [-1, 1]
                (one + 1, one + 4097), (NEG + one + 1, NEG + one + 4097),  # just outside: NaN
                (0x7f800000, 0x7f800002), (0xff800000, 0xff800002), (0x7fc00000, 0x7fc00001))
    assert rep.mismatches == 0, rep.describe()


def atan2_structured():
    """+-0, +-inf, NaN, y = +-x, |y / x| = 2^+-30 and its neighbours, subnormal operands, against assorted values."""
    tiny, sub = np.float32(2.0 ** -149), np.float32(2.0 ** -130)
    base = [0.0, -0.0, np.inf, -np.inf, np.nan, 1.0, -1.0, 0.5, 3.0, -7.25, 1e-30, 1e30, tiny, -tiny, sub, -sub,
            np.float32(np.finfo(np.float32).tiny), np.finfo(np.float32).max]
    ys, xs = [], []
    for y in base:
        for x in base:
            ys.append(y)
            xs.append(x)
    rng = np.random.default_rng(5)
    for x in rng.uniform(-4, 4, 2000).astype(np.float32).tolist() + [1.0, -1.0, 2.0 ** -126, 3.0e38]:
        for s in (1.0, -1.0):
            ys.append(s * x)  # y = +-x
            xs.append(x)
            for e in (30, -30, 60, -60, 61, -61):  # |y / x| = 2^e: atan2f's k > 60 / k < -60 cut-offs and the ratio path
                for nb in (-1, 0, 1):
                    if abs(s * x * 2.0 ** e) < 3e38:
                        y = np.float32(s * x * 2.0 ** e)
                        ys.append(float(np.nextafter(y, np.float32(np.inf) * nb)) if nb else float(y))
                        xs.append(x)
    return np.array(ys, np.float32), np.array(xs, np.float32)


def test_atan2f_equals_glibc(dm):
    rep = Report()
    assert dm.dm_check_atan2(GLIBC, None, None, 17, 200_000_000, C.byref(rep)) == 0
    ys, xs = atan2_structured()
    assert dm.dm_check_atan2(GLIBC, fp(ys), fp(xs), 0, len(ys), C.byref(rep)) == 0
    assert rep.mismatches == 0, rep.describe()


@pytest.mark.parametrize("f", [PHI_COS, PHI_SIN], ids=["cos", "sin"])
def test_double_cos_sin_of_every_tr_sample11_phi_equal_glibc(dm, f):
    """tr_sample11's normal-incidence branch: cos / sin((double)phi), phi = (float)(6.28318530718 * (double)U2), for every
    float U2 in [0, 1) (1 065 353 216 values), against the 64 bits of glibc's ::cos / ::sin."""
    rep = unary(dm, f, GLIBC, (0, f32bits(1.0)))
    assert rep.checked == 1065353216
    assert rep.mismatches == 0, rep.describe(wide=True)


# ---------------------------------------------------------------------------------------------------- composites
ONE_MINUS_EPS = float.fromhex("0x1.fffffep-1")  # PT_ONE_MINUS_EPS


def axis():
    """4096 values in [0, 1): the edges, then a stratified set."""
    edges = [0.0, 2.0 ** -149, 2.0 ** -24, float(np.nextafter(np.float32(0.5), np.float32(0))), 0.5,
             float(np.nextafter(np.float32(0.5), np.float32(1))), ONE_MINUS_EPS, 0.25, 0.75, 2.0 ** -126]
    n = 4096 - len(edges)
    rng = np.random.default_rng(3)
    rest = ((np.arange(n) + rng.uniform(0, 1, n)) / n).astype(np.float32)
    return np.clip(np.concatenate([np.array(edges, np.float32), rest]), 0, np.float32(ONE_MINUS_EPS))


def around(x, k):
    """The 2k + 1 floats centred on float32(x)."""
    v = np.float32(x)
    out = [v]
    up = dn = v
    for _ in range(k):
        up, dn = np.nextafter(up, np.float32(2)), np.nextafter(dn, np.float32(-2))
        out += [up, dn]
    return sorted(float(t) for t in out)


COMPOSITES = ([(DISK, [], "concentric_sample_disk")] +
              [(HG, [g, 0.3, -0.5, 0.81], "hg_sample_p g=%g" % g) for g in (0.0, 1e-4, -1e-4, 0.4, -0.4, 0.95, -0.95)] +
              [(TR11, [c], "tr_sample11 cosTheta=%a" % c) for c in around(0.9999, 3) + [1.0, 0.5]] +
              [(TR_WH, [0.25, 0.25, 0, 0, 1], "tr_sample_wh normal"), (TR_WH, [0.3, 0.1, 0.2, -0.4, 0.9], "tr_sample_wh"),
               (TR_WH, [0.5, 0.5, 0.3, 0.3, -0.9], "tr_sample_wh flipped"),
               (SPHDIR, [0.2, -0.7, 0.4], "spherical_direction"),
               (SPH_AREA, [1.0, -2.0, 0.5, 0.75], "sphere_sample_area"),
               (SPH_CONE, [1.0, -2.0, 0.5, 0.75, -3.0, 4.0, 2.5], "sphere_sample cone"),
               (DISCRETE, [], "sample_discrete")] +
              [(HALTON, [b], "halton_radical_inverse base %d" % b) for b in (3, 7, 61)])


@pytest.mark.parametrize("which,params,name", COMPOSITES, ids=[c[2] for c in COMPOSITES])
def test_sampling_helpers_equal_the_host_build(dm, which, params, name):
    """2^24 (u0, u1) grid points, edges 0, 2^-149, 2^-24, 0.5 +- 1 ulp and PT_ONE_MINUS_EPS included."""
    ax = axis()
    prm = np.zeros(8, np.float32)
    prm[:len(params)] = params
    rep = Report()
    assert dm.dm_check_composite(which, fp(prm), fp(ax), len(ax), fp(ax), len(ax), C.byref(rep), None, 0) == 0
    assert rep.checked == len(ax) ** 2 * WORDS
    assert rep.mismatches == 0, name + ": " + rep.describe()


# tr_sample11 at normal incidence (cosTheta = 1): (U1, U2) bits and the host build's (glibc's) slope bits.  libdevice's
# double cos differs from glibc's by one unit at these phi, and r * cos lies on a float rounding boundary, so a device
# build that called libdevice's cos returned slope_x one float off (0x3f6c9bfb, 0x3f9efe23).
TR11_KNOWN = [(0x3ef99996, 0x3d53da41, 0x3f6c9bfa, 0x3e9f702f), (0x3f2377f1, 0x3d6d3171, 0x3f9efe24, 0x3ef22e36)]


@pytest.mark.parametrize("u1,u2,sx,sy", TR11_KNOWN, ids=["U2=%08x" % k[1] for k in TR11_KNOWN])
def test_tr_sample11_normal_incidence_known_answers(dm, u1, u2, sx, sy):
    prm = np.zeros(8, np.float32)
    prm[0] = 1.0
    ax, ay = np.array([u1], np.uint32).view(np.float32), np.array([u2], np.uint32).view(np.float32)
    got = np.zeros(WORDS, np.uint32)
    rep = Report()
    assert dm.dm_check_composite(TR11, fp(prm), fp(ax), 1, fp(ay), 1, C.byref(rep), got.ctypes.data, 1) == 0
    assert (int(got[0]), int(got[1])) == (sx, sy), "device slopes 0x%08x 0x%08x" % (got[0], got[1])
    assert rep.mismatches == 0, rep.describe()


# ---------------------------------------------------------------------------------------------------- samplers
@pytest.fixture(scope="module")
def ctx(pkg):
    c = pkg.Context(0)
    yield c
    c.close()


@pytest.mark.parametrize("table", [True, False], ids=["byte-table", "bit-loop"])
def test_sobol_at_indices_beyond_the_golden_probe(pkg, abi, scenes, ctx, ob, monkeypatch, table):
    """A 64k x 64k sample-bound (2^32 pixel indices) on a 16 x 16 film, 16 spp (the sample number passed to debug_sobol
    is not limited by it): the pixel fills the low four index bytes, the sample number byte 4 and the bits 40..51 that
    the byte tables leave to the bit loop."""
    if not table:
        monkeypatch.setenv("B200PT_NO_SOBOL_TABLE", "1")
    arr = scenes.SceneArrays(10, materials=("matte",), soup_version=1)
    scene = pkg.Scene(ctx, arr.desc(), keepalive=arr)
    oracle = ob.Oracle(abi, arr)
    setup = scenes.RenderSetup(16, 16, 16, max_depth=4)
    sb = [0, 0, 1 << 16, 1 << 16]
    setup.sampler.sample_bounds[:] = sb
    setup._sobol_tables(sb)
    r = pkg.Render(scene, setup)
    n = setup.sampler.n_dimensions
    for px, py in ((0xabcd, 0x7531), (0xffff, 0xffff), (1, 0x8000)):
        for sample in (0, 1, 0xff, 0x1234, 0xabcde, (1 << 20) - 1, 1 << 19):  # indices < 2^52, the matrices' size
            got = r.debug_sobol(px, py, sample, 0, n)
            want = oracle.sobol(setup, px, py, sample, 0, n)
            assert np.array_equal(bits(got), bits(want)), (px, py, sample)
    r.close()
    scene.close()
    oracle.close()


def test_halton_at_indices_beyond_2_pow_32(pkg, abi, scenes, ctx, ob):
    """Halton's dimension 0 reverses the index bits with __brev on the device; indices >= 2^32 (and >= 2^39, so that the
    shifted index still has bits above 32) against the oracle."""
    arr = scenes.SceneArrays(10, materials=("matte",), soup_version=1)
    scene = pkg.Scene(ctx, arr.desc(), keepalive=arr)
    oracle = ob.Oracle(abi, arr)
    setup = scenes.RenderSetup(16, 16, 16, max_depth=4, sampler="halton")
    setup.sampler.sample_bounds[:] = [0, 0, 1024, 1024]
    r = pkg.Render(scene, setup)
    n = min(setup.sampler.n_dimensions, 64)
    for px, py in ((5, 7), (1000, 3), (127, 1023)):
        for sample in (0, 1, 140_000, 1 << 24, 123_456_789, (1 << 30) - 1):
            got = r.debug_sobol(px, py, sample, 0, n)
            want = oracle.sobol(setup, px, py, sample, 0, n)
            assert np.array_equal(bits(got), bits(want)), (px, py, sample)
    r.close()
    scene.close()
    oracle.close()
