"""CPU tests of the texture half of the devmath harness (tests/devmath/devmath.cu, used on the device by
tests/test_zz_texlookup_gpu.py): the same input sets at reduced size, run host-compiled through the same functions of
pt_texture.cuh and pt_core.cuh, against the reference's own MIPMap, InfiniteAreaLight, ComputeDifferentials and
RoughnessToAlpha (oracle/_ref/ref_probe); the comparison reports exactly the input where an answer differs; the harness
refuses EWA footprints and st it does not accept; the reference's tables committed in tests/golden/ (what the GPU tests use
where ref_probe is not built) are what the reference builds."""
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT
import texlookup as T

needs_probe = pytest.mark.skipif(not os.path.exists(T.PROBE),
                                 reason="oracle/_ref/ref_probe is not built: `make -C oracle ref` needs the reference sources")
DEVMATH = os.path.join(ROOT, "tests", "devmath")


@pytest.fixture(scope="module")
def dm(tmp_path_factory):
    lib = os.environ.get("B200PT_DEVMATH_LIB")
    if not lib:
        lib = str(tmp_path_factory.mktemp("devmath") / "libdevmath.so")
        r = subprocess.run(["make", "-C", DEVMATH, "OUT=" + lib], capture_output=True, text=True)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    return T.bind(lib)


@pytest.fixture(scope="module")
def tmp(tmp_path_factory):
    return str(tmp_path_factory.mktemp("texlookup"))


def assert_clean(res):
    bad = ["%s: %s" % (name, rep.describe(T.OUT_WORDS[fam])) for name, fam, rep in res if rep.mismatches]
    assert all(rep.checked for _, _, rep in res)
    assert not bad, "\n".join(bad[:8])


@needs_probe
@pytest.mark.parametrize("w,h,ch,huge", T.mip_cases(), ids=["%dx%d-ch%d%s" % (c[0], c[1], c[2], "-1e37" if c[3] else "")
                                                           for c in T.mip_cases()])
def test_mipmap_lookups_host(dm, tmp, w, h, ch, huge):
    res, nq = T.run_mip_case(dm, tmp, w, h, ch, huge, T.ON_HOST, n_random=256, n_width=256)
    assert nq > 10000
    assert_clean(res)


@needs_probe
@pytest.mark.parametrize("mapname", T.SKY_MAPS)
@pytest.mark.parametrize("xform", T.SKY_XFORMS)
def test_sky_sample_pdf_le_host(dm, tmp, mapname, xform):
    ax = T.axis()[::64]
    res = T.sky_runs(dm, tmp, mapname, xform, T.ON_HOST, T.grid(ax, ax), 2048)
    assert_clean(res)


@needs_probe
def test_black_sky_samples_have_pdf_zero(tmp):
    sky = T.Sky(tmp, "black", "identity", u=T.grid(T.axis()[::256], T.axis()[::256]))
    a = sky.sample.view(np.float32).reshape(-1, 10)
    assert sky.marg_func_int == 0 and np.all(a == 0)


@needs_probe
def test_sky_tables_have_black_rows(tmp):
    """The hot-texel and top-black maps give Distribution2D rows with funcInt == 0, whose cdf is i / n."""
    for name in ("hot-texel", "top-black"):
        sky = T.Sky(tmp, name, "identity")
        assert np.any(sky.cond_func_int == 0) and np.any(sky.cond_func_int > 0), name


@needs_probe
def test_compute_differentials_host(dm, tmp):
    q = T.diff_cases(1 << 14, 11)
    want = T.probe_diff(tmp, q)
    rep = T.Report()
    assert T.check_geom(dm, T.DIFF, q, want, T.ON_HOST, rep) == 0
    assert rep.checked == 4 * len(q) and rep.mismatches == 0, rep.describe(4)
    a = want.view(np.float32).reshape(-1, 4)
    assert np.any(np.all(a == 0, axis=1)) and np.any(np.all(a != 0, axis=1))  # failed and solved cases both present


@needs_probe
def test_roughness_to_alpha_host(dm):
    rep = T.Report()
    for x, want in T.roughness_chunks(T.roughness_ranges(full=False)):
        assert T.check_geom(dm, T.ROUGH, x, want, T.ON_HOST, rep) == 0
    assert rep.checked > 300000 and rep.mismatches == 0, rep.describe()


@needs_probe
def test_comparison_reports_a_planted_mismatch_at_its_input(dm, tmp):
    """One flipped bit in the reference's answers of each family is reported at exactly that query and word."""
    eq = T.ewa_queries(dm, 8, 4, 8.0, 512, 3)
    m = T.Mip(tmp, T.mip_texels(8, 4, 3, 1), T.REPEAT, False, 8.0, eq, T.width_queries(8, 4, 64, 1))
    sky = T.Sky(tmp, "8x4", "oblique", u=T.grid(T.axis()[::128], T.axis()[::128]), w=T.sky_dirs(256, 1),
                d=T.sky_dirs(256, 2))
    q = T.diff_cases(256, 1)
    dwant = T.probe_diff(tmp, q)
    ((x, rwant),) = T.roughness_chunks([(T.bits_of(0.25), T.bits_of(0.25) + 1000)])
    cases = [(lambda want, rep: m.check(dm, T.EWA, T.ON_HOST, rep, want), m.want(T.EWA)),
             (lambda want, rep: m.check(dm, T.WIDTH, T.ON_HOST, rep, want), m.want(T.WIDTH)),
             (lambda want, rep: sky.check(dm, T.SAMPLE, T.ON_HOST, rep, want), sky.sample),
             (lambda want, rep: sky.check(dm, T.PDF, T.ON_HOST, rep, want), sky.pdf),
             (lambda want, rep: sky.check(dm, T.LE, T.ON_HOST, rep, want), sky.le),
             (lambda want, rep: T.check_geom(dm, T.DIFF, q, want, T.ON_HOST, rep), dwant),
             (lambda want, rep: T.check_geom(dm, T.ROUGH, x, want, T.ON_HOST, rep), rwant)]
    for run, want in cases:
        want = np.array(want, np.uint32).ravel()
        rep = T.Report()
        assert run(want, rep) == 0 and rep.mismatches == 0, rep.describe()
        k = len(want) * 2 // 3
        while want[k] & 0x7fffffff > 0x7f800000:  # a NaN stays NaN with one bit flipped
            k += 1
        want[k] ^= 1
        rep = T.Report()
        assert run(want, rep) == 0
        assert (rep.mismatches, rep.n_first, rep.input[0]) == (1, 1, k)
        assert rep.want[0] == want[k] and rep.got[0] == want[k] ^ 1


@needs_probe
def test_harness_refuses_footprints_and_st_it_does_not_accept(dm, tmp):
    """A long, thin ellipse at the finest level (box > 2^12 texels) and |st * size| >= 2^30: refused (-2) before anything
    runs, the accepted neighbours not."""
    ok = np.array([[0.5, 0.5, 0.001, 0.0, 0.0, 0.001]], np.float32)
    long = np.array([[0.5, 0.5, 0.7, 0.7, -0.7 / 64, 0.7 / 64]], np.float32)
    far = np.array([[2.0 ** 30 / 64, 0.5, 0.001, 0.0, 0.0, 0.001]], np.float32)
    assert T.footprints(dm, 64, 64, 64.0, long)[0] > T.EWA_MAX_TEXELS
    assert T.footprints(dm, 64, 64, 64.0, ok)[0] <= T.EWA_MAX_TEXELS
    tex = T.mip_texels(64, 64, 3, 2)
    for q, rc in ((ok, 0), (long, -2), (far, -2)):
        m = T.Mip(tmp, tex, T.REPEAT, False, 64.0, q, np.zeros((0, 3), np.float32))
        assert m.check(dm, T.EWA, T.ON_HOST, T.Report()) == rc
    wq = np.array([[2.0 ** 30 / 64, 0.5, 0.01]], np.float32)
    m = T.Mip(tmp, tex, T.REPEAT, True, 8.0, np.zeros((0, 6), np.float32), wq)
    assert m.check(dm, T.WIDTH, T.ON_HOST, T.Report()) == -2


@needs_probe
def test_golden_tables_are_what_the_reference_builds(tmp):
    """tests/golden/texlookup_tables.npz equals, bit for bit, what ref_probe builds now (`python tests/texlookup.py`
    regenerates it)."""
    want = T.build_golden(tmp)
    with np.load(T.GOLDEN) as z:
        assert sorted(z.files) == sorted(want)
        for k, v in want.items():
            g = z[k]
            assert g.dtype == v.dtype and g.shape == v.shape, k
            assert np.array_equal(g.view(np.uint8), np.ascontiguousarray(v).view(np.uint8)), k


def test_golden_tables_serve_every_input_set(dm, tmp, monkeypatch):
    """Without ref_probe every MIPMap and sky of the GPU input sets loads from the committed tables and the host-compiled
    build answers (this is the GPU tests' path where the reference sources are absent); with it, the tables agree."""
    monkeypatch.setattr(T, "have_probe", lambda: False)
    q = np.array([[0.3, 0.7, 0.01, 0.0, 0.0, 0.004]], np.float32)
    for (w, h, ch, huge) in T.mip_cases():
        tex = T.mip_texels(w, h, ch, seed=w * 131 + h * 7 + ch, huge=huge)
        for wrap in (T.REPEAT, T.BLACK, T.CLAMP):
            m = T.Mip(tmp, tex, wrap, False, 8.0, q, np.zeros((0, 3), np.float32))
            assert len(m.dims) == len(T.pyramid_dims(w, h)) and m.pyramid.size == sum(a * b for a, b in m.dims) * ch
            rep = T.Report()
            assert m.check(dm, T.EWA, T.ON_HOST, rep) == 0 and rep.checked == 3 and rep.mismatches == 0
    for name in T.SKY_MAPS:
        for x in T.SKY_XFORMS:
            res = T.sky_runs(dm, tmp, name, x, T.ON_HOST, T.grid(T.axis()[::512], T.axis()[::512]), 16)
            assert_clean(res)
    dq = T.diff_cases(16, 3)
    rep = T.Report()
    assert T.check_geom(dm, T.DIFF, dq, T.probe_diff(tmp, dq, dm), T.ON_HOST, rep) == 0 and rep.mismatches == 0
    ((x, want),) = T.roughness_chunks([(T.bits_of(1.0), T.bits_of(1.0) + 64)], dm=dm)
    assert len(want) == 64 and want.view(np.float32)[0] == np.float32(1.62142)  # log(1) = 0: the constant term
