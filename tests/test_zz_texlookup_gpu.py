"""GPU tests: ImageTexture's MIPMap lookups, InfiniteAreaLight's Sample_Li / Pdf_Li / Le, ComputeDifferentials and
RoughnessToAlpha as nvcc compiles them for the H100 (pt_texture.cuh and pt_core.cuh, run by tests/devmath/libdevmath.so
with the product's flags) against the reference's own MIPMap, InfiniteAreaLight, SurfaceInteraction and
TrowbridgeReitzDistribution (oracle/_ref/ref_probe), bit for bit (both NaN also passes).  Where ref_probe is not built
(it needs the reference sources), the device runs over the reference's tables committed in tests/golden/ and is compared
with the host-compiled build of the same functions, which tests/test_texlookup.py pins to the reference's answers.
Renders look a texture up only at a path's first textured hit, about 10^4 times per test scene and almost always in the
common branch; these tests reach every branch's edge (tests/texlookup.py) and at least 10^6 stratified random points per
family."""
import os

import numpy as np
import pytest

from conftest import ROOT
import texlookup as T

pytestmark = pytest.mark.gpu

# B200PT_DEVMATH_LIB: the same harness built against another copy of the headers (tests/devmath/Makefile CSRC=)
LIB = os.environ.get("B200PT_DEVMATH_LIB") or os.path.join(ROOT, "tests", "devmath", "libdevmath.so")


@pytest.fixture(scope="module")
def dm():
    assert os.path.exists(LIB), "%s is missing: build() compiles it (tests/devmath/Makefile)" % LIB
    return T.bind(LIB)


@pytest.fixture(scope="module")
def tmp(tmp_path_factory):
    return str(tmp_path_factory.mktemp("texlookup"))


def assert_clean(res):
    bad = ["%s: %s" % (name, rep.describe(T.OUT_WORDS[fam])) for name, fam, rep in res if rep.mismatches]
    assert all(rep.checked for _, _, rep in res)
    assert not bad, "\n".join(bad[:8])


@pytest.mark.parametrize("w,h,ch,huge", T.mip_cases(), ids=["%dx%d-ch%d%s" % (c[0], c[1], c[2], "-1e37" if c[3] else "")
                                                           for c in T.mip_cases()])
def test_mipmap_lookups_equal_the_reference(dm, tmp, w, h, ch, huge):
    """Three wraps x (EWA at maxAnisotropy 1, 8, 64 and trilinear): 4096 random Lookup(st, dst0, dst1) per setting and
    16384 random Lookup(st, width) per wrap besides the edges; over the 22 maps, 10^6 of each."""
    res, nq = T.run_mip_case(dm, tmp, w, h, ch, huge, T.ON_DEVICE, n_random=4096, n_width=16384)
    assert_clean(res)


@pytest.mark.parametrize("mapname", T.SKY_MAPS)
@pytest.mark.parametrize("xform", T.SKY_XFORMS)
def test_sky_sample_pdf_le_equal_the_reference(dm, tmp, mapname, xform):
    """Sample_Li at every CDF entry and 1 ulp below it and on the 4096 x 4096 grid of the devmath test (1024 x 1024 of
    it under the non-identity transforms), then Pdf_Li and Le at 2^20 random and the edge directions and at every wi
    Sample_Li returned."""
    ax = T.axis() if xform == "identity" else T.axis()[::4]
    res = T.sky_runs(dm, tmp, mapname, xform, T.ON_DEVICE, T.grid(ax, ax), 1 << 20)
    assert_clean(res)


def test_compute_differentials_equals_the_reference(dm, tmp):
    q = T.diff_cases(1 << 21, 7)
    want = T.probe_diff(tmp, q, dm)
    rep = T.Report()
    assert T.check_geom(dm, T.DIFF, q, want, T.ON_DEVICE, rep) == 0
    assert rep.checked == 4 * len(q) and rep.mismatches == 0, rep.describe(4)


def test_roughness_to_alpha_equals_the_reference_on_every_float_in_its_range(dm):
    """Every float in [2^-10, 2) (92 274 688 values), 0, subnormals, -0, negatives, large values, inf and NaN."""
    rep = T.Report()
    for x, want in T.roughness_chunks(T.roughness_ranges(full=True), dm=dm):
        assert T.check_geom(dm, T.ROUGH, x, want, T.ON_DEVICE, rep) == 0
    assert rep.checked > 92274688 and rep.mismatches == 0, rep.describe()
