"""Sweeps of the golden scene set against the oracle under the other integrators and spectrum types: every golden scene
with 60-bin SampledSpectrum and in fog under volpath, the film options that look at a sample's luminance in both spectrum
builds, and the 60-bin and volpath renders over many small batches.  The same functions serve the H100 (pkg / ctx) and
the CPU check build (tests/test_hostcheck.py passes the check library); on the H100 they put the nvcc-compiled 60-bin
and medium kernels, and k_trace2 under them for the instanced scenes, on every scene of the set."""
import json
import os

import numpy as np
import pytest

import test_zz_spectral_gpu as GS
import test_zz_volpath_gpu as GV
from conftest import GOLDEN, bits
from render_cases import EXTRA, RENDERS
from test_gpu_parity import ctx  # noqa: F401  (module-scoped context fixture)

pytestmark = pytest.mark.gpu


def no_overflows(st):
    assert st["stack_overflows"] == 0 and st["dimension_overflows"] == 0, st


@pytest.mark.parametrize("spectral", [False, True])
def test_sample_clamp_crop_and_scale_vs_oracle(pkg, abi, scenes, ob, ctx, spectral):
    """Film options that look at the sample's luminance -- "maxsampleluminance" (film.h:124-125, y() of the sample: the
    60-bin y() rounds differently from ToXYZ's Y) --, a crop window and the film scale, box and Gaussian filter."""
    tables = json.load(open(os.path.join(GOLDEN, "spectral_tables.json"))) if spectral else None
    arr = scenes.SceneArrays(3000, materials=("matte", "glass", "metal", "plastic"), soup_version=1)
    if spectral:
        arr.attach_spectral(tables)
    scene = pkg.Scene(ctx, arr.desc(), keepalive=arr)
    o = ob.Oracle(abi, arr, spectral_tables=tables)
    for kw in (dict(max_sample_luminance=3.0, film_scale=0.5, crop_window=(0.1, 0.9, 0.2, 0.8)),
               dict(max_sample_luminance=1.5, pixel_filter="gaussian")):
        setup = scenes.RenderSetup(48, 32, 8, max_depth=5, strategy=abi.LIGHTS_UNIFORM, **kw)
        film, _ = o.render(setup, threads=4)
        r = pkg.Render(scene, setup)
        r.render_tiles()
        assert np.array_equal(bits(r.read_raw()), bits(film))
        assert np.array_equal(bits(r.read_rgb()), bits(o.film_rgb(setup, film)))
        no_overflows(r.stats())
        clamped = float(np.nan_to_num(r.read_rgb()).max())
        r.close()
        r2 = pkg.Render(scene, scenes.RenderSetup(48, 32, 8, max_depth=5, strategy=abi.LIGHTS_UNIFORM,
                                                   **{k: v for k, v in kw.items() if k != "max_sample_luminance"}))
        r2.render_tiles()
        assert float(np.nan_to_num(r2.read_rgb()).max()) > clamped  # the clamp really was active
        r2.close()
    scene.close()
    o.close()


@pytest.mark.parametrize("name", sorted(RENDERS))
def test_every_golden_scene_under_sampled_spectrum_vs_oracle(pkg, abi, scenes, ob, ctx, name):
    """Every scene of the RGB golden set again with a SampledSpectrum host (where the fixtures hold its spectra): the 60-bin
    kernels against the 60-bin oracle (itself pinned against the SampledSpectrum reference on seven of these scenes)."""
    tables = json.load(open(os.path.join(GOLDEN, "spectral_tables.json")))
    nt, mats, w, h, spp, depth, strat, nl = RENDERS[name]
    ex = EXTRA.get(name, {})
    arr = scenes.SceneArrays(nt, materials=mats, soup_version=1, n_lights=nl, **ex.get("scene", {}))
    try:
        arr.attach_spectral(tables)
    except KeyError as e:
        pytest.skip("no 60-bin fixture: %s" % e)
    setup = scenes.RenderSetup(w, h, spp, max_depth=depth, strategy=getattr(abi, GV.STRATEGY[strat]), **ex.get("camera", {}))
    o = ob.Oracle(abi, arr, spectral_tables=tables)
    film, ostats = o.render(setup, threads=4)
    scene = pkg.Scene(ctx, arr.desc(), keepalive=arr)
    r = pkg.Render(scene, setup)
    r.render_tiles()
    assert np.array_equal(bits(r.read_raw()), bits(film))
    st = r.stats()
    # (MIS rays towards a sphere light that miss the sphere are not traced on the device -- Sphere::Pdf is non-zero for
    # them, the reference traces them in vain --, so "regular" rays are only bounded)
    assert st["camera_rays"] == ostats["camera_rays"] and st["shadow_rays"] == ostats["shadow_rays"]
    assert st["regular_rays"] <= ostats["regular_rays"]
    no_overflows(st)
    r.close()
    scene.close()
    o.close()


@pytest.mark.parametrize("name", sorted(RENDERS))
def test_every_golden_scene_in_fog_under_volpath_vs_oracle(pkg, abi, scenes, ob, ctx, name):
    """Every scene of the golden set again with `Integrator "volpath"` inside a homogeneous medium: the medium pass meets
    every shape, light, sampler, filter and camera option of the set; device against the oracle's VolPathLi (itself
    pinned against the reference's volpath on four of these scenes)."""
    fog = dict(sigma_a=(0.04, 0.06, 0.08), sigma_s=(0.25, 0.2, 0.3), g=0.35)
    nt, mats, w, h, spp, depth, strat, nl = RENDERS[name]
    ex = EXTRA.get(name, {})
    arr = scenes.SceneArrays(nt, materials=mats, soup_version=1, n_lights=nl, **ex.get("scene", {}))
    setup = scenes.RenderSetup(w, h, spp, max_depth=depth, strategy=getattr(abi, GV.STRATEGY[strat]), integrator="volpath",
                               medium=fog, **ex.get("camera", {}))
    o = ob.Oracle(abi, arr)
    ob.set_volpath(o.lib, True, fog)
    try:
        film, ostats = o.render(setup, threads=4)
    finally:
        ob.set_volpath(o.lib, False)
    scene = pkg.Scene(ctx, arr.desc(), keepalive=arr)
    r = pkg.Render(scene, setup)
    r.render_tiles()
    assert np.array_equal(bits(r.read_raw()), bits(film))
    st = r.stats()
    assert st["camera_rays"] == ostats["camera_rays"]
    no_overflows(st)
    r.close()
    scene.close()
    o.close()


def test_new_paths_in_several_batches(pkg, abi, scenes, ob, ctx, monkeypatch):
    """The 60-bin state arrays are planar [bin][capacity] and the medium pass shares the per-slot direct-lighting records
    with the shading kernels: render with a capacity of three tiles per batch (many batches) and compare as before."""
    monkeypatch.setenv("B200PT_BATCH_PATHS", str(256 * 8 * 3))
    GS.test_spectral_render_and_counters_vs_oracle(pkg, abi, scenes, ob, ctx, ("matte", "glass", "metal", "plastic"), 8, "power", None)
    GV.test_volpath_render_vs_oracle(pkg, abi, scenes, ob, ctx, ("matte", "plastic"), 12, "uniform",
                                     dict(sigma_a=(0.2, 0.2, 0.2), sigma_s=(1.5, 1.2, 0.9), g=-0.5), {})
    GS.test_spectral_volpath_render_vs_sampled_spectrum_reference(pkg, abi, scenes, ob, ctx, "spectral_volpath_fog", "volpath_fog")
