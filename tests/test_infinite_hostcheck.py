"""CPU pre-flight of the infinite-light path (tests/test_zz_infinite_gpu.py) on the check build of the library
(tests/emu: api.cu and kernels.cu compiled as plain C++), and the refusals of the C ABI and of the drop-in binaries,
which need no device."""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

import test_zz_infinite_gpu as I
from conftest import GOLDEN

HC_PLUGIN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu", "pbrt_b200_hostcheck")


@pytest.fixture(scope="module")
def hc_plugin(hostcheck):
    if not (os.path.exists(I.REF) and os.path.exists(I.PLUGIN)):
        pytest.skip("pbrt_ref / pbrt_b200 are built where the reference sources exist")
    r = subprocess.run(["make", "plugins"], cwd=os.path.dirname(HC_PLUGIN), capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    return HC_PLUGIN


@pytest.mark.parametrize("name", sorted(I.CASES))
def test_dropin_infinite_light_on_the_check_library(hc_plugin, scenes, tmp_path, name):
    I.test_dropin_infinite_light_vs_reference(scenes, tmp_path, name, plugin=hc_plugin)


@pytest.mark.parametrize("name", ["const_area", "two_skies_delta"])
def test_harness_infinite_light_on_the_check_library(hc_plugin, hostcheck, abi, scenes, tmp_path, name):
    I.test_harness_infinite_light_vs_reference(hostcheck, abi, scenes, tmp_path, name, plugin=hc_plugin)


def test_known_answer_on_the_check_library(hc_plugin, scenes, tmp_path):
    I.test_known_answer_matte_sphere_under_constant_sky(scenes, tmp_path, plugin=hc_plugin)


def test_dropin_refuses_volpath_and_spectral_hosts_without_a_device(scenes, tmp_path):
    """The refusals come from the host's flattening, before any device is touched: the real binaries show them here."""
    if not os.path.exists(I.PLUGIN):
        pytest.skip("pbrt_b200 is built where the reference sources exist")
    I.test_dropin_refuses_volpath_and_spectral_hosts(scenes, tmp_path)


def _tables(w=8, h=4):
    """A small but well-formed set of InfiniteAreaLight tables (a constant map)."""
    nu, nv = 2 * w, 2 * h
    func = np.ones((nv, nu), np.float32)
    cdf = np.tile(np.linspace(0, 1, nu + 1, dtype=np.float32), (nv, 1))
    return dict(texels=np.ones((h, w, 3), np.float32), light_to_world=np.eye(4, dtype=np.float32).reshape(-1),
                cond_func=func, cond_cdf=cdf, cond_func_int=np.ones(nv, np.float32), marg_func=np.ones(nv, np.float32),
                marg_cdf=np.linspace(0, 1, nv + 1, dtype=np.float32), marg_func_int=1.0, power_rgb=np.ones(3, np.float32))


@pytest.fixture
def hc_scene(hostcheck, scenes):
    """A soup with its area lights, one delta light and one infinite light (the last light) on the check library."""
    ctx = hostcheck.Context(0)
    arr = scenes.SceneArrays(500, materials=("matte", "plastic"), soup_version=1, n_lights=1,
                             delta_lights=[dict(kind="point", from_=(0, 1, -1), I=1.0)], infinite_lights=[dict(L=1.0)])
    scene = hostcheck.Scene(ctx, arr.desc(), keepalive=arr)
    yield hostcheck, arr, scene
    scene.close()
    ctx.close()


def test_set_infinite_light_refuses_bad_descriptors(hc_scene, abi):
    hc, arr, scene = hc_scene
    last = arr.n_lights - 1
    assert arr._lights[last].kind == abi.LIGHT_INFINITE
    for light in (0, last - 1, last + 1, -1):  # an area light, the point light, out of range
        with pytest.raises(hc.B200ptError, match="not an infinite light"):
            scene.set_infinite_light(light, _tables())
    with pytest.raises(hc.B200ptError, match="bad map"):
        scene.set_infinite_light(last, dict(_tables(), texels=np.ones((0, 8, 3), np.float32)))
    rec = abi.InfiniteLight()
    rec.width, rec.height, rec.nu, rec.nv = 8, 4, 16, 8  # sizes, but no tables
    assert hc.lib.b200pt_scene_set_infinite_light(scene.h, last, C.byref(rec)) == -1
    assert "NULL" in hc.lib.b200pt_last_error().decode()
    rec.width = -8
    assert hc.lib.b200pt_scene_set_infinite_light(scene.h, last, C.byref(rec)) == -1
    assert hc.lib.b200pt_scene_set_infinite_light(scene.h, last, None) == -1


def test_render_create_refuses_unset_maps_and_volpath(hc_scene, scenes):
    hc, arr, scene = hc_scene
    with pytest.raises(hc.B200ptError, match="has no map"):
        hc.Render(scene, scenes.RenderSetup(16, 16, 1))
    scene.set_infinite_light(arr.n_lights - 1, _tables())
    with pytest.raises(hc.B200ptError, match="volumetric integrator"):
        hc.Render(scene, scenes.RenderSetup(16, 16, 1, integrator="volpath"))
    r = hc.Render(scene, scenes.RenderSetup(16, 16, 1))  # with the map set, PathIntegrator renders
    r.render_tiles()
    assert np.isfinite(r.read_rgb()).all()
    r.close()


def test_render_create_refuses_sampled_spectrum_hosts(hostcheck, scenes):
    tables = json.load(open(os.path.join(GOLDEN, "spectral_tables.json")))
    arr = scenes.SceneArrays(500, materials=("matte", "plastic"), soup_version=1, n_lights=1,
                             infinite_lights=[dict(L=1.0)]).attach_spectral(tables)
    ctx = hostcheck.Context(0)
    scene = hostcheck.Scene(ctx, arr.desc(), keepalive=arr)
    scene.set_infinite_light(arr.n_lights - 1, _tables())
    with pytest.raises(hostcheck.B200ptError, match="SampledSpectrum"):
        hostcheck.Render(scene, scenes.RenderSetup(16, 16, 1, spectral_tables=tables))
    scene.close()
    ctx.close()
