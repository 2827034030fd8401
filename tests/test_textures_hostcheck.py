"""CPU pre-flight of the image-texture path (tests/test_zz_textures_gpu.py) on the check build of the library (tests/emu:
api.cu and kernels.cu compiled as plain C++), including its drop-in binaries, and the refusals of the new C ABI entry
points, which need no device."""
import json
import os

import numpy as np
import pytest

import test_infinite_hostcheck as IH
import test_zz_textures_gpu as T
from conftest import GOLDEN

hc_plugin = IH.hc_plugin


@pytest.mark.parametrize("name", sorted(T.CASES))
def test_dropin_textures_on_the_check_library(hc_plugin, scenes, tmp_path, name):
    T.test_dropin_textures_vs_reference(scenes, tmp_path, name, plugin=hc_plugin)


@pytest.mark.parametrize("name", ["ewa_matte_plastic", "thinlens_halton_aniso"])
def test_harness_textures_on_the_check_library(hc_plugin, hostcheck, abi, scenes, tmp_path, name):
    T.test_harness_textures_vs_reference(hostcheck, abi, scenes, tmp_path, name, plugin=hc_plugin)


def test_known_answer_on_the_check_library(hc_plugin, scenes, tmp_path):
    T.test_known_answer_image_textured_sphere_under_constant_sky(scenes, tmp_path, plugin=hc_plugin)


@pytest.mark.parametrize("case", sorted(T.REFUSED))
def test_dropin_refuses_out_of_scope_textures_without_a_device(scenes, tmp_path, case):
    """The refusals come from the host's flattening, before any device is touched: the real binaries show them here."""
    if not os.path.exists(T.PLUGIN):
        pytest.skip("pbrt_b200 is built where the reference sources exist")
    T.test_dropin_refuses_out_of_scope_textures(scenes, tmp_path, case)


def test_dropin_refuses_spectral_hosts_without_a_device(scenes, tmp_path):
    if not os.path.exists(T.PLUGIN):
        pytest.skip("pbrt_b200 is built where the reference sources exist")
    T.test_dropin_refuses_image_textures_on_spectral_hosts(scenes, tmp_path)


def _pyramid(w, h, channels=3):
    """MIPMap's level sizes for a power-of-two w x h map (mipmap.h:184-207), filled with 0.5."""
    levels = []
    while True:
        levels.append(np.full((h, w, 3) if channels == 3 else (h, w), 0.5, np.float32))
        if w == 1 and h == 1:
            return levels
        w, h = max(1, w // 2), max(1, h // 2)


@pytest.fixture
def hc_scene(hostcheck, scenes):
    ctx = hostcheck.Context(0)
    arr = scenes.SceneArrays(500, materials=("matte", "plastic", "metal", "glass", "mirror"), soup_version=1, n_lights=1)
    scene = hostcheck.Scene(ctx, arr.desc(), keepalive=arr)
    yield hostcheck, arr, scene
    scene.close()
    ctx.close()


def test_add_mipmap_refuses_bad_pyramids(hc_scene, abi):
    hc, _, scene = hc_scene
    lut = np.ones(128, np.float32)
    with pytest.raises(hc.B200ptError, match="not powers of two"):
        scene.add_mipmap([np.zeros((6, 8, 3), np.float32)], abi.WRAP_REPEAT, 0, 8.0, lut)
    with pytest.raises(hc.B200ptError, match="levels for a"):
        scene.add_mipmap(_pyramid(8, 4)[:-1], abi.WRAP_REPEAT, 0, 8.0, lut)
    bad = _pyramid(8, 4)
    bad[2] = np.zeros((2, 2, 3), np.float32)  # level 2 of 8 x 4 is 2 x 1
    with pytest.raises(hc.B200ptError, match="level 2 is 2 x 2"):
        scene.add_mipmap(bad, abi.WRAP_REPEAT, 0, 8.0, lut)
    with pytest.raises(hc.B200ptError, match="wrap mode"):
        scene.add_mipmap(_pyramid(4, 4), 3, 0, 8.0, lut)
    assert scene.add_mipmap(_pyramid(8, 4), abi.WRAP_CLAMP, 1, 8.0, lut) == 0
    assert scene.add_mipmap(_pyramid(1, 16, 1), abi.WRAP_BLACK, 0, 1.0, lut) == 1


def test_bind_texture_refuses_bad_ids_and_slots(hc_scene, abi):
    hc, arr, scene = hc_scene
    lut = np.ones(128, np.float32)
    rgb = scene.add_mipmap(_pyramid(4, 4), abi.WRAP_REPEAT, 0, 8.0, lut)
    gray = scene.add_mipmap(_pyramid(4, 4, 1), abi.WRAP_REPEAT, 0, 8.0, lut)
    mat = {n: arr.material_names.index(n) for n in ("matte", "plastic", "metal", "glass", "mirror")}
    with pytest.raises(hc.B200ptError, match="material .* out of range"):
        scene.bind_texture(len(arr.material_names), abi.TEX_KD, rgb)
    with pytest.raises(hc.B200ptError, match="slot .* out of range"):
        scene.bind_texture(mat["matte"], abi.TEX_SLOTS, rgb)
    with pytest.raises(hc.B200ptError, match="mipmap .* out of range"):
        scene.bind_texture(mat["matte"], abi.TEX_KD, 2)
    for m, slot in (("matte", abi.TEX_KS), ("metal", abi.TEX_KD), ("glass", abi.TEX_ETA), ("mirror", abi.TEX_KT),
                    ("plastic", abi.TEX_ROUGHNESS_V), ("glass", abi.TEX_ROUGHNESS_U)):
        with pytest.raises(hc.B200ptError, match="has no slot"):
            scene.bind_texture(mat[m], slot, gray if slot >= abi.TEX_ROUGHNESS_U else rgb)
    with pytest.raises(hc.B200ptError, match="1-channel map"):
        scene.bind_texture(mat["plastic"], abi.TEX_ROUGHNESS_U, rgb)
    with pytest.raises(hc.B200ptError, match="3-channel map"):
        scene.bind_texture(mat["matte"], abi.TEX_KD, gray)
    scene.bind_texture(mat["matte"], abi.TEX_KD, rgb, 2.0, 1.0, 0.1, 0.0)
    scene.bind_texture(mat["metal"], abi.TEX_ROUGHNESS_V, gray, remap_roughness=True)


def test_textured_render_on_the_check_library(hc_scene, abi, scenes):
    """With a texture bound, the render runs the textured path end to end (pFilm kept, differentials rebuilt)."""
    hc, arr, scene = hc_scene
    rgb = scene.add_mipmap(_pyramid(8, 8), abi.WRAP_REPEAT, 0, 8.0, np.ones(128, np.float32))
    scene.bind_texture(arr.material_names.index("matte"), abi.TEX_KD, rgb)
    r = hc.Render(scene, scenes.RenderSetup(16, 16, 2))
    r.render_tiles()
    assert np.isfinite(r.read_rgb()).all()
    r.close()


def test_sampled_spectrum_scenes_refuse_textures(hostcheck, abi, scenes):
    tables = json.load(open(os.path.join(GOLDEN, "spectral_tables.json")))
    arr = scenes.SceneArrays(500, materials=("matte", "plastic"), soup_version=1, n_lights=1).attach_spectral(tables)
    ctx = hostcheck.Context(0)
    scene = hostcheck.Scene(ctx, arr.desc(), keepalive=arr)
    with pytest.raises(hostcheck.B200ptError, match="SampledSpectrum"):
        scene.add_mipmap(_pyramid(4, 4), abi.WRAP_REPEAT, 0, 8.0, np.ones(128, np.float32))
    with pytest.raises(hostcheck.B200ptError, match="SampledSpectrum"):
        scene.bind_texture(0, abi.TEX_KD, 0)
    scene.close()
    ctx.close()
