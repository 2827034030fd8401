"""CPU pre-flight of the alpha masks (tests/test_zz_alpha_gpu.py) on the check build of the library (tests/emu: api.cu
and kernels.cu compiled as plain C++, where every traversal is traverse_wbvh), including its drop-in binaries, the
refusals of the new C ABI entry points, and the host's refusals of out-of-scope masks, which need no device."""
import json
import os
import subprocess

import numpy as np
import pytest

import test_infinite_hostcheck as IH
import test_zz_alpha_gpu as A
from conftest import GOLDEN

hc_plugin = IH.hc_plugin


@pytest.mark.parametrize("name", sorted(A.CASES))
def test_dropin_alpha_on_the_check_library(hc_plugin, scenes, tmp_path, name):
    A.test_dropin_alpha_vs_reference(scenes, tmp_path, name, plugin=hc_plugin)


def test_all_zero_mask_on_the_check_library(hc_plugin, scenes, tmp_path):
    A.test_dropin_all_zero_mask_renders_as_without_the_mesh(scenes, tmp_path, plugin=hc_plugin)


@pytest.fixture
def hc_scene(hostcheck, scenes):
    ctx = hostcheck.Context(0)
    arr = scenes.SceneArrays(500, materials=("matte", "plastic"), soup_version=1, n_lights=1)
    scene = hostcheck.Scene(ctx, arr.desc(), keepalive=arr)
    yield hostcheck, arr, scene
    scene.close()
    ctx.close()


def test_add_alpha_mask_refuses_bad_masks(hc_scene, abi):
    hc, arr, scene = hc_scene
    with pytest.raises(hc.B200ptError, match="wrap mode"):
        scene.add_alpha_mask(np.ones((4, 4), np.float32), 3)
    with pytest.raises(ValueError):
        scene.add_alpha_mask(np.ones((4, 4, 3), np.float32))
    rec = abi.AlphaMask()
    rec.width, rec.height = 4, 0
    out = hc.C.c_int32()
    assert hc.lib.b200pt_scene_add_alpha_mask(scene.h, hc.C.byref(rec), hc.C.byref(out)) == -1  # bad size
    rec.width, rec.height = 4, 4  # texels NULL
    assert hc.lib.b200pt_scene_add_alpha_mask(scene.h, hc.C.byref(rec), hc.C.byref(out)) == -1
    assert scene.add_alpha_mask(np.ones((4, 8), np.float32), abi.WRAP_CLAMP) == 0
    assert scene.add_alpha_mask(None) == 1  # ConstantTexture(0)


def test_set_alpha_masks_refuses_bad_ids_and_late_calls(hc_scene, abi, scenes):
    hc, arr, scene = hc_scene
    m = scene.add_alpha_mask(np.ones((4, 4), np.float32))
    n = scene.n_triangles
    with pytest.raises(hc.B200ptError, match="out of range"):
        scene.set_alpha_masks(np.full(n, m + 1, np.int32))
    with pytest.raises(hc.B200ptError, match="shadowalpha mask -2"):
        scene.set_alpha_masks(None, np.full(n, -2, np.int32))
    with pytest.raises(ValueError):
        scene.set_alpha_masks(np.zeros(n - 1, np.int32))
    scene.set_alpha_masks(np.where(arr.material_id == 1, m, -1), None)
    r = hc.Render(scene, scenes.RenderSetup(16, 16, 2))
    r.render_tiles()
    assert np.isfinite(r.read_rgb()).all()
    r.close()
    with pytest.raises(hc.B200ptError, match="already traced or rendered"):
        scene.set_alpha_masks(None, None)
    with pytest.raises(hc.B200ptError, match="already traced or rendered"):
        scene.add_alpha_mask(np.ones((4, 4), np.float32))


def test_sampled_spectrum_scenes_take_alpha_masks(hostcheck, abi, scenes):
    """Masks are Float textures and traversal is shared by both spectrum builds: SampledSpectrum scenes take them."""
    tables = json.load(open(os.path.join(GOLDEN, "spectral_tables.json")))
    arr = scenes.SceneArrays(500, materials=("matte", "plastic"), soup_version=1, n_lights=1).attach_spectral(tables)
    ctx = hostcheck.Context(0)
    scene = hostcheck.Scene(ctx, arr.desc(), keepalive=arr)
    m = scene.add_alpha_mask(A.leaf(30, 8, 8))
    scene.set_alpha_masks(np.full(scene.n_triangles, m, np.int32), None)
    scene.close()
    ctx.close()


# out-of-scope masks: (alpha texture statement, message of the host's refusal)
REFUSED = {
    "checkerboard": ('Texture "a" "float" "checkerboard" "float tex1" [0] "float tex2" [1]', "alpha masks other than"),
    "spherical": ('Texture "a" "float" "imagemap" "string filename" "m.pfm" "string mapping" "spherical"', "mapping other than"),
}


@pytest.mark.parametrize("case", sorted(REFUSED))
def test_dropin_refuses_out_of_scope_masks_without_a_device(scenes, tmp_path, case):
    """The refusals come from the host's flattening, before any device is touched: the real binaries show them here."""
    if not os.path.exists(A.PLUGIN):
        pytest.skip("pbrt_b200 is built where the reference sources exist")
    arr = scenes.SceneArrays(300, soup_version=1, materials=("matte",), alphas={"matte": {"alpha": 0}})
    path = scenes.write_pbrt(str(tmp_path), "refused", arr, 16, 16, 1)
    scenes.write_pfm(os.path.join(str(tmp_path), "m.pfm"), np.ones((4, 4, 3), np.float32))
    tex, why = REFUSED[case]
    text = open(path).read().replace('"float alpha" [0]', '"texture alpha" "a"').replace("WorldBegin\n", "WorldBegin\n" + tex + "\n")
    open(path, "w").write(text)
    r = subprocess.run([A.PLUGIN, "--quiet", os.path.basename(path)], cwd=str(tmp_path), capture_output=True, text=True)
    assert "Error" in r.stdout + r.stderr and why in r.stdout + r.stderr, r.stdout + r.stderr
    assert not os.path.exists(os.path.join(str(tmp_path), "refused.pfm"))


def test_dropin_refuses_tangents_without_a_device(scenes, tmp_path):
    if not os.path.exists(A.PLUGIN):
        pytest.skip("pbrt_b200 is built where the reference sources exist")
    path = os.path.join(str(tmp_path), "tangents.pbrt")
    open(path, "w").write('LookAt 0 0 -3 0 0 0 0 1 0\nCamera "perspective"\nFilm "image" "integer xresolution" [8] '
                          '"integer yresolution" [8] "string filename" "tangents.pfm"\nWorldBegin\n'
                          'LightSource "point" "rgb I" [1 1 1]\nMaterial "matte"\n'
                          'Shape "trianglemesh" "integer indices" [0 1 2] "point P" [-1 -1 0 1 -1 0 0 1 0] '
                          '"vector S" [1 0 0 1 0 0 1 0 0]\nWorldEnd\n')
    r = subprocess.run([A.PLUGIN, "--quiet", os.path.basename(path)], cwd=str(tmp_path), capture_output=True, text=True)
    assert "Error" in r.stdout + r.stderr and "meshes with per-vertex tangents" in r.stdout + r.stderr, r.stdout + r.stderr
    assert not os.path.exists(os.path.join(str(tmp_path), "tangents.pfm"))


@pytest.mark.parametrize("name", ["leaf_uvs_spatial", "textures_behind_cutouts"])
def test_harness_alpha_on_the_check_library(hc_plugin, hostcheck, abi, scenes, tmp_path, name):
    A.test_harness_alpha_vs_reference(hostcheck, abi, scenes, tmp_path, name, plugin=hc_plugin)


def test_dump_without_masks_has_no_alpha_tables(hc_plugin, abi, scenes, tmp_path):
    """A scene without masks dumps no alpha marker: its file ends where the texture tables (or the descriptors) end."""
    arr = scenes.SceneArrays(300, soup_version=1, materials=("matte", "plastic"), n_lights=1)
    path = scenes.write_pbrt(str(tmp_path), "plain", arr, 16, 16, 1)
    dump = os.path.join(str(tmp_path), "plain.dump")
    r = IH.I.run(hc_plugin, path, os.path.join(str(tmp_path), "plain.pfm"), env=dict(B200PT_DUMP_SCENE=dump))
    assert r.returncode == 0, r.stdout + r.stderr
    assert scenes.read_dump_alpha(dump, abi) == ([], None, None)
    assert scenes.read_dump_textures(dump, abi) == ([], [])


def test_trace_vs_reference_per_ray_on_the_check_library(hostcheck, abi, tmp_path):
    if not os.path.exists(A.alpha_rays.PROBE):
        pytest.skip("alpha_probe is built where the reference sources exist")
    ctx = hostcheck.Context(0)
    try:
        A.check_per_ray(hostcheck, abi, ctx, tmp_path)
    finally:
        ctx.close()
