"""ImageTexture (textures/imagemap.h) under UVMapping2D on matte, plastic, metal, glass and mirror parameters: EWA and
trilinear filtering from the camera rays' differentials, the three wrap modes, per-hit lobe sets from black texels,
Clamp() of negative texels, roughness maps with and without remapping, on meshes with and without uvs, spheres, object
instances, the thin lens, both samplers, every light strategy and both integrators.  Through the drop-in binary (the
host hands over its own MIPMap pyramids) and through the C ABI from Python (the same tables, taken from the host's
B200PT_DUMP_SCENE file); every image is compared bit for bit, and the ray counters exactly, with what the unmodified
reference renders from the same .pbrt file.  The maps are small PFMs generated from a seed."""
import os
import sys

import numpy as np
import pytest

from conftest import ROOT, bits
import test_zz_infinite_gpu as I

pytestmark = pytest.mark.gpu

REF, PLUGIN, PLUGIN_SPECTRAL, needs_binaries = I.REF, I.PLUGIN, I.PLUGIN_SPECTRAL, I.needs_binaries


def rgb_map(seed, w, h, lo=-0.2, hi=1.6):
    """Texels in [lo, hi): negative ones (Clamp() matters), ones above 1, and a black block (the lobe rules per hit)."""
    m = np.random.default_rng(seed).uniform(lo, hi, (h, w, 3)).astype(np.float32)
    m[h // 4:h // 2, w // 4:w // 2] = 0
    return m


def gray_map(seed, w, h, lo=0.02, hi=0.6):
    """A float texture's image (the host reads y() of each texel, imagemap.h convertIn)."""
    g = np.random.default_rng(seed).uniform(lo, hi, (h, w, 1)).astype(np.float32)
    return np.repeat(g, 3, axis=2)


INSTANCES = dict(objects=(dict(n_tris=300, seed=5, material="plastic", size=0.4),),
                 instances=(dict(object=0, center=(0.0, 0.0, -2.2)),
                            dict(object=0, center=(1.0, 0.6, -1.8), rotate=(35, 0.3, 1, 0.2)),
                            dict(object=0, center=(-1.0, -0.6, -2.0), scale=(1.0, -1.2, 1.0), rotate=(-50, 1, 0, 0))))

# name: (scene arguments, film w, h, spp, maxdepth, strategy, write_pbrt extras)
CASES = {
    # EWA on a non-power-of-two map (the host resamples it) and on a square one, per-vertex uvs, shading normals on the
    # matte mesh (its shading dpdu is not the geometric one ComputeDifferentials uses), a constant sky
    "ewa_matte_plastic": (dict(n_tris=3000, materials=("matte", "plastic"), uvs=(0, 1), shading_normals=(0,), n_lights=2,
                               infinite_lights=[dict(L=0.5)],
                               textures={"matte": {"Kd": dict(map=rgb_map(31, 24, 10), uscale=2.5, vdelta=0.3)},
                                         "plastic": {"Kd": dict(map=rgb_map(32, 32, 32), vscale=1.5, udelta=-0.2)}}),
                          40, 32, 8, 5, "spatial", {}),
    # trilinear maps with clamp and black wraps on every other textured slot; roughness maps through RoughnessToAlpha
    "trilinear_slots": (dict(n_tris=3000, materials=("plastic", "metal", "glass", "mirror"), uvs=(0, 1, 2, 3),
                             textures={"plastic": {"Ks": dict(map=rgb_map(33, 16, 16), trilinear=True, wrap="clamp", uscale=3),
                                                   "roughness": dict(map=gray_map(34, 16, 8), trilinear=True, wrap="black",
                                                                     uscale=2, vdelta=-0.5)},
                                       "metal": {"eta": dict(map=rgb_map(35, 8, 8, 0.1, 2.0), trilinear=True, wrap="black", uscale=1.7),
                                                 "k": dict(map=rgb_map(36, 16, 8, 0.5, 4.0), trilinear=True, wrap="clamp"),
                                                 "uroughness": dict(map=gray_map(37, 8, 8), trilinear=True),
                                                 "vroughness": dict(map=gray_map(38, 16, 16, 0.2, 0.9), trilinear=True, wrap="clamp")},
                                       "glass": {"Kr": dict(map=rgb_map(39, 16, 16, 0.0, 1.2), trilinear=True, wrap="black", udelta=0.4),
                                                 "Kt": dict(map=rgb_map(40, 8, 16), trilinear=True)},
                                       "mirror": {"Kr": dict(map=rgb_map(41, 16, 16), trilinear=True, wrap="clamp", vscale=2)}}),
                        40, 32, 8, 7, "uniform", {}),
    # metal roughness maps used as alphas ("remaproughness" false), EWA, a gamma-decoded scaled map
    "metal_no_remap": (dict(n_tris=3000, materials=("metal", "matte"), uvs=(0,),
                            textures={"metal": {"roughness": dict(map=gray_map(42, 32, 16, 0.01, 0.3)), "params": '"bool remaproughness" "false"'},
                                      "matte": {"Kd": dict(map=rgb_map(43, 16, 16, 0.0, 1.0), gamma=True, scale=0.8)}}),
                       40, 32, 8, 5, "power", {}),
    # textured spheres (one of them partial), textured objects in rotated and mirrored instances, meshes without uvs
    "shapes_instances": (dict(n_tris=2000, materials=("matte", "plastic"), n_lights=2,
                              spheres=[dict(center=(0.3, -0.2, 0.5), radius=0.45, material="matte"),
                                       dict(center=(-0.7, 0.4, 0.2), radius=0.35, material="matte", zmin=-0.2, zmax=0.3, phimax=270)],
                              textures={"matte": {"Kd": dict(map=rgb_map(44, 32, 16), uscale=4)},
                                        "plastic": {"Kd": dict(map=rgb_map(45, 16, 16), wrap="clamp", uscale=2, vscale=3)}},
                              **INSTANCES),
                         40, 32, 8, 5, "spatial", {}),
    # the thin lens (differentials from the second ConcentricSampleDisk) with Halton; maxanisotropy 1 clamps every
    # elongated footprint of the soup's grazing triangles
    "thinlens_halton_aniso": (dict(n_tris=3000, materials=("matte", "plastic"), uvs=(0, 1),
                                   textures={"matte": {"Kd": dict(map=rgb_map(46, 64, 64), maxanisotropy=1, uscale=6, vscale=6)},
                                             "plastic": {"Kd": dict(map=rgb_map(47, 32, 8), maxanisotropy=2)}}),
                              40, 32, 6, 5, "spatial", dict(sampler="halton", lens_radius=0.08, focal_distance=4.3)),
    # VolPathIntegrator in fog: camera rays keep their differentials through the medium
    "volpath_fog": (dict(n_tris=3000, materials=("matte", "plastic"), uvs=(0, 1),
                         textures={"matte": {"Kd": dict(map=rgb_map(48, 32, 32), uscale=2)},
                                   "plastic": {"Ks": dict(map=rgb_map(49, 16, 16), trilinear=True)}}),
                    40, 32, 8, 5, "uniform", dict(integrator="volpath", medium=dict(sigma_a=(0.02, 0.03, 0.04), sigma_s=(0.05, 0.04, 0.03)))),
    # a cloud some camera rays cross before their textured hit: those rays are spawned anew and lose their differentials
    "volpath_cloud": (dict(n_tris=3000, materials=("matte", "plastic"), uvs=(0, 1),
                           spheres=[dict(center=(0.0, 0.0, -2.5), radius=0.8, boundary=dict(sigma_a=(0.3, 0.3, 0.3), sigma_s=(0.5, 0.5, 0.5)))],
                           textures={"matte": {"Kd": dict(map=rgb_map(50, 32, 32), uscale=3)},
                                     "plastic": {"Kd": dict(map=rgb_map(51, 16, 32))}}),
                      40, 32, 8, 5, "uniform", dict(integrator="volpath")),
}


def write_case(scenes, tmp_path, name):
    kw, w, h, spp, depth, strat, extra = CASES[name]
    kw = dict(kw)
    arr = scenes.SceneArrays(kw.pop("n_tris"), soup_version=1, **kw)
    path = scenes.write_pbrt(str(tmp_path), name, arr, w, h, spp, max_depth=depth, strategy=strat, **extra)
    return arr, path


def render_pair(scenes, tmp_path, name, plugin):
    _, path = write_case(scenes, tmp_path, name)
    ref = I.run(REF, path, os.path.join(str(tmp_path), "ref.pfm"))
    assert ref.returncode == 0, ref.stdout + ref.stderr
    got = I.run(plugin, path, os.path.join(str(tmp_path), "got.pfm"))
    assert got.returncode == 0 and "Error" not in got.stderr, got.stdout + got.stderr
    return (scenes.read_pfm(os.path.join(str(tmp_path), "got.pfm")), scenes.read_pfm(os.path.join(str(tmp_path), "ref.pfm")),
            I.counters(got.stdout + got.stderr), I.counters(ref.stdout + ref.stderr))


@needs_binaries
@pytest.mark.parametrize("name", sorted(CASES))
def test_dropin_textures_vs_reference(scenes, tmp_path, name, plugin=PLUGIN):
    got, ref, cg, cr = render_pair(scenes, tmp_path, name, plugin)
    I.assert_same(got, ref, cg, cr, name)


def harness_render(pkg, abi, scenes, ctx, tmp_path, name, plugin):
    """The case through the Python harness: the host's dumped descriptors, its infinite-light and texture tables."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from replay_dump import DumpScene
    _, path = write_case(scenes, tmp_path, name)
    dump = os.path.join(str(tmp_path), "scene.dump")
    r = I.run(plugin, path, os.path.join(str(tmp_path), "unused.pfm"), env=dict(B200PT_DUMP_SCENE=dump))
    assert r.returncode == 0, r.stdout + r.stderr
    mips, binds = scenes.read_dump_textures(dump, abi)
    assert mips and binds
    ds = DumpScene(dump, abi, scenes)
    setup = ds.setup()
    scene = pkg.Scene(ctx, ds.desc(), keepalive=ds)
    for light, t in scenes.read_dump_infinite(dump, abi).items():
        scene.set_infinite_light(light, t)
    ids = [scene.add_mipmap(m["levels"], m["wrap"], m["trilinear"], m["max_anisotropy"], m["weight_lut"]) for m in mips]
    for b in binds:
        scene.bind_texture(b["material"], b["slot"], ids[b["mipmap"]], b["su"], b["sv"], b["du"], b["dv"], b["remap"])
    rend = pkg.Render(scene, setup)
    rend.render_tiles()
    rgb, st = rend.read_rgb(), rend.stats()
    rend.close()
    scene.close()
    return rgb, st, path


HARNESS_CASES = ["ewa_matte_plastic", "trilinear_slots", "thinlens_halton_aniso", "volpath_fog"]


@needs_binaries
@pytest.mark.parametrize("name", HARNESS_CASES)
def test_harness_textures_vs_reference(pkg, abi, scenes, tmp_path, name, plugin=PLUGIN):
    ctx = pkg.Context(0)
    try:
        rgb, st, path = harness_render(pkg, abi, scenes, ctx, tmp_path, name, plugin)
    finally:
        ctx.close()
    ref_run = I.run(REF, path, os.path.join(str(tmp_path), "ref.pfm"))
    ref = scenes.read_pfm(os.path.join(str(tmp_path), "ref.pfm"))
    cref = I.counters(ref_run.stdout + ref_run.stderr)
    # (pbrt's statistics print-out omits a counter that stayed 0: volpath counts its shadow rays elsewhere)
    cgot = {"Camera rays traced": st["camera_rays"], "Regular ray intersection tests": st["regular_rays"],
            "Shadow ray intersection tests": st["shadow_rays"] or None}
    I.assert_same(rgb, ref, cgot, cref, name)


KNOWN_ANSWER = I.KNOWN_ANSWER.replace('LightSource "infinite"', 'Texture "half" "spectrum" "imagemap" "string filename" "half.pfm"\n'
                                      'LightSource "infinite"').replace(
    'Material "matte" "rgb Kd" [0.5 0.5 0.5]', 'Material "matte" "texture Kd" "half"')


@needs_binaries
def test_known_answer_image_textured_sphere_under_constant_sky(scenes, tmp_path, plugin=PLUGIN):
    """A convex Lambertian sphere whose Kd is an imagemap of uniform 0.5 texels, under a constant sky of radiance 1,
    reflects 0.5 in expectation inside its silhouette; the drop-in matches the reference bit for bit too."""
    scenes.write_pfm(os.path.join(str(tmp_path), "half.pfm"), np.full((8, 16, 3), 0.5, np.float32))
    path = os.path.join(str(tmp_path), "ka.pbrt")
    open(path, "w").write(KNOWN_ANSWER)
    r = I.run(plugin, path, os.path.join(str(tmp_path), "ka.pfm"))
    assert r.returncode == 0 and "Error" not in r.stderr, r.stdout + r.stderr
    img = scenes.read_pfm(os.path.join(str(tmp_path), "ka.pfm"))
    inside, outside = I.known_answer_masks()
    assert abs(float(img[inside].mean()) - 0.5) < 0.02, img[inside].mean()
    assert np.abs(img[outside] - 1.0).max() < 1e-5
    rr = I.run(REF, path, os.path.join(str(tmp_path), "ka_ref.pfm"))
    assert rr.returncode == 0, rr.stdout + rr.stderr
    assert np.array_equal(bits(img), bits(scenes.read_pfm(os.path.join(str(tmp_path), "ka_ref.pfm"))))


@needs_binaries
@pytest.mark.parametrize("strategy", ["uniform", "power", "spatial"])
def test_larger_textured_render_vs_reference(scenes, tmp_path, strategy, plugin=PLUGIN):
    """160 x 120 at 64 spp, maxdepth 8, EWA and trilinear maps on every family next to the area lights: the image bit for
    bit and the ray counters exactly."""
    kw = dict(materials=("matte", "glass", "metal", "plastic"), uvs=(0, 1, 2, 3), n_lights=4,
              textures={"matte": {"Kd": dict(map=rgb_map(61, 64, 48), uscale=3)},
                        "glass": {"Kt": dict(map=rgb_map(62, 32, 32, 0.0, 1.0), trilinear=True)},
                        "metal": {"k": dict(map=rgb_map(63, 32, 32, 0.5, 4.0)), "roughness": dict(map=gray_map(64, 16, 16))},
                        "plastic": {"Kd": dict(map=rgb_map(65, 32, 16), wrap="black"), "Ks": dict(map=rgb_map(66, 16, 16))}})
    arr = scenes.SceneArrays(20000, soup_version=1, **kw)
    path = scenes.write_pbrt(str(tmp_path), "large_" + strategy, arr, 160, 120, 64, max_depth=8, strategy=strategy)
    ref = I.run(REF, path, os.path.join(str(tmp_path), "ref.pfm"))
    assert ref.returncode == 0, ref.stdout + ref.stderr
    got = I.run(plugin, path, os.path.join(str(tmp_path), "got.pfm"))
    assert got.returncode == 0, got.stdout + got.stderr
    I.assert_same(scenes.read_pfm(os.path.join(str(tmp_path), "got.pfm")), scenes.read_pfm(os.path.join(str(tmp_path), "ref.pfm")),
                  I.counters(got.stdout + got.stderr), I.counters(ref.stdout + ref.stderr), "large " + strategy)


REFUSED_BASE = """LookAt 0 0 -4  0 0 0  0 1 0
Camera "perspective" "float fov" [40]
Film "image" "integer xresolution" [16] "integer yresolution" [16] "string filename" "r.pfm"
Sampler "sobol" "integer pixelsamples" [1]
Integrator "path"
WorldBegin
LightSource "point" "rgb I" [1 1 1] "point from" [0 0 -3]
%s
AttributeBegin
  %s
  Shape "sphere" "float radius" [1]
AttributeEnd
WorldEnd
"""
MAP = 'Texture "m" "spectrum" "imagemap" "string filename" "m.pfm"'
FMAP = 'Texture "f" "float" "imagemap" "string filename" "m.pfm"'
REFUSED = {
    "checkerboard": ('Texture "c" "spectrum" "checkerboard"', 'Material "matte" "texture Kd" "c"',
                     'textures other than "constant" and "imagemap"'),
    "spherical_mapping": ('Texture "s" "spectrum" "imagemap" "string filename" "m.pfm" "string mapping" "spherical"',
                          'Material "matte" "texture Kd" "s"', 'mapping other than "uv"'),
    "matte_sigma": (FMAP, 'Material "matte" "texture sigma" "f"', 'textured matte "sigma"'),
    "glass_index": (FMAP, 'Material "glass" "texture index" "f"', 'textured glass "index"'),
    "glass_roughness": (FMAP, 'Material "glass" "texture uroughness" "f"', "textured glass roughness"),
    "bump_map": (MAP + "\n" + FMAP, 'Material "matte" "texture Kd" "m" "texture bumpmap" "f"', "bump maps"),
}


def refused_run(binary, scenes, tmp_path, texture, material):
    scenes.write_pfm(os.path.join(str(tmp_path), "m.pfm"), rgb_map(70, 8, 8, 0.1, 0.9))
    path = os.path.join(str(tmp_path), "r.pbrt")
    open(path, "w").write(REFUSED_BASE % (texture, material))
    out = os.path.join(str(tmp_path), "refused.pfm")
    r = I.subprocess.run([binary, "--quiet", "--outfile", out, "r.pbrt"], cwd=str(tmp_path), capture_output=True, text=True)
    assert not os.path.exists(out), "no image may be written"
    return r.stdout + r.stderr


@needs_binaries
@pytest.mark.parametrize("case", sorted(REFUSED))
def test_dropin_refuses_out_of_scope_textures(scenes, tmp_path, case, plugin=PLUGIN):
    texture, material, why = REFUSED[case]
    msg = refused_run(plugin, scenes, tmp_path, texture, material)
    assert "Error" in msg and why in msg, msg


@needs_binaries
def test_dropin_refuses_image_textures_on_spectral_hosts(scenes, tmp_path, plugin_spectral=PLUGIN_SPECTRAL):
    if not os.path.exists(plugin_spectral):
        pytest.skip("pbrt_b200_spectral is built where the reference sources exist")
    msg = refused_run(plugin_spectral, scenes, tmp_path, MAP, 'Material "matte" "texture Kd" "m"')
    assert "Error" in msg and "image textures in a SampledSpectrum build" in msg, msg
