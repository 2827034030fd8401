"""InfiniteAreaLight (lights/infinite.cpp) under Integrator "path": constant and image-mapped skies, rotated and scaled,
alone or next to area, sphere and delta lights, through the drop-in binary (the host hands over Lmap's level 0 and its
Distribution2D) and through the C ABI from Python (the same tables, taken from the host's B200PT_DUMP_SCENE file).
Every image is compared bit for bit, and the ray counters exactly, with what the unmodified reference renders from the
same .pbrt file.  The environment maps are small PFMs generated from a seed."""
import os
import re
import subprocess

import numpy as np
import pytest

from conftest import ROOT, bits

pytestmark = pytest.mark.gpu

REF = os.path.join(ROOT, "oracle", "_ref", "pbrt_ref")
PLUGIN = os.path.join(ROOT, "oracle", "_ref", "plugin", "pbrt_b200")
PLUGIN_SPECTRAL = os.path.join(ROOT, "oracle", "_ref", "plugin", "pbrt_b200_spectral")
needs_binaries = pytest.mark.skipif(not (os.path.exists(REF) and os.path.exists(PLUGIN)),
                                    reason="pbrt_ref / pbrt_b200 are built where the reference sources exist")


def sky_pow2(seed=11, w=32, h=16):
    """A power-of-two map with a black band (rows whose Distribution2D entries are 0) and one bright texel."""
    m = np.random.default_rng(seed).uniform(0.2, 1.5, (h, w, 3)).astype(np.float32)
    m[h // 2 - 2:h // 2] = 0
    m[3, 5] = (60.0, 50.0, 40.0)
    return m


def sky_npot(seed=12, w=24, h=10):
    """A map the host's MIPMap resamples to a power of two (mipmap.h:126-190)."""
    return np.random.default_rng(seed).uniform(0.0, 2.0, (h, w, 3)).astype(np.float32)


INSTANCES = dict(objects=(dict(n_tris=400, seed=5, material="plastic", size=0.35), dict(n_tris=150, seed=9, material="glass", size=0.5)),
                 instances=(dict(object=0, center=(0.0, 0.0, -2.4)), dict(object=0, center=(1.2, 0.8, -2.0), scale=(0.7, 1.4, 1.0)),
                            dict(object=1, center=(-1.1, -0.7, -2.2), scale=(1.0, 1.0, -1.3))))

# name: (scene arguments, film w, h, spp, maxdepth, strategy, write_pbrt extras)
CASES = {
    # a constant sky next to the area-light quads, uniform light sampling
    "const_area": (dict(n_tris=3000, materials=("matte", "glass", "metal", "plastic"), n_lights=2,
                        infinite_lights=[dict(L=(0.6, 0.7, 0.9))]), 40, 32, 8, 5, "uniform", {}),
    # the mapped sky rotated and scaled, spatial strategy; mirror and glass: escapes at the end of specular chains
    "map_rotate_scale": (dict(n_tris=3000, materials=("matte", "glass", "mirror", "plastic"),
                              infinite_lights=[dict(map=sky_pow2(), scale=(1.5, 1.2, 1.0), steps=[("Rotate", (-90, 1, 0, 0))])]),
                         40, 32, 8, 7, "spatial", {}),
    # the resampled map, power strategy, Halton
    "npot_power_halton": (dict(n_tris=3000, materials=("matte", "metal"), infinite_lights=[dict(map=sky_npot(), L=0.8)]),
                          40, 32, 6, 5, "power", dict(sampler="halton")),
    # the sky as the only light over spheres and object instances (worldRadius from all shapes), Gaussian filter
    "sky_only_shapes": (dict(n_tris=2000, materials=("matte", "glass", "plastic"), n_lights=0,
                             infinite_lights=[dict(map=sky_pow2(13), steps=[("Rotate", (30, 0, 1, 0))])],
                             spheres=[dict(center=(0.3, -0.2, 0.5), radius=0.4, material="glass"),
                                      dict(center=(-0.6, 0.4, 0.2), radius=0.3, material="matte")], **INSTANCES),
                        40, 32, 4, 5, "spatial", dict(pixel_filter="gaussian")),
    # two infinite lights (one constant, one mapped) next to a point and a distant light
    "two_skies_delta": (dict(n_tris=3000, materials=("matte", "plastic"),
                             infinite_lights=[dict(L=0.3), dict(map=sky_npot(14), steps=[("Rotate", (45, 0, 0, 1))])],
                             delta_lights=[dict(kind="point", from_=(0.5, 1.5, -1.0), I=3.0),
                                           dict(kind="distant", from_=(1, 1, -1), to=(0, 0, 0), L=0.7)]),
                        40, 32, 8, 5, "power", {}),
}
COUNTERS = ("Camera rays traced", "Regular ray intersection tests", "Shadow ray intersection tests")


def counters(text):
    """The ray counters of pbrt's statistics print-out (the drop-in reports its own with a " (GPU)" suffix)."""
    out = {}
    for name in COUNTERS:
        m = re.search(r"^\s*%s(?: \(GPU\))?\s+(\d+)\s*$" % re.escape(name), text, re.M)
        out[name] = int(m.group(1)) if m else None
    return out


def write_case(scenes, tmp_path, name, **over):
    kw, w, h, spp, depth, strat, extra = CASES[name]
    kw = dict(kw, **over)
    nt = kw.pop("n_tris")
    arr = scenes.SceneArrays(nt, soup_version=1, **kw)
    path = scenes.write_pbrt(str(tmp_path), name, arr, w, h, spp, max_depth=depth, strategy=strat, **extra)
    return arr, path


def run(binary, path, out, env=None):
    """Renders `path` with `binary` into `out` (the reference with one thread: the film merge order of a serial run)."""
    cmd = [binary, "--outfile", out, os.path.basename(path)]
    if binary == REF:
        cmd[1:1] = ["--nthreads", "1"]
    r = subprocess.run(cmd, cwd=os.path.dirname(path), capture_output=True, text=True, env=dict(os.environ, **(env or {})))
    return r


def render_pair(scenes, tmp_path, name, plugin=PLUGIN, **over):
    """(drop-in image, reference image, drop-in counters, reference counters) of one case."""
    _, path = write_case(scenes, tmp_path, name, **over)
    ref = run(REF, path, os.path.join(str(tmp_path), "ref.pfm"))
    assert ref.returncode == 0, ref.stdout + ref.stderr
    got = run(plugin, path, os.path.join(str(tmp_path), "got.pfm"))
    assert got.returncode == 0 and "Error" not in got.stderr, got.stdout + got.stderr
    return (scenes.read_pfm(os.path.join(str(tmp_path), "got.pfm")), scenes.read_pfm(os.path.join(str(tmp_path), "ref.pfm")),
            counters(got.stdout + got.stderr), counters(ref.stdout + ref.stderr))


def assert_same(got, ref, cgot, cref, what):
    diff = bits(got) != bits(ref)
    assert got.shape == ref.shape
    assert not diff.any(), "%s: %d of %d components differ from the reference (max abs %.3g)" % (
        what, diff.sum(), diff.size, np.abs(got - ref).max())
    assert cref["Regular ray intersection tests"] and cgot == cref, "%s: ray counters %s, reference %s" % (what, cgot, cref)


@needs_binaries
@pytest.mark.parametrize("name", sorted(CASES))
def test_dropin_infinite_light_vs_reference(scenes, tmp_path, name, plugin=PLUGIN):
    got, ref, cg, cr = render_pair(scenes, tmp_path, name, plugin)
    assert_same(got, ref, cg, cr, name)


def harness_render(pkg, abi, scenes, ctx, tmp_path, name, plugin=PLUGIN):
    """The case through the Python harness: SceneArrays' own descriptor plus the tables the host hands over."""
    arr, path = write_case(scenes, tmp_path, name)
    dump = os.path.join(str(tmp_path), "scene.dump")
    run(plugin, path, os.path.join(str(tmp_path), "unused.pfm"), env=dict(B200PT_DUMP_SCENE=dump))
    tables = scenes.read_dump_infinite(dump, abi)
    kinds = [arr._lights[i].kind for i in range(arr.n_lights)]
    assert sorted(tables) == [i for i, k in enumerate(kinds) if k == abi.LIGHT_INFINITE]
    _, w, h, spp, depth, strat, extra = CASES[name]
    setup = scenes.RenderSetup(w, h, spp, max_depth=depth, strategy={"uniform": abi.LIGHTS_UNIFORM, "power": abi.LIGHTS_POWER,
                                                                     "spatial": abi.LIGHTS_SPATIAL}[strat], **extra)
    scene = pkg.Scene(ctx, arr.desc(), keepalive=arr)
    for light, t in tables.items():
        scene.set_infinite_light(light, t)
    r = pkg.Render(scene, setup)
    r.render_tiles()
    rgb, st = r.read_rgb(), r.stats()
    r.close()
    scene.close()
    return rgb, st, path


@needs_binaries
@pytest.mark.parametrize("name", ["const_area", "map_rotate_scale", "npot_power_halton", "two_skies_delta"])
def test_harness_infinite_light_vs_reference(pkg, abi, scenes, tmp_path, name, plugin=PLUGIN):
    ctx = pkg.Context(0)
    try:
        rgb, st, path = harness_render(pkg, abi, scenes, ctx, tmp_path, name, plugin)
    finally:
        ctx.close()
    ref_run = run(REF, path, os.path.join(str(tmp_path), "ref.pfm"))
    ref = scenes.read_pfm(os.path.join(str(tmp_path), "ref.pfm"))
    cref = counters(ref_run.stdout + ref_run.stderr)
    cgot = {"Camera rays traced": st["camera_rays"], "Regular ray intersection tests": st["regular_rays"],
            "Shadow ray intersection tests": st["shadow_rays"]}
    assert_same(rgb, ref, cgot, cref, name)


KNOWN_ANSWER = """LookAt 0 0 -4  0 0 0  0 1 0
Camera "perspective" "float fov" [40]
Film "image" "integer xresolution" [64] "integer yresolution" [64] "string filename" "ka.pfm"
Sampler "sobol" "integer pixelsamples" [64]
Integrator "path" "integer maxdepth" [12]
WorldBegin
LightSource "infinite" "rgb L" [1 1 1]
AttributeBegin
  Material "matte" "rgb Kd" [0.5 0.5 0.5]
  Shape "sphere" "float radius" [1]
AttributeEnd
AttributeBegin
  Material "matte" "rgb Kd" [0 0 0]
  Translate 0 0 -60
  Shape "trianglemesh" "integer indices" [0 1 2] "point P" [0 0 0  0.001 0 0  0 0.001 0]
AttributeEnd
WorldEnd
"""


def known_answer_masks(n=64):
    """Pixels whose footprint lies inside the sphere's image / entirely outside it (camera at distance 4, fov 40)."""
    half = np.tan(np.radians(20.0))
    c = (np.arange(n) + 0.5) / n * 2 - 1
    x, y = np.meshgrid(c * half, c * half)
    # angle of the pixel's ray from the axis against the sphere's angular radius asin(1/4)
    ang = np.arctan(np.hypot(x, y))
    rad = np.arcsin(0.25)
    px = 2 * half / n
    return ang < rad - 2 * px, ang > rad + 2 * px


@needs_binaries
def test_known_answer_matte_sphere_under_constant_sky(scenes, tmp_path, plugin=PLUGIN):
    """A convex Lambertian sphere with Kd 0.5 under a constant sky of radiance 1 reflects 0.5 in expectation (it never
    sees itself); every camera ray that misses it returns 1.  (The tiny black triangle far behind the camera
    only gives the triangle arrays something to hold.)"""
    path = os.path.join(str(tmp_path), "ka.pbrt")
    open(path, "w").write(KNOWN_ANSWER)
    r = run(plugin, path, os.path.join(str(tmp_path), "ka.pfm"))
    assert r.returncode == 0, r.stdout + r.stderr
    img = scenes.read_pfm(os.path.join(str(tmp_path), "ka.pfm"))
    inside, outside = known_answer_masks()
    assert inside.sum() > 300 and outside.sum() > 2000
    assert abs(float(img[inside].mean()) - 0.5) < 0.02, img[inside].mean()
    # (the film's XYZ round trip, film.cpp:117-130 and :174-203, may move 1 by an ulp or so)
    assert np.abs(img[outside] - 1.0).max() < 1e-5, np.abs(img[outside] - 1.0).max()
    rr = run(REF, path, os.path.join(str(tmp_path), "ka_ref.pfm"))
    assert rr.returncode == 0, rr.stdout + rr.stderr
    assert np.array_equal(bits(img), bits(scenes.read_pfm(os.path.join(str(tmp_path), "ka_ref.pfm"))))


@needs_binaries
@pytest.mark.parametrize("strategy", ["uniform", "power", "spatial"])
def test_larger_render_vs_reference(scenes, tmp_path, strategy, plugin=PLUGIN):
    """160 x 120 at 64 spp, maxdepth 8, the mapped sky next to the area lights, under each light sample strategy: the
    image bit for bit and the ray counters exactly."""
    kw = dict(n_tris=20000, materials=("matte", "glass", "mirror", "plastic"), n_lights=4,
              infinite_lights=[dict(map=sky_pow2(21, 64, 32), steps=[("Rotate", (-90, 1, 0, 0))])])
    arr = scenes.SceneArrays(kw.pop("n_tris"), soup_version=1, **kw)
    path = scenes.write_pbrt(str(tmp_path), "large_" + strategy, arr, 160, 120, 64, max_depth=8, strategy=strategy)
    ref = run(REF, path, os.path.join(str(tmp_path), "ref.pfm"))
    assert ref.returncode == 0, ref.stdout + ref.stderr
    got = run(plugin, path, os.path.join(str(tmp_path), "got.pfm"))
    assert got.returncode == 0, got.stdout + got.stderr
    assert_same(scenes.read_pfm(os.path.join(str(tmp_path), "got.pfm")), scenes.read_pfm(os.path.join(str(tmp_path), "ref.pfm")),
                counters(got.stdout + got.stderr), counters(ref.stdout + ref.stderr), "large " + strategy)


def refused(binary, scenes, tmp_path, name, **write_kw):
    """Runs `binary` on the case written with `write_kw`; returns its output after checking it wrote no image."""
    kw, w, h, spp, depth, strat, extra = CASES[name]
    kw = dict(kw)
    arr = scenes.SceneArrays(kw.pop("n_tris"), soup_version=1, **kw)
    path = scenes.write_pbrt(str(tmp_path), name, arr, w, h, spp, max_depth=depth, strategy=strat, **dict(extra, **write_kw))
    out = os.path.join(str(tmp_path), "refused.pfm")
    r = subprocess.run([binary, "--quiet", "--outfile", out, os.path.basename(path)], cwd=str(tmp_path), capture_output=True, text=True)
    assert not os.path.exists(out), "no image may be written"
    return r.stdout + r.stderr


@needs_binaries
def test_dropin_refuses_volpath_and_spectral_hosts(scenes, tmp_path, plugin=PLUGIN, plugin_spectral=PLUGIN_SPECTRAL):
    msg = refused(plugin, scenes, tmp_path, "map_rotate_scale", integrator="volpath")
    assert "Error" in msg and "infinite area lights under the volumetric integrator" in msg, msg
    if os.path.exists(plugin_spectral):
        msg = refused(plugin_spectral, scenes, tmp_path, "const_area")
        assert "Error" in msg and "infinite area lights in a SampledSpectrum build" in msg, msg
