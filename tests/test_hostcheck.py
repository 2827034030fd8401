"""CPU pre-flight of the product's sources (no GPU needed): tests/emu compiles api.cu and kernels.cu -- the files nvcc
compiles into libb200pt.so -- as plain C++ against a stand-in <cuda_runtime.h> in which a kernel launch runs the kernel
function once per thread index.  The GPU parity tests are then replayed against that library: the host logic (scene and
render set-up, batching, wavefront sequencing, film read-back) and the scalar logic of every kernel except the
warp-synchronous k_trace (its rays take traverse_wbvh, the per-ray routine the kernel's lanes step through) are checked
against the reference's golden images and the oracle before any GPU time is spent.  What this cannot show -- nvcc's
code generation, the real warp-level execution, performance -- is what the `-m gpu` run of the same tests is for."""
import os

import numpy as np
import pytest

import test_gpu_parity as G
import test_zz_spectral_gpu as GS
import test_zz_sweeps_gpu as GW
import test_zz_volpath_gpu as GV
from render_cases import RENDERS


@pytest.fixture(scope="module")
def hctx(hostcheck):
    c = hostcheck.Context(0)
    yield c
    c.close()


def test_hostcheck_exports_the_abi(hostcheck, pkg):
    assert hostcheck.lib._name.endswith("libb200pt_hostcheck.so") and pkg.lib._name.endswith("libb200pt.so")
    assert hostcheck.MISSING_SYMBOLS == [] and hostcheck.lib.b200pt_abi_version() == pkg.lib.b200pt_abi_version()


def test_streams_cameras_intersections(hostcheck, abi, scenes, hctx, probe_json):
    G.test_sobol_stream_vs_reference(hostcheck, abi, scenes, hctx, probe_json)
    G.test_halton_stream_vs_reference(hostcheck, abi, scenes, hctx)
    G.test_camera_rays_vs_reference(hostcheck, abi, scenes, hctx, probe_json)
    G.test_intersections_vs_reference_bvhaccel(hostcheck, abi, scenes, hctx)


def test_triangle_watertight(hostcheck, abi, scenes, hctx):
    G.test_triangle_watertight(hostcheck, abi, scenes, hctx)


def test_trace_entry_points_vs_oracle(hostcheck, abi, scenes, ob, hctx):
    G.test_trace_vs_oracle(hostcheck, abi, scenes, ob, hctx, 37, 20000)
    G.test_trace_vs_oracle(hostcheck, abi, scenes, ob, hctx, 20000, 40000)
    G.test_trace_spheres_vs_oracle(hostcheck, abi, scenes, ob, hctx)
    G.test_trace_instances_vs_oracle(hostcheck, abi, scenes, ob, hctx)


# every golden render of the reference (tests/render_cases.py)
FAST = sorted(RENDERS)


@pytest.mark.parametrize("name", FAST)
def test_render_vs_reference_pfm(hostcheck, abi, scenes, ob, hctx, name):
    G.test_render_vs_reference_pfm(hostcheck, abi, scenes, ob, hctx, name)


@pytest.mark.parametrize("gname,base", [("spectral_four", "four"), ("spectral_rough", "rough"), ("spectral_instances", "instances"),
                                        ("spectral_spheres", "spheres"), ("spectral_delta_lights", "delta_lights")])
def test_spectral_render_vs_sampled_spectrum_reference(hostcheck, abi, scenes, ob, hctx, gname, base):
    GS.test_spectral_render_vs_sampled_spectrum_reference(hostcheck, abi, scenes, ob, hctx, gname, base)


@pytest.mark.parametrize("gname,vname", [("spectral_volpath_fog", "volpath_fog"), ("spectral_volpath_fog_spheres", "volpath_fog_spheres")])
def test_spectral_volpath_render_vs_sampled_spectrum_reference(hostcheck, abi, scenes, ob, hctx, gname, vname):
    GS.test_spectral_volpath_render_vs_sampled_spectrum_reference(hostcheck, abi, scenes, ob, hctx, gname, vname)


def test_spectral_counters_power_and_filter(hostcheck, abi, scenes, ob, hctx):
    GS.test_spectral_render_and_counters_vs_oracle(hostcheck, abi, scenes, ob, hctx, ("matte", "glass", "metal", "plastic"), 8, "power", None)
    GS.test_spectral_render_and_counters_vs_oracle(hostcheck, abi, scenes, ob, hctx, ("matte", "metal"), 5, "uniform", "gaussian")


@pytest.mark.parametrize("gname", sorted(GV.VOLPATH))
def test_volpath_render_vs_reference_pfm(hostcheck, abi, scenes, ob, hctx, gname):
    GV.test_volpath_render_vs_reference_pfm(hostcheck, abi, scenes, ob, hctx, gname)


def test_volpath_render_vs_oracle(hostcheck, abi, scenes, ob, hctx):
    thin = dict(sigma_a=(0.01, 0.02, 0.03), sigma_s=(0.4, 0.35, 0.3), g=0.6)
    thick = dict(sigma_a=(0.2, 0.2, 0.2), sigma_s=(1.5, 1.2, 0.9), g=-0.5)
    GV.test_volpath_render_vs_oracle(hostcheck, abi, scenes, ob, hctx, ("matte", "glass", "metal", "plastic"), 8, "power", thin, {})
    GV.test_volpath_render_vs_oracle(hostcheck, abi, scenes, ob, hctx, ("matte", "plastic"), 12, "uniform", thick, {})
    GV.test_volpath_render_vs_oracle(hostcheck, abi, scenes, ob, hctx, ("matte", "metal"), 5, "uniform",
                                     dict(sigma_a=(0.05, 0.05, 0.05), sigma_s=(0.1, 0.1, 0.1), g=0.0), {"pixel_filter": "gaussian"})
    GV.test_volpath_render_vs_oracle(hostcheck, abi, scenes, ob, hctx, ("matte", "glass"), 6, "uniform", None, {})
    # the Halton sampler (ten dimensions per bounce inside a medium) and a thin lens
    GV.test_volpath_render_vs_oracle(hostcheck, abi, scenes, ob, hctx, ("matte", "plastic"), 7, "spatial", thin,
                                     {"sampler": "halton", "lens_radius": 0.05, "focal_distance": 4.0})


@pytest.mark.parametrize("name", ["analytic_point", "analytic_4points", "analytic_area"])
def test_analytic_scenes_known_answer_volpath(hostcheck, abi, scenes, ob, hctx, name):
    GV.test_analytic_scenes_known_answer_volpath(hostcheck, abi, scenes, ob, hctx, name)


@pytest.mark.parametrize("gname", ["volpath_cloud", "volpath_cloud_fog"])
def test_volpath_bounded_media_vs_reference_pfm(hostcheck, abi, scenes, ob, hctx, gname):
    GV.test_volpath_bounded_media_vs_reference_pfm(hostcheck, abi, scenes, ob, hctx, gname)


def test_bounded_media_larger_render_vs_oracle(hostcheck, abi, scenes, ob, hctx):
    GV.test_bounded_media_larger_render_vs_oracle(hostcheck, abi, scenes, ob, hctx)


def test_volpath_instances_and_partial_spheres_vs_oracle(hostcheck, abi, scenes, ob, hctx):
    GV.test_volpath_instances_and_partial_spheres_vs_oracle(hostcheck, abi, scenes, ob, hctx)


def test_render_and_counters_vs_oracle(hostcheck, abi, scenes, ob, hctx):
    G.test_render_and_counters_vs_oracle(hostcheck, abi, scenes, ob, hctx, ("matte", "glass", "metal", "plastic"), 16, "power")


def test_pixel_samples_and_shards(hostcheck, abi, scenes, ob, hctx):
    G.test_pixel_samples_vs_oracle(hostcheck, abi, scenes, ob, hctx)


def test_host_logic_shards_batches_edges(hostcheck, abi, scenes, hctx, monkeypatch):
    """Batching, tile shards, pixelbounds shards, partial tiles, empty ray batches, the ordered merge of FilmTiles."""
    G.test_empty_and_ragged_inputs(hostcheck, abi, scenes, hctx)
    G.test_tile_shards_sum_to_full_render(hostcheck, abi, scenes, hctx)
    G.test_render_is_deterministic_and_batch_independent(hostcheck, abi, scenes, hctx, monkeypatch)


def test_fullsize_checks_at_a_small_film(hostcheck, abi, scenes, ob, hctx, monkeypatch):
    """The benchmark-size tests (tests/test_zz_fullsize_gpu.py) at 160x90 with 7 tiles per batch: nine batches, a partial
    last one, half-height bottom tiles -- the tile set, masks, launch-count arithmetic and comparisons on the CPU."""
    import test_zz_fullsize_gpu as F
    F.test_fullsize_rgb_cfg4_shape(hostcheck, abi, scenes, ob, hctx, monkeypatch, film=(160, 90, 16), n_tris=20000, batch_tiles=7)
    F.test_fullsize_spectral_cfg5_shape(hostcheck, abi, scenes, ob, hctx, monkeypatch, film=(160, 90, 8), n_tris=2000, batch_tiles=7)
    F.test_fullsize_volpath_cfg2fog_shape(hostcheck, abi, scenes, ob, hctx, monkeypatch, film=(160, 90, 16), n_tris=20000,
                                          batch_tiles=7)


def test_instance_lattice_checks_at_a_small_size(hostcheck, abi, scenes, ob, hctx, monkeypatch, tmp_path):
    """The benchmark-lattice tests (tests/test_zz_instances_gpu.py) with small objects, a 5000-triangle soup and 4000 rays
    per family.  The check build has no k_trace2: both arms of the comparison are k_spheres' InstanceWalk here, so this
    checks the tests' own logic (the child process, the ray families, the near-tie rule, the films) and the oracle side,
    not the two-level kernel."""
    import test_zz_instances_gpu as I
    I.test_lattices_are_the_benchmarks()
    I.check_lattice(hostcheck, abi, scenes, ob, hctx, monkeypatch, tmp_path / "cfg5", "cfg5", n_soup=5000, n_tris=2000, n_rays=4000)
    I.check_lattice(hostcheck, abi, scenes, ob, hctx, monkeypatch, tmp_path / "cfg5s", "cfg5s", n_soup=5000, n_tris=5000, n_rays=4000)
    for spectral in (False, True):
        I.test_separated_lattice_renders_vs_oracle(hostcheck, abi, scenes, ob, hctx, monkeypatch, spectral, n_soup=5000, n_tris=2000)


def test_device_bvh_builder_is_refused(hostcheck, abi, scenes, hctx):
    """The check build has no device BVH builder; asking for it must fail loudly, not fall back to the host builder."""
    arr = scenes.SceneArrays(500, materials=("matte",), soup_version=1)
    c = hostcheck.Context(0)
    c.set_option("gpu_bvh_build", 1)
    with pytest.raises(Exception):
        hostcheck.Scene(c, arr.desc(), keepalive=arr)
    c.close()


# ---- the drop-in binaries linked against the check library: gpupath.cpp end to end on the CPU ---------------------------
import test_dropin_plugin as P  # noqa: E402

HC_PLUGIN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu", "pbrt_b200_hostcheck")
HC_PLUGIN_SPECTRAL = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu", "pbrt_b200_spectral_hostcheck")


@pytest.fixture(scope="module")
def hc_plugins(hostcheck):
    import subprocess
    ref = os.path.dirname(os.path.dirname(P.PLUGIN))  # oracle/_ref
    objs = [os.path.join(os.path.dirname(P.PLUGIN), f) for f in ("gpupath.o", "libpbrt_host.a", "gpupath_spectral.o",
                                                                  "libpbrt_host_spectral.a")]
    objs += [os.path.join(ref, d, "main", "pbrt.o") for d in ("obj", "obj_spectral")]
    if not all(os.path.exists(f) for f in objs):
        pytest.skip("the drop-in's objects are built where the reference sources exist")
    r = subprocess.run(["make", "plugins"], cwd=os.path.dirname(HC_PLUGIN), capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]


def test_dropin_binary_on_the_check_library(hc_plugins, scenes, tmp_path, monkeypatch):
    """pbrt's parser and scene construction -> gpupath.cpp's flattening -> C ABI -> the check build: unmodified .pbrt
    files (all materials, PLY meshes with normals / uvs, Halton, spheres, instances, delta lights, a Gaussian filter)
    render bit-identically to the reference."""
    monkeypatch.setattr(P, "PLUGIN", HC_PLUGIN)
    P.test_dropin_binary_matches_reference(scenes, tmp_path)


def test_dropin_three_ranks_one_image_on_the_check_library(hc_plugins, scenes, tmp_path):
    """Multi-process drop-in (B200PT_RANK / B200PT_WORLD_SIZE): three processes render tiles i mod 3 of one film, the
    partial films meet on rank 0, one image comes out and it is the reference's, bit for bit."""
    got, logs = P.run_ranks(HC_PLUGIN, scenes, tmp_path, 3)
    ref = scenes.read_pfm(os.path.join(P.GOLDEN, "render_four.pfm"))
    assert np.array_equal(P.bits(got), P.bits(ref)), "merged image of three ranks differs from the reference PFM"


def test_spectral_dropin_binary_on_the_check_library(hc_plugins, scenes, tmp_path, monkeypatch):
    """The same through the SampledSpectrum host: the 60-bin tables gpupath.cpp extracts give the image of the reference
    built with `typedef SampledSpectrum Spectrum`."""
    monkeypatch.setattr(GS, "PLUGIN_SPECTRAL", HC_PLUGIN_SPECTRAL)
    GS.test_spectral_dropin_binary_matches_sampled_spectrum_reference(scenes, tmp_path)


def test_spectral_volpath_dropin_binary_on_the_check_library(hc_plugins, scenes, tmp_path, monkeypatch):
    monkeypatch.setattr(GS, "PLUGIN_SPECTRAL", HC_PLUGIN_SPECTRAL)
    GS.test_spectral_volpath_dropin_binary_matches_sampled_spectrum_reference(scenes, tmp_path)


def test_volpath_dropin_binary_on_the_check_library(hc_plugins, scenes, tmp_path, monkeypatch):
    """`Integrator "volpath"` with a named homogeneous medium through the drop-in binary."""
    monkeypatch.setattr(GV, "PLUGIN", HC_PLUGIN)
    GV.test_volpath_dropin_binary_matches_reference(scenes, tmp_path)


def test_bounded_media_dropin_binary_on_the_check_library(hc_plugins, scenes, tmp_path, monkeypatch):
    """Null-material spheres around named media through the drop-in binary (medium transitions, SURVEY 8(f) row 4)."""
    monkeypatch.setattr(GV, "PLUGIN", HC_PLUGIN)
    GV.test_bounded_media_dropin_binary_matches_reference(scenes, tmp_path)


@pytest.mark.skipif(not os.path.exists(os.path.join(P.KILLEROO_DIR, "killeroo-simple-ref.pfm")),
                    reason="oracle/_ref/scenes is staged by `make -C oracle ref` where the reference sources exist")
def test_killeroo_as_shipped_on_the_check_library(hc_plugins, scenes, tmp_path, monkeypatch):
    """BASELINE configs[0], scenes/killeroo-simple.pbrt as the reference ships it (700x700, 8 spp)."""
    monkeypatch.setattr(P, "PLUGIN", HC_PLUGIN)
    P.test_killeroo_matches_reference(scenes, tmp_path, "simple", 700)


# ---- error behaviour of the C ABI: bad descriptors are refused with B200PT_ERR_INVALID and a message, never a crash ------
def _expect(hostcheck, what, fn):
    with pytest.raises(hostcheck.B200ptError) as e:
        fn()
    assert what in str(e.value), (what, str(e.value))


def test_bad_scene_descriptors_are_refused(hostcheck, abi, scenes, hctx):
    import ctypes as C

    def scene_with(mutate, **kw):
        arr = scenes.SceneArrays(300, materials=("matte", "plastic"), soup_version=1, **kw)
        d = arr.desc()
        keep = mutate(arr, d)
        try:
            hostcheck.Scene(hctx, d, keepalive=(arr, keep)).close()
        finally:
            del keep

    def bad_material_id(arr, d):
        arr.material_id[7] = 9
    _expect(hostcheck, "has material 9", lambda: scene_with(bad_material_id))

    def bad_light_id(arr, d):
        arr.light_id[3] = 1000
    _expect(hostcheck, "has light 1000", lambda: scene_with(bad_light_id))

    def no_materials(arr, d):
        d.n_materials = 0
    _expect(hostcheck, "no materials", lambda: scene_with(no_materials))

    def bad_material_type(arr, d):
        arr._materials[1].type = 17
    _expect(hostcheck, "unsupported type 17", lambda: scene_with(bad_material_type))

    def no_vertices(arr, d):
        d.vertices = None
    _expect(hostcheck, "vertices / material_id missing", lambda: scene_with(no_vertices))

    def bad_light_kind(arr, d):
        arr._lights[0].kind = 9
    _expect(hostcheck, "unknown kind 9", lambda: scene_with(bad_light_kind))

    def light_disagrees(arr, d):
        arr._lights[0].triangle = 5  # triangle 5 does not name light 0 in light_id[]
    _expect(hostcheck, "disagree", lambda: scene_with(light_disagrees))

    def bad_bins(arr, d):
        d.n_spectrum_samples = 30
    _expect(hostcheck, "n_spectrum_samples is 30", lambda: scene_with(bad_bins))

    def bins_without_tables(arr, d):
        d.n_spectrum_samples = abi.SPECTRUM_SAMPLES
    _expect(hostcheck, "must pass material_spectra", lambda: scene_with(bins_without_tables))

    def bad_sphere(arr, d):
        arr._spheres[0].radius = -1.0
    _expect(hostcheck, "bad radius", lambda: scene_with(bad_sphere, spheres=(dict(center=(0, 0, 0), radius=0.3, material="matte"),)))

    inst = dict(objects=(dict(n_tris=50, seed=5, material="plastic", size=0.3),), instances=(dict(object=0, center=(0, 0, 0)),))

    def bad_instance_range(arr, d):
        arr._instances[0].n_triangles = 10 ** 6
    _expect(hostcheck, "outside the object range", lambda: scene_with(bad_instance_range, **inst))

    def bad_toplevel(arr, d):
        d.n_toplevel_triangles = d.n_triangles + 1
    _expect(hostcheck, "bad n_toplevel_triangles", lambda: scene_with(bad_toplevel, **inst))

    # NULL handles
    with pytest.raises(hostcheck.B200ptError):
        hostcheck._check(hostcheck.lib.b200pt_scene_create(hctx.h, None, C.byref(C.c_void_p())))
    # a scene without any geometry is legal (an empty world renders black, like the reference)
    arr = scenes.SceneArrays(0, materials=("matte",), soup_version=1, n_lights=0)
    s = hostcheck.Scene(hctx, arr.desc(), keepalive=arr)
    r = hostcheck.Render(s, scenes.RenderSetup(16, 16, 2))
    r.render_tiles()
    raw = r.read_raw()
    assert np.all(raw[..., :3] == 0) and np.all(raw[..., 3] >= 2)
    r.close()
    s.close()


def test_bad_render_descriptors_are_refused(hostcheck, abi, scenes, hctx):
    arr = scenes.SceneArrays(300, materials=("matte",), soup_version=1)
    scene = hostcheck.Scene(hctx, arr.desc(), keepalive=arr)

    def render_with(mutate, **kw):
        setup = scenes.RenderSetup(32, 32, 4, **kw)
        mutate(setup)
        hostcheck.Render(scene, setup).close()

    def spp3(s):
        s.sampler.samples_per_pixel = 3
    _expect(hostcheck, "power of two", lambda: render_with(spp3))

    def depth(s):
        s.integrator.max_depth = -1
    _expect(hostcheck, "bad max_depth", lambda: render_with(depth))

    def deep(s):
        s.integrator.max_depth = 100  # more bounces than the Sobol' tables of this set-up have dimensions for
        s.sampler.n_dimensions = 200
    _expect(hostcheck, "sampler dimensions", lambda: render_with(deep))

    def strategy(s):
        s.integrator.light_strategy = 11
    _expect(hostcheck, "unsupported light sample strategy", lambda: render_with(strategy))

    def sampler_type(s):
        s.sampler.type = 5
    _expect(hostcheck, "unknown sampler type 5", lambda: render_with(sampler_type))

    def empty_bounds(s):
        s.sampler.sample_bounds[2] = s.sampler.sample_bounds[0]
    _expect(hostcheck, "empty sample bounds", lambda: render_with(empty_bounds))

    def wide_filter(s):
        s.film.filter_radius[0] = 9.0
    _expect(hostcheck, "pixel filter radius", lambda: render_with(wide_filter))

    def no_tables(s):
        s.sampler.matrices32 = None
    _expect(hostcheck, "tables missing", lambda: render_with(no_tables))

    fog = dict(sigma_a=(0.1, 0.1, 0.1), sigma_s=(0.2, 0.2, 0.2), g=0.2)

    def medium_without_volpath(s):
        s.integrator.volumetric = 0
    _expect(hostcheck, "needs the volumetric integrator", lambda: render_with(medium_without_volpath, integrator="volpath", medium=fog))

    def empty_medium(s):
        s.integrator.medium.sigma_a[1] = 0.0
        s.integrator.medium.sigma_s[1] = 0.0
    _expect(hostcheck, "sigma_t > 0", lambda: render_with(empty_medium, integrator="volpath", medium=fog))

    def bad_g(s):
        s.integrator.medium.g = 1.0
    _expect(hostcheck, "must lie in (-1, 1)", lambda: render_with(bad_g, integrator="volpath", medium=fog))

    r = hostcheck.Render(scene, scenes.RenderSetup(32, 32, 4))
    _expect(hostcheck, "out of range", lambda: r.render_tiles(np.array([0, 99], np.int32)))
    _expect(hostcheck, "more tiles than the film has", lambda: r.render_tiles(None, n=50))
    _expect(hostcheck, "outside the sample bounds", lambda: r.debug_pixel_samples(40, 3))
    r.render_tiles(np.zeros(0, np.int32))  # an empty shard is legal (a rank without tiles)
    assert np.all(r.read_raw() == 0)
    r.close()
    scene.close()


def test_new_paths_in_several_batches(hostcheck, abi, scenes, ob, hctx, monkeypatch):
    GW.test_new_paths_in_several_batches(hostcheck, abi, scenes, ob, hctx, monkeypatch)


def test_dropin_refuses_media_it_does_not_support(hc_plugins, scenes, tmp_path):
    """Error behaviour of the host side: a surface that separates two media, a heterogeneous medium, or a medium under
    `Integrator "path"`'s stricter flattening produce pbrt's `Error:` line and no image -- never a silently wrong render."""
    import subprocess
    fog = dict(sigma_a=(0.05, 0.05, 0.05), sigma_s=(0.2, 0.2, 0.2), g=0.1)
    arr = scenes.SceneArrays(300, materials=("matte",), soup_version=1)

    def run(name, edit, **kw):
        path = scenes.write_pbrt(str(tmp_path), name, arr, 16, 16, 2, max_depth=3, strategy="uniform", **kw)
        text = edit(open(path).read())
        open(path, "w").write(text)
        r = subprocess.run([HC_PLUGIN, "--quiet", os.path.basename(path)], cwd=str(tmp_path), capture_output=True, text=True)
        return r.stdout + r.stderr, os.path.exists(os.path.join(str(tmp_path), name + ".pfm"))

    # a shape whose inside is vacuum while the world outside is fog: a medium transition
    out, wrote = run("transition", lambda t: t.replace('MediumInterface "fog" "fog"', 'MediumInterface "" "fog"'),
                     integrator="volpath", medium=fog)
    assert "separate two media" in out and not wrote, out
    # a heterogeneous medium around the camera
    out, wrote = run("grid", lambda t: t.replace('"string type" "homogeneous"', '"string type" "heterogeneous" "integer nx" [1] '
                                                 '"integer ny" [1] "integer nz" [1] "float density" [1]'),
                     integrator="volpath", medium=fog)
    assert "only homogeneous media" in out and not wrote, out
    # the fine case still renders
    out, wrote = run("fine", lambda t: t, integrator="volpath", medium=fog)
    assert wrote, out



import test_zz_combos_gpu as GC  # noqa: E402


@pytest.mark.parametrize("combo", range(len(GC.COMBOS)))
def test_feature_combinations_vs_oracle(hostcheck, abi, scenes, ob, hctx, combo):
    GC.test_feature_combinations_vs_oracle(hostcheck, abi, scenes, ob, hctx, combo)


@pytest.mark.parametrize("spectral", [False, True])
def test_sample_clamp_crop_and_scale_vs_oracle(hostcheck, abi, scenes, ob, hctx, spectral):
    GW.test_sample_clamp_crop_and_scale_vs_oracle(hostcheck, abi, scenes, ob, hctx, spectral)


@pytest.mark.parametrize("name", sorted(RENDERS))
def test_every_golden_scene_under_sampled_spectrum_vs_oracle(hostcheck, abi, scenes, ob, hctx, name):
    GW.test_every_golden_scene_under_sampled_spectrum_vs_oracle(hostcheck, abi, scenes, ob, hctx, name)


@pytest.mark.parametrize("name", sorted(RENDERS))
def test_every_golden_scene_in_fog_under_volpath_vs_oracle(hostcheck, abi, scenes, ob, hctx, name):
    GW.test_every_golden_scene_in_fog_under_volpath_vs_oracle(hostcheck, abi, scenes, ob, hctx, name)
