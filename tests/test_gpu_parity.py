"""GPU parity tests (run with -m gpu on the H100): the CUDA path through the
C ABI against (1) golden vectors produced by the unmodified reference and
(2) the oracle restatement on the same seeded inputs.  Integer / index results
and float results are compared bit for bit."""
import os

import numpy as np
import pytest

from conftest import GOLDEN, bits, golden_camera, hexf

pytestmark = pytest.mark.gpu

from render_cases import EXTRA, RENDERS  # noqa: E402  (the table shared with tests/golden/make_golden.py)


@pytest.fixture(scope="module")
def ctx(pkg):
    c = pkg.Context(0)
    yield c
    c.close()


def make(pkg, abi, scenes, ctx, nt, mats, w, h, spp, depth=5, strat="uniform", nl=None, seed=1234, **kw):
    arr = scenes.SceneArrays(nt, materials=mats, soup_version=1, n_lights=nl, seed=seed)
    setup = scenes.RenderSetup(w, h, spp, max_depth=depth,
                               strategy={"uniform": abi.LIGHTS_UNIFORM, "power": abi.LIGHTS_POWER, "spatial": abi.LIGHTS_SPATIAL}[strat], **kw)
    scene = pkg.Scene(ctx, arr.desc(), keepalive=arr)
    return arr, setup, scene


def test_sobol_stream_vs_reference(pkg, abi, scenes, ctx, probe_json):
    arr = scenes.SceneArrays(10, materials=("matte",), soup_version=1)
    scene = pkg.Scene(ctx, arr.desc(), keepalive=arr)
    for rec in probe_json["sobol"]:
        b = rec["bounds"]
        setup = scenes.RenderSetup(b[2], b[3], rec["spp"], max_depth=16)
        r = pkg.Render(scene, setup)
        got = r.debug_sobol(rec["px"], rec["py"], rec["sample"], rec["dim0"], len(rec["values"]))
        assert np.array_equal(bits(got), bits(hexf(rec["values"])))
        r.close()
    scene.close()


def test_halton_stream_vs_reference(pkg, abi, scenes, ctx):
    import json
    import os
    arr = scenes.SceneArrays(10, materials=("matte",), soup_version=1)
    scene = pkg.Scene(ctx, arr.desc(), keepalive=arr)
    for rec in json.load(open(os.path.join(scenes.GOLDEN_DIR, "probe_halton.json"))):
        b = rec["bounds"]
        setup = scenes.RenderSetup(b[2], b[3], rec["spp"], max_depth=10, sampler="halton")
        setup.sampler.sample_bounds[:] = b
        setup.film.cropped_bounds[:] = b
        setup.integrator.pixel_bounds[:] = b
        r = pkg.Render(scene, setup)
        got = r.debug_sobol(rec["px"], rec["py"], rec["sample"], rec["dim0"], len(rec["values"]))
        assert np.array_equal(bits(got), bits(hexf(rec["values"])))
        r.close()
    scene.close()


def test_camera_rays_vs_reference(pkg, abi, scenes, ctx, probe_json):
    arr = scenes.SceneArrays(10, materials=("matte",), soup_version=1)
    scene = pkg.Scene(ctx, arr.desc(), keepalive=arr)
    for rec in probe_json["camrays"]:
        w, h = rec["res"]
        setup = scenes.RenderSetup(w, h, rec["spp"], camera=golden_camera(abi, probe_json, w, h))
        r = pkg.Render(scene, setup)
        got = r.debug_camera_rays(rec["px"], rec["py"], len(rec["rays"]))
        want = np.array([hexf(x) for x in rec["rays"]])
        assert np.array_equal(bits(got["o"]), bits(want[:, 0:3]))
        assert np.array_equal(bits(got["d"]), bits(want[:, 3:6]))
        assert np.array_equal(bits(got["t_max"]), bits(want[:, 6]))
        r.close()
    scene.close()


def test_intersections_vs_reference_bvhaccel(pkg, abi, scenes, ctx):
    rays = np.load(os.path.join(GOLDEN, "isect_rays.npy"))
    ref = np.load(os.path.join(GOLDEN, "isect_ref.npy"))
    arr = scenes.SceneArrays(3000, materials=("matte",), soup_version=1, seed=99)
    scene = pkg.Scene(ctx, arr.desc(), keepalive=arr)
    hits = scene.trace_closest(rays)
    assert np.array_equal(hits["triangle"], ref["tri"])
    m = ref["tri"] >= 0
    assert np.array_equal(bits(hits["t"][m]), bits(ref["t"][m]))
    assert np.array_equal(scene.trace_any(rays).astype(np.int32), ref["occluded"])
    scene.close()


@pytest.mark.parametrize("n_tris,n_rays", [(1, 2000), (37, 20000), (20000, 200000), (400000, 400000)])
def test_trace_vs_oracle(pkg, abi, scenes, ob, ctx, n_tris, n_rays):
    arr = scenes.SceneArrays(n_tris, materials=("matte",), soup_version=1, seed=n_tris)
    scene = pkg.Scene(ctx, arr.desc(), keepalive=arr)
    o = ob.Oracle(abi, arr)
    rng = np.random.default_rng(n_rays)
    rays = np.zeros(n_rays, dtype=abi.RAY_DTYPE)
    rays["o"] = rng.uniform(-1.5, 1.5, (n_rays, 3)).astype(np.float32)
    rays["d"] = rng.normal(size=(n_rays, 3)).astype(np.float32)
    rays["t_max"] = np.inf
    rays["t_max"][::3] = rng.uniform(0.05, 2.0, len(rays[::3])).astype(np.float32)
    rays["d"][::17, 0] = 0.0                      # axis-parallel components
    rays["d"][5::101] = [0.0, 0.0, 1.0]           # axis-aligned rays
    tgt = arr.vertices[rng.integers(0, arr.n_triangles, len(rays[7::31])), 0]
    rays["d"][7::31] = tgt - rays["o"][7::31]     # aimed exactly at vertices
    got, want = scene.trace_closest(rays), o.trace_closest(rays)
    same = got["triangle"] == want["triangle"]
    # an exact-t tie may pick the other of two triangles; everything else must be identical
    tie = ~same & (got["triangle"] >= 0) & (want["triangle"] >= 0) & (bits(got["t"]) == bits(want["t"]))
    assert (same | tie).all(), "%d rays disagree" % (~(same | tie)).sum()
    aimed = np.zeros(len(rays), bool)
    aimed[7::31] = True  # rays aimed at a vertex shared by the two triangles of a light quad tie by design
    assert not (tie & ~aimed).any()
    hit = same & (want["triangle"] >= 0)
    assert hit.sum() > 0
    for k in ("t", "b0", "b1"):
        assert np.array_equal(bits(got[k][hit]), bits(want[k][hit])), k
    assert np.array_equal(scene.trace_any(rays), o.trace_any(rays))
    o.close()
    scene.close()


def test_trace_spheres_vs_oracle(pkg, abi, scenes, ob, ctx):
    """Scene::Intersect / IntersectP with Sphere shapes next to the triangle soup: a sphere hit is reported as
    primitive n_triangles + k with Sphere::Intersect's tHit (EFloat quadratic), bit-exact."""
    spheres = (dict(center=(1.2, 1.8, -1.5), radius=0.35, emit=60.0),
               dict(center=(0.1, 0.0, -0.2), radius=0.45, material="matte"),
               dict(center=(-0.9, -0.6, 0.3), radius=0.4, material="matte", scale=(1.3, 0.7, -1.1)),
               dict(center=(0.6, -0.3, 0.9), radius=0.3, material="matte", reverse_orientation=True))
    for n_tris in (0, 4000):
        arr = scenes.SceneArrays(n_tris, materials=("matte",), soup_version=1, seed=11, n_lights=0, spheres=spheres)
        scene = pkg.Scene(ctx, arr.desc(), keepalive=arr)
        o = ob.Oracle(abi, arr)
        n_rays = 60000
        rng = np.random.default_rng(5)
        rays = np.zeros(n_rays, dtype=abi.RAY_DTYPE)
        rays["o"] = rng.uniform(-1.5, 1.5, (n_rays, 3)).astype(np.float32)
        rays["d"] = rng.normal(size=(n_rays, 3)).astype(np.float32)
        rays["t_max"] = np.inf
        rays["t_max"][::3] = rng.uniform(0.05, 2.0, len(rays[::3])).astype(np.float32)
        rays["o"][::7] = np.array([0.1, 0.0, -0.2], np.float32) + rng.uniform(-0.2, 0.2, (len(rays[::7]), 3)).astype(np.float32)
        got, want = scene.trace_closest(rays), o.trace_closest(rays)
        assert np.array_equal(got["triangle"], want["triangle"])
        assert (want["triangle"] >= arr.n_triangles).sum() > 1000
        assert np.array_equal(bits(got["t"]), bits(want["t"]))
        assert np.array_equal(scene.trace_any(rays), o.trace_any(rays))
        o.close()
        scene.close()


def test_trace_instances_vs_oracle(pkg, abi, scenes, ob, ctx):
    """TransformedPrimitive::Intersect / IntersectP: rays are transformed into the object, the object's own tree is
    traversed, the hit is reported with the object triangle's index and the object-space t, bit-exact."""
    objects = (dict(n_tris=600, seed=5, material="matte", size=0.35), dict(n_tris=200, seed=9, material="matte", size=0.5))
    instances = (dict(object=0, center=(0.0, 0.0, -0.4)), dict(object=0, center=(0.9, 0.6, 0.2), scale=(0.7, 1.4, 1.0)),
                 dict(object=1, center=(-0.8, -0.5, 0.0), scale=(1.0, 1.0, -1.3)), dict(object=1),
                 dict(object=0, center=(-0.9, 0.7, 0.4), scale=(1.5, 1.5, 1.5)))
    # 5 instances are tested one by one; 40 go through the tree over their leaf boxes
    lattice = tuple(dict(object=k % 2, center=(-0.9 + 0.45 * (k % 5), -0.7 + 0.45 * ((k // 5) % 4), -0.5 + 0.9 * (k // 20)),
                         scale=(0.5, 0.5, -0.5 if k % 3 == 0 else 0.5)) for k in range(40))
    # the same lattice under rotations about oblique axes in three step orders, every third one mirrored: full 3x3 linear
    # parts (non-orthogonal ones for T S R) in the ray transform, its error offset and the instances' world boxes
    affine = tuple(dict(ins, scale=(0.5, 0.4 + 0.05 * (k % 4), ins["scale"][2]), rotate=((17.0 + 23.0 * k) % 360, 1.0, k % 7 - 3.0,
                                                                                           0.5 + k % 3), order=("TSR", "TRS", "RTS")[k % 3])
                   for k, ins in enumerate(lattice))
    for n_tris, instances in ((0, instances), (3000, instances), (3000, lattice), (3000, affine)):
        arr = scenes.SceneArrays(n_tris, materials=("matte",), soup_version=1, seed=21, n_lights=0, objects=objects,
                                 instances=instances)
        scene = pkg.Scene(ctx, arr.desc(), keepalive=arr)
        o = ob.Oracle(abi, arr)
        n_rays = 60000
        rng = np.random.default_rng(6)
        rays = np.zeros(n_rays, dtype=abi.RAY_DTYPE)
        rays["o"] = rng.uniform(-1.5, 1.5, (n_rays, 3)).astype(np.float32)
        rays["d"] = rng.normal(size=(n_rays, 3)).astype(np.float32)
        rays["t_max"] = np.inf
        rays["t_max"][::3] = rng.uniform(0.05, 2.0, len(rays[::3])).astype(np.float32)
        rays["d"][::17, 2] = 0.0   # becomes -0.0 inside the mirrored instance
        got, want = scene.trace_closest(rays), o.trace_closest(rays)
        same = got["triangle"] == want["triangle"]
        tie = ~same & (got["triangle"] >= 0) & (want["triangle"] >= 0) & (bits(got["t"]) == bits(want["t"]))
        assert (same | tie).all(), "%d rays disagree" % (~(same | tie)).sum()
        assert (want["triangle"] >= arr.n_toplevel).sum() > 1000
        hit = same & (want["triangle"] >= 0)
        assert np.array_equal(bits(got["t"][hit]), bits(want["t"][hit]))
        assert np.array_equal(scene.trace_any(rays), o.trace_any(rays))
        o.close()
        scene.close()


def test_device_bvh_build(pkg, abi, scenes, ob, monkeypatch):
    """SURVEY 8f row 1: the on-device builder (Morton order -> binary radix tree -> 8-wide collapse).  The tree passes
    the structural validation, traversal answers equal the oracle's (and the host-built tree's) bit for bit, and a
    render through it is identical to the reference PFM."""
    monkeypatch.setenv("B200PT_VALIDATE_BVH", "1")
    gctx = pkg.Context(0)
    gctx.set_option("gpu_bvh_build", 1)
    for n_tris in (0, 1, 2, 5, 3000, 120000):
        arr = scenes.SceneArrays(n_tris, materials=("matte",), soup_version=1, seed=n_tris + 3)
        if n_tris >= 5:  # never-hittable triangles must stay out of the tree but keep their records
            arr.vertices[3] = arr.vertices[3][0]
        scene = pkg.Scene(gctx, arr.desc(), keepalive=arr)
        o = ob.Oracle(abi, arr)
        n_rays = 40000
        rng = np.random.default_rng(n_tris)
        rays = np.zeros(n_rays, dtype=abi.RAY_DTYPE)
        rays["o"] = rng.uniform(-1.5, 1.5, (n_rays, 3)).astype(np.float32)
        rays["d"] = rng.normal(size=(n_rays, 3)).astype(np.float32)
        rays["t_max"] = np.inf
        rays["t_max"][::3] = rng.uniform(0.05, 2.0, len(rays[::3])).astype(np.float32)
        rays["o"][::5] = [0, 0, -4.5]
        got, want = scene.trace_closest(rays), o.trace_closest(rays)
        same = got["triangle"] == want["triangle"]
        tie = ~same & (got["triangle"] >= 0) & (want["triangle"] >= 0) & (bits(got["t"]) == bits(want["t"]))
        assert (same | tie).all(), "%d rays disagree (n_tris %d)" % ((~(same | tie)).sum(), n_tris)
        hit = same & (want["triangle"] >= 0)
        for k in ("t", "b0", "b1"):
            assert np.array_equal(bits(got[k][hit]), bits(want[k][hit])), k
        assert np.array_equal(scene.trace_any(rays), o.trace_any(rays))
        o.close()
        scene.close()
    for name in ("four", "normals_uv", "spheres"):
        nt, mats, w, h, spp, depth, strat, nl = RENDERS[name]
        ex = EXTRA.get(name, {})
        arr = scenes.SceneArrays(nt, materials=mats, soup_version=1, n_lights=nl, **ex.get("scene", {}))
        setup = scenes.RenderSetup(w, h, spp, max_depth=depth,
                                   strategy={"uniform": abi.LIGHTS_UNIFORM, "power": abi.LIGHTS_POWER,
                                             "spatial": abi.LIGHTS_SPATIAL}[strat], **ex.get("camera", {}))
        scene = pkg.Scene(gctx, arr.desc(), keepalive=arr)
        r = pkg.Render(scene, setup)
        r.render_tiles()
        ref = scenes.read_pfm(os.path.join(GOLDEN, "render_%s.pfm" % name))
        assert np.array_equal(bits(r.read_rgb()), bits(ref)), name
        r.close()
        scene.close()
    gctx.close()


def test_empty_and_ragged_inputs(pkg, abi, scenes, ctx):
    arr = scenes.SceneArrays(500, materials=("matte",), soup_version=1)
    scene = pkg.Scene(ctx, arr.desc(), keepalive=arr)
    assert len(scene.trace_closest(np.zeros(0, dtype=abi.RAY_DTYPE))) == 0
    rays = np.zeros(33, dtype=abi.RAY_DTYPE)        # not a multiple of the warp size
    rays["o"] = [0, 0, -4.5]
    rays["d"] = [0, 0, 1]
    rays["t_max"] = np.inf
    h = scene.trace_closest(rays)
    assert (h["triangle"] == h["triangle"][0]).all()
    setup = scenes.RenderSetup(17, 9, 2)            # partial tiles in x and y
    r = pkg.Render(scene, setup)
    r.render_tiles()
    raw = r.read_raw()
    assert raw.shape == (9, 17, 4) and np.all(raw[..., 3] >= 2)
    r.close()
    scene.close()


@pytest.mark.parametrize("name", sorted(RENDERS))
def test_render_vs_reference_pfm(pkg, abi, scenes, ob, ctx, name):
    nt, mats, w, h, spp, depth, strat, nl = RENDERS[name]
    ex = EXTRA.get(name, {})
    arr = scenes.SceneArrays(nt, materials=mats, soup_version=1, n_lights=nl, **ex.get("scene", {}))
    setup = scenes.RenderSetup(w, h, spp, max_depth=depth,
                               strategy={"uniform": abi.LIGHTS_UNIFORM, "power": abi.LIGHTS_POWER, "spatial": abi.LIGHTS_SPATIAL}[strat],
                               **ex.get("camera", {}))
    scene = pkg.Scene(ctx, arr.desc(), keepalive=arr)
    r = pkg.Render(scene, setup)
    r.render_tiles()
    rgb = r.read_rgb()
    ref = scenes.read_pfm(os.path.join(GOLDEN, "render_%s.pfm" % name))
    nbad = int((bits(rgb) != bits(ref)).sum())
    if nbad:
        o = ob.Oracle(abi, arr)
        ys, xs, _ = np.nonzero(bits(rgb) != bits(ref))
        y, x = int(ys[0]), int(xs[0])
        print("first differing pixel", x, y, rgb[y, x], ref[y, x])
        print("gpu samples", r.debug_pixel_samples(x, y))
        print("oracle samples", o.pixel_samples(setup, x, y))
    assert nbad == 0, "%d of %d components differ from the reference render" % (nbad, rgb.size)
    st = r.stats()
    cb = setup.sample_bounds
    assert st["camera_rays"] == (cb[2] - cb[0]) * (cb[3] - cb[1]) * setup.sampler.samples_per_pixel
    r.close()
    scene.close()


@pytest.mark.parametrize("mats,depth,strat", [(("matte",), 5, "uniform"), (("glass",), 8, "uniform"),
                                             (("metal",), 5, "power"), (("plastic",), 5, "spatial"),
                                             (("matte", "glass", "metal", "plastic"), 16, "power"),
                                             (("matte", "glass", "metal", "plastic"), 5, "spatial"),
                                             (("matte_rough", "glass_rough"), 8, "uniform")])
def test_render_and_counters_vs_oracle(pkg, abi, scenes, ob, ctx, mats, depth, strat):
    arr, setup, scene = make(pkg, abi, scenes, ctx, 60000, mats, 96, 64, 16, depth, strat)
    o = ob.Oracle(abi, arr)
    film, ostats = o.render(setup)
    r = pkg.Render(scene, setup)
    r.render_tiles()
    raw = r.read_raw()
    nbad = int((bits(raw) != bits(film)).sum())
    if nbad:
        ys, xs, _ = np.nonzero(bits(raw) != bits(film))
        y, x = int(ys[0]), int(xs[0])
        print("first differing pixel", x, y, raw[y, x], film[y, x])
        g, w_ = r.debug_pixel_samples(x, y), o.pixel_samples(setup, x, y)
        print("differing samples", np.nonzero((bits(g) != bits(w_)).any(axis=1))[0], g[:4], w_[:4])
    assert nbad == 0, "%d of %d raw film values differ from the oracle" % (nbad, raw.size)
    st = r.stats()
    for k in ("camera_rays", "regular_rays", "shadow_rays"):
        assert st[k] == ostats[k], (k, st[k], ostats[k])
    assert np.array_equal(bits(r.read_rgb()), bits(o.film_rgb(setup, film)))
    o.close()
    r.close()
    scene.close()


def test_pixel_samples_vs_oracle(pkg, abi, scenes, ob, ctx):
    arr, setup, scene = make(pkg, abi, scenes, ctx, 30000, ("matte", "glass", "metal", "plastic"), 64, 64, 64, 8)
    o = ob.Oracle(abi, arr)
    r = pkg.Render(scene, setup)
    for (x, y) in [(0, 0), (31, 17), (63, 63), (40, 5)]:
        assert np.array_equal(bits(r.debug_pixel_samples(x, y)), bits(o.pixel_samples(setup, x, y)))
    o.close()
    r.close()
    scene.close()


def test_tile_shards_sum_to_full_render(pkg, abi, scenes, ctx):
    """SURVEY 8(e): disjoint tile sets rendered with the full-film sampler add up to the full film."""
    arr, setup, scene = make(pkg, abi, scenes, ctx, 20000, ("matte", "plastic"), 80, 48, 8)
    r = pkg.Render(scene, setup)
    r.render_tiles()
    full = r.read_raw()
    parts = []
    for k in range(3):
        r.clear()
        r.render_tiles(np.arange(r.n_tiles)[k::3])
        parts.append(r.read_raw())
    assert np.array_equal(bits(parts[0] + parts[1] + parts[2]), bits(full))
    # pixelbounds sharding (path.cpp:195-207): left/right halves
    halves = []
    for pb in ([0, 0, 40, 48], [40, 0, 80, 48]):
        s2 = scenes.RenderSetup(80, 48, 8, pixel_bounds=pb)
        r2 = pkg.Render(scene, s2)
        r2.render_tiles()
        halves.append(r2.read_raw())
        r2.close()
    # interior pixels are bit-identical; a pixel next to the cut can receive a box-filter bleed from the other
    # shard, which is then added after the RGB->XYZ conversion instead of before (same as the reference, SURVEY 5)
    both = halves[0] + halves[1]
    interior = np.ones(80, bool)
    interior[39:41] = False
    assert np.array_equal(bits(both[:, interior]), bits(full[:, interior]))
    assert np.allclose(both, full, rtol=1e-5, atol=1e-6)
    r.close()
    scene.close()


def test_render_is_deterministic_and_batch_independent(pkg, abi, scenes, ctx, monkeypatch):
    arr, setup, scene = make(pkg, abi, scenes, ctx, 20000, ("matte", "glass"), 64, 64, 16)
    r = pkg.Render(scene, setup)
    r.render_tiles()
    a = r.read_raw()
    r.clear()
    r.render_tiles()
    assert np.array_equal(bits(a), bits(r.read_raw()))
    r.close()
    monkeypatch.setenv("B200PT_BATCH_PATHS", str(256 * 16 * 3))  # 3 tiles per batch
    r = pkg.Render(scene, setup)
    r.render_tiles()
    assert np.array_equal(bits(a), bits(r.read_raw()))
    r.close()
    scene.close()


@pytest.mark.parametrize("name", ["analytic_point", "analytic_4points", "analytic_area"])
def test_analytic_scenes_known_answer(pkg, abi, scenes, ctx, name):
    """src/tests/analytic_scenes.cpp: camera inside a unit sphere of Kd 0.5 lit from its centre (or emitting 0.5):
    the image mean is 1 +- 0.02 (CheckSceneAverage, :54-66)."""
    nt, mats, w, h, spp, depth, strat, nl = RENDERS[name]
    ex = EXTRA[name]
    arr = scenes.SceneArrays(nt, materials=mats, soup_version=1, n_lights=nl, **ex["scene"])
    setup = scenes.RenderSetup(w, h, spp, max_depth=depth, strategy=abi.LIGHTS_SPATIAL, **ex["camera"])
    scene = pkg.Scene(ctx, arr.desc(), keepalive=arr)
    r = pkg.Render(scene, setup)
    r.render_tiles()
    assert abs(float(r.read_rgb().mean()) - 1.0) < 0.02
    r.close()
    scene.close()


def test_pixel_filter_many_batches_and_shards(pkg, abi, scenes, ctx, monkeypatch):
    """Wide pixel filters with the film split over many wavefront batches (the tiles of a batch are merged in tile
    order, batches follow each other in tile order) and over two tile shards: the first must stay bit-identical to
    the single-threaded reference image, the shard sum must equal it up to the order of the float additions."""
    nt, mats, w, h, spp, depth, strat, nl = RENDERS["filter_gaussian"]
    arr = scenes.SceneArrays(nt, materials=mats, soup_version=1, n_lights=nl)
    setup = scenes.RenderSetup(w, h, spp, max_depth=depth, strategy=abi.LIGHTS_SPATIAL, pixel_filter="gaussian")
    scene = pkg.Scene(ctx, arr.desc(), keepalive=arr)
    ref = scenes.read_pfm(os.path.join(GOLDEN, "render_filter_gaussian.pfm"))
    monkeypatch.setenv("B200PT_BATCH_PATHS", str(256 * spp * 2))  # two tiles per batch
    r = pkg.Render(scene, setup)
    r.render_tiles()
    assert np.array_equal(bits(r.read_rgb()), bits(ref))
    full = r.read_raw()
    r.clear()
    tiles = np.arange(r.n_tiles, dtype=np.int32)
    r.render_tiles(tiles[0::2])
    a = r.read_raw()
    r.clear()
    r.render_tiles(tiles[1::2])
    b = r.read_raw()
    np.testing.assert_allclose(a + b, full, rtol=2e-6, atol=1e-7)
    r.close()
    scene.close()


def test_large_scene_properties(pkg, abi, scenes, ctx):
    """BASELINE-size scene (1M triangles): properties that need no CPU oracle at full size."""
    arr, setup, scene = make(pkg, abi, scenes, ctx, 1000000, ("matte",), 256, 256, 4)
    rng = np.random.default_rng(3)
    n = 300000
    rays = np.zeros(n, dtype=abi.RAY_DTYPE)
    rays["o"] = rng.uniform(-1, 1, (n, 3)).astype(np.float32)
    rays["d"] = rng.normal(size=(n, 3)).astype(np.float32)
    rays["t_max"] = np.inf
    h = scene.trace_closest(rays)
    hit = h["triangle"] >= 0
    assert 0.3 < hit.mean() < 1.0
    # a hit found with t_max = inf must also be found with t_max slightly above t, and be occluding
    r2 = rays[hit].copy()
    r2["t_max"] = np.nextafter(h["t"][hit], np.float32(np.inf))
    h2 = scene.trace_closest(r2)
    assert np.array_equal(h2["triangle"], h["triangle"][hit]) and np.array_equal(bits(h2["t"]), bits(h["t"][hit]))
    assert scene.trace_any(r2).all()
    # and nothing is hit strictly before it
    r3 = rays[hit].copy()
    r3["t_max"] = h["t"][hit] * np.float32(1 - 1e-4)  # well below t: the scaled range test (triangle.cpp:258-261) is not ulp-exact
    assert not (scene.trace_closest(r3)["triangle"] == h["triangle"][hit]).any()
    # reconstruct the hit point from the barycentrics: must lie on the ray
    v = arr.vertices[h["triangle"][hit]]
    b0, b1 = h["b0"][hit, None], h["b1"][hit, None]
    p = b0 * v[:, 0] + b1 * v[:, 1] + (1 - b0 - b1) * v[:, 2]
    q = rays["o"][hit] + h["t"][hit, None] * rays["d"][hit]
    assert np.abs(p - q).max() < 1e-3
    r = pkg.Render(scene, setup)
    r.render_tiles()
    raw = r.read_raw()
    assert np.isfinite(raw).all() and (raw[..., 3] >= 4).all() and raw[..., 1].mean() > 0
    r.close()
    scene.close()


def watertight_mesh(rng, n_theta=16, n_phi=16):
    """The closed mesh of the reference's Triangle.Watertight test (src/tests/shapes.cpp:28-93): a triangulated sphere whose
    vertices are pushed out randomly along their normals; pole vertices and the seam coincide exactly."""
    verts = []
    for t in range(n_theta):
        theta = np.float32(np.pi) * np.float32(t) / np.float32(n_theta - 1)
        for p in range(n_phi):
            phi = np.float32(2 * np.pi) * np.float32(p) / np.float32(n_phi - 1)
            if t == 0:
                verts.append((0.0, 0.0, 1.0))
            elif t == n_theta - 1:
                verts.append((0.0, 0.0, -1.0))
            elif p == n_phi - 1:
                verts.append(verts[len(verts) - (n_phi - 1)])
            else:
                r = 1.0 + 5.0 * rng.random()
                verts.append((r * np.sin(theta) * np.cos(phi), r * np.sin(theta) * np.sin(phi), r * np.cos(theta)))
    verts = np.array(verts, np.float32)
    off = lambda t, p: t * n_phi + p  # noqa: E731
    idx = []
    for p in range(n_phi - 1):
        idx += [off(0, 0), off(1, p), off(1, p + 1)]
    for t in range(1, n_theta - 2):
        for p in range(n_phi - 1):
            idx += [off(t, p), off(t + 1, p), off(t + 1, p + 1), off(t, p), off(t + 1, p + 1), off(t, p + 1)]
    for p in range(n_phi - 1):
        idx += [off(n_theta - 1, 0), off(n_theta - 2, p), off(n_theta - 2, p + 1)]
    return verts, verts[np.array(idx).reshape(-1, 3)]


def test_triangle_watertight(pkg, abi, scenes, ctx):
    """Triangle.Watertight of the reference's test-suite (src/tests/shapes.cpp:28-128) for the traversal kernels: 100 000 rays
    from inside a closed, randomly perturbed mesh -- in random directions and aimed exactly at mesh vertices -- must all hit
    (closest-hit and any-hit)."""
    rng = np.random.default_rng(12111)
    verts, tris = watertight_mesh(rng)
    arr = scenes.SceneArrays(len(tris), materials=("matte",), soup_version=1, n_lights=0)
    assert arr.vertices.shape == tris.shape
    arr.vertices[:] = tris
    scene = pkg.Scene(ctx, arr.desc(), keepalive=arr)
    n = 100000

    def sphere(k):
        z = 1 - 2 * rng.random(k)
        r = np.sqrt(np.maximum(0, 1 - z * z))
        phi = 2 * np.pi * rng.random(k)
        return np.stack([r * np.cos(phi), r * np.sin(phi), z], 1).astype(np.float32)
    rays = np.zeros(2 * n, dtype=abi.RAY_DTYPE)
    rays["o"][:n] = rays["o"][n:] = np.float32(0.5) * sphere(n)
    rays["d"][:n] = sphere(n)
    rays["d"][n:] = verts[rng.integers(0, len(verts), n)] - rays["o"][n:]   # tougher: directly at a vertex
    rays["t_max"] = np.inf
    hits = scene.trace_closest(rays)
    assert (hits["triangle"] >= 0).all(), "%d rays leaked through the mesh" % (hits["triangle"] < 0).sum()
    assert scene.trace_any(rays).all()
    scene.close()
