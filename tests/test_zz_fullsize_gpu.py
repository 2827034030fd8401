"""Benchmark-size renders against the oracle (collected last, like the other test_zz files; tests/test_hostcheck.py
replays the same functions against the CPU check build at a small film).

Every other comparison with an independent reference renders one wavefront batch with fewer paths than the persistent
grids have lanes.  The benchmark's jobs run many batches with a partial last one, slot indices up to 96 Mi - 1, queue
counts that make the persistent warps refill thousands of times, half-height tiles on the bottom row of a 1080-line
film and pixel coordinates above 1024, where pFilm = px + u rounds up to the neighbour often enough to bleed across
tile borders.  Each test here takes one workload's film, samples, depth, materials, lights, strategy, sampler and box
filter with a smaller scene, renders a tile set T that touches those places against the oracle, then the whole film at
the default batch sizing, at another batch size and (RGB) twice, and compares the images bit for bit.

Pixels next to a corner where three or four rendered tiles meet take box-filter bleed from each of them; k_film adds a
tile's contribution with atomicAdd, the oracle in tile order (DESIGN.md section 2), so those pixels are compared with a
tight tolerance and the number that differed is printed.  Every other pixel is compared bit for bit."""
import json
import os
import time

import numpy as np
import pytest

from conftest import GOLDEN, bits
from test_gpu_parity import ctx  # noqa: F401  (module-scoped context fixture)

pytestmark = pytest.mark.gpu

MATS4 = ("matte", "glass", "metal", "plastic")


def tiles_per_batch(n_tiles, spp, spectral):
    """The batch rule of b200pt_render_create (api.cu): whole 16x16 tiles of 256 * spp path slots, about
    B200PT_BATCH_PATHS slots per batch -- 96 Mi by default, 16 Mi with a 60-bin host --, at least one tile and at most
    the film."""
    target = int(os.environ.get("B200PT_BATCH_PATHS", (16 << 20) if spectral else (96 << 20)))
    return min(max(1, target // (256 * spp)), n_tiles)


def n_batches(n_tiles, tpb):
    return -(-n_tiles // tpb)


def tile_set(tiles_x, tiles_y, tpb, n_random=5, seed=2024):
    """The first tile, the last one of the top row, the first and last of the bottom row, the last tile of batch 0 and
    the first of batch 1, the first and last of the last batch, a 2x2 block at x >= 1024, y >= 512 (or as close to it
    as the film allows) and a few seeded random tiles, sorted."""
    n = tiles_x * tiles_y
    nb = n_batches(n, tpb)
    bx, by = min(1024 // 16, tiles_x - 2), min(512 // 16, tiles_y - 2)
    block = [by * tiles_x + bx, by * tiles_x + bx + 1, (by + 1) * tiles_x + bx, (by + 1) * tiles_x + bx + 1]
    fixed = {0, tiles_x - 1, (tiles_y - 1) * tiles_x, n - 1, tpb - 1, tpb, (nb - 1) * tpb} | set(block)
    rng = np.random.default_rng(seed)
    t = set(fixed)
    while len(t) < len(fixed) + n_random:
        t.add(int(rng.integers(0, n)))
    return np.array(sorted(t), np.int32)


def junction_pixels(width, height, tiles_x, tiles_y, rendered):
    """The 2x2 pixels around each corner where at least three rendered tiles meet."""
    r = np.zeros(tiles_x * tiles_y, np.int32)
    r[rendered] = 1
    r = r.reshape(tiles_y, tiles_x)
    corners = (r[:-1, :-1] + r[:-1, 1:] + r[1:, :-1] + r[1:, 1:]) >= 3  # corner (j + 1, i + 1) in tile units
    m = np.zeros((height, width), bool)
    for j, i in zip(*np.nonzero(corners)):
        y, x = 16 * (j + 1), 16 * (i + 1)
        m[y - 1:y + 1, x - 1:x + 1] = True
    return m


def tile_pixels(width, height, tiles_x, tiles, ring):
    """Pixels of the given tiles: their one-pixel border ring (ring=True) or what lies inside it."""
    m = np.zeros((height, width), bool)
    for t in tiles:
        x0, y0 = 16 * (t % tiles_x), 16 * (t // tiles_x)
        x1, y1 = min(x0 + 16, width), min(y0 + 16, height)
        inner = np.zeros((y1 - y0, x1 - x0), bool)
        inner[1:-1, 1:-1] = True
        m[y0:y1, x0:x1] = ~inner if ring else inner
    return m


def compare(what, got, want, loose, explain, region=None):
    """Over `region` (default: the whole film), bit for bit outside `loose` and tightly close inside it; returns how many
    `loose` pixels differed."""
    diff = (bits(got) != bits(want)).any(axis=2)
    if region is not None:
        diff &= region
        loose = loose & region
    strict = diff & ~loose
    if strict.any():
        ys, xs = np.nonzero(strict)
        explain(what, int(xs[0]), int(ys[0]), got, want)
    assert not strict.any(), "%s: %d pixels differ (outside the multi-tile corners)" % (what, int(strict.sum()))
    np.testing.assert_allclose(got[loose], want[loose], rtol=1e-5, atol=1e-5, err_msg=what + ": multi-tile corner pixels")
    n = int((diff & loose).sum())
    if loose.any():
        print("%s: %d of %d multi-tile corner pixels differ in the last bits" % (what, n, int(loose.sum())))
    return n


def check_fullsize(pkg, abi, ob, ctx, monkeypatch, arr, setup, medium, batch_tiles, other_batch, repeat):
    """(1) T against the oracle, (2) the full film at the default batch sizing, (4) repeated on the same Render when
    `repeat`, (3) a new Render at `other_batch` tiles per batch when given.  `batch_tiles` (CPU replays) sets the
    default batch size in tiles."""
    t_start = time.time()
    spectral = getattr(arr, "cie_xyz", None) is not None
    volpath = setup.integrator.volumetric != 0
    spp = setup.sampler.samples_per_pixel
    if batch_tiles:
        monkeypatch.setenv("B200PT_BATCH_PATHS", str(batch_tiles * 256 * spp))
    scene = pkg.Scene(ctx, arr.desc(), keepalive=arr)
    o = ob.Oracle(abi, arr)
    ob.set_volpath(o.lib, volpath, medium)
    r = None
    try:
        r = pkg.Render(scene, setup)
        W, H, tx, ty = r.width, r.height, r.tiles_x, r.tiles_y
        n = r.n_tiles
        tpb = tiles_per_batch(n, spp, spectral)
        nb = n_batches(n, tpb)
        assert nb > 1, "the film fits one batch: %d tiles of %d" % (n, tpb)
        T = tile_set(tx, ty, tpb)
        print("%dx%d, %d spp: %d tiles, %d per batch, %d batches (last %d tiles); T = %s" %
              (W, H, spp, n, tpb, nb, n - (nb - 1) * tpb, T.tolist()))

        def explain(what, x, y, got, want):
            print(what, "first differing pixel", x, y, got[y, x], want[y, x])
            print("gpu samples", r.debug_pixel_samples(x, y)[:8])
            print("oracle samples", o.pixel_samples(setup, x, y)[:8])

        def counters_agree(st, ost):
            assert st["camera_rays"] == ost["camera_rays"], (st["camera_rays"], ost["camera_rays"])
            if volpath:  # VisibilityTester::Tr goes through Scene::Intersect: shadow rays are counted as regular ones
                assert st["regular_rays"] + st["shadow_rays"] == ost["regular_rays"] + ost["shadow_rays"]
            else:
                for k in ("regular_rays", "shadow_rays"):
                    assert st[k] == ost[k], (k, st[k], ost[k])

        def no_overflows(st):
            assert st["stack_overflows"] == 0 and st["dimension_overflows"] == 0, st

        # (1) T on the device and in the oracle: the whole film bit for bit, the ray counters equal
        t0 = time.time()
        film_o, ost = o.render(setup, tiles=T)
        t1 = time.time()
        r.clear()
        r.render_tiles(T)
        sub = r.read_raw()  # waits for the render
        print("oracle %.1f s, device %.2f s for T" % (t1 - t0, time.time() - t1))
        st = r.stats()
        corners = {"T vs oracle": compare("T vs oracle", sub, film_o, junction_pixels(W, H, tx, ty, T), explain)}
        counters_agree(st, ost)
        no_overflows(st)
        nb_T = n_batches(len(T), tpb)
        assert st["closest_launches"] % nb_T == 0
        per_batch = st["closest_launches"] // nb_T  # 1 + 2 max_depth without bounded media, whatever the batch holds

        # (2) the full film at the default batch sizing
        everything = np.arange(n, dtype=np.int32)
        all_corners = junction_pixels(W, H, tx, ty, everything)
        r.reset_stats()
        r.clear()
        r.render_tiles()
        full = r.read_raw()
        st_full = r.stats()
        assert st_full["camera_rays"] == W * H * spp
        assert st_full["closest_launches"] == nb * per_batch, (st_full["closest_launches"], nb, per_batch)
        no_overflows(st_full)
        assert (full[..., 3] >= spp).all(), "pixels without all their samples: %d" % int((full[..., 3] < spp).sum())
        # Inside the border ring of a tile of T only that tile contributes.  The ring also takes the bleed of tiles
        # outside T: each bleeding sample adds 1 to the weight, so where the weights agree the same samples arrived and
        # the values must agree too; elsewhere only a few extra samples may have arrived.
        inner, ring = tile_pixels(W, H, tx, T, False), tile_pixels(W, H, tx, T, True)
        compare("full film vs T (tile interiors)", full, sub, np.zeros_like(inner), explain, region=inner)
        same_w = full[..., 3] == sub[..., 3]
        compare("full film vs T (tile rings without outside bleed)", full, sub, all_corners, explain, region=ring & same_w)
        extra = (full[..., 3] - sub[..., 3])[ring & ~same_w]
        assert (extra > 0).all() and (extra <= 2 + spp // 64).all(), np.unique(extra)
        print("ring pixels with bleed from outside T: %d of %d" % (len(extra), int(ring.sum())))

        # (4) the same film again on the same Render
        if repeat:
            r.reset_stats()
            r.clear()
            r.render_tiles()
            corners["repeat"] = compare("repeat", r.read_raw(), full, all_corners, explain)
            assert r.stats()["camera_rays"] == st_full["camera_rays"]

        # (3) another batch split: one large Render at a time on a shared card
        if other_batch:
            r.close()
            monkeypatch.setenv("B200PT_BATCH_PATHS", str(other_batch * 256 * spp))
            r = pkg.Render(scene, setup)
            nb2 = n_batches(n, tiles_per_batch(n, spp, spectral))
            assert nb2 != nb
            r.clear()
            r.render_tiles()
            corners["%d tiles per batch" % other_batch] = compare("%d tiles per batch" % other_batch, r.read_raw(), full,
                                                                  all_corners, explain)
            st2 = r.stats()
            for k in ("camera_rays", "regular_rays", "shadow_rays"):
                assert st2[k] == st_full[k], (k, st2[k], st_full[k])
            assert st2["closest_launches"] == nb2 * per_batch
            no_overflows(st2)
        print("batches asserted: %d; corner pixels that differed: %s; %.1f s" % (nb, corners, time.time() - t_start))
    finally:
        ob.set_volpath(o.lib, False)
        if r is not None:
            r.close()
        scene.close()
        o.close()


def test_fullsize_rgb_cfg4_shape(pkg, abi, scenes, ob, ctx, monkeypatch, film=(1920, 1080, 1024), n_tris=1000000,
                                 batch_tiles=None):
    """bench.py's cfg4: 1920x1080, 1024 spp, depth 5, four materials, 16 area lights, uniform light strategy, Sobol',
    box filter; cfg2's 1 M-triangle soup instead of 10 M."""
    w, h, spp = film
    arr = scenes.SceneArrays(n_tris, materials=MATS4, soup_version=1, n_lights=16)
    setup = scenes.RenderSetup(w, h, spp, max_depth=5)
    check_fullsize(pkg, abi, ob, ctx, monkeypatch, arr, setup, None, batch_tiles, 37, True)


def test_fullsize_spectral_cfg5_shape(pkg, abi, scenes, ob, ctx, monkeypatch, film=(1920, 1080, 64), n_tris=20000,
                                      batch_tiles=None):
    """bench.py's cfg5: 1920x1080, 64 spp, depth 16, four materials, the 100 k-triangle soup with its lights, a
    SampledSpectrum host (60 bins), instanced plastic objects with every third instance mirrored or stretched; 64
    instances of a 20 k-triangle object instead of 1000 of a 50 k one."""
    w, h, spp = film
    inst = []
    for k in range(64):  # 4 x 4 x 4 lattice through the soup's volume
        c = (-0.9 + 0.6 * (k % 4), -0.9 + 0.6 * ((k // 4) % 4), -0.9 + 0.6 * (k // 16))
        sc = (1.0, 1.0, 1.0) if k % 3 == 0 else ((1.2, 0.8, 1.0) if k % 3 == 1 else (1.0, 1.0, -1.1))
        inst.append(dict(object=0, center=c, scale=sc))
    arr = scenes.SceneArrays(100000, materials=MATS4, soup_version=1,
                             objects=(dict(n_tris=n_tris, seed=77, material="plastic", size=0.25),), instances=tuple(inst))
    arr.attach_spectral(json.load(open(os.path.join(GOLDEN, "spectral_tables.json"))))
    setup = scenes.RenderSetup(w, h, spp, max_depth=16)
    check_fullsize(pkg, abi, ob, ctx, monkeypatch, arr, setup, None, batch_tiles, 37, False)


def test_fullsize_volpath_cfg2fog_shape(pkg, abi, scenes, ob, ctx, monkeypatch, film=(1024, 1024, 256), n_tris=1000000,
                                        batch_tiles=None):
    """bench.py's cfg2fog: 1024x1024, 256 spp, depth 5, matte, VolPathIntegrator in its homogeneous medium, uniform
    light strategy, Sobol', box filter, the 1 M-triangle soup."""
    w, h, spp = film
    medium = dict(sigma_a=(0.05, 0.08, 0.12), sigma_s=(0.3, 0.25, 0.2), g=0.4)
    arr = scenes.SceneArrays(n_tris, materials=("matte",), soup_version=1)
    setup = scenes.RenderSetup(w, h, spp, max_depth=5, integrator="volpath", medium=medium)
    check_fullsize(pkg, abi, ob, ctx, monkeypatch, arr, setup, medium, batch_tiles, None, False)
