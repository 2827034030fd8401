"""The benchmark's instance lattices through the two-level traversal kernel (collected last, like the other test_zz files;
tests/test_hostcheck.py replays the same functions at a small size against the CPU check build).

bench.py's cfg5 / cfg5rgb scene is 1000 overlapping instances of a 50 k-triangle object around a 100 k-triangle soup,
cfg5s 50 instances of a 1 M-triangle object.  k_trace2 walks them in one persistent launch with a resumable walk over
the tree of instances; the separate pass (B200PT_NO_TRACE2=1: k_trace for the top level, then k_spheres' InstanceWalk)
visits the instances in the same order, so its answers must be the same bit for bit.  The flag is read once per
process, so the separate pass runs in a child process on the same scene and rays.

Against the oracle, which walks the instances in index order: two hits in different instances whose distances lie
within the offset `dt` that Transform(Ray) adds to the origin (DESIGN.md section 2) may resolve either way.  Such a
disagreement is admitted only when both sides hit, one hit is an object triangle, and |t - t'| <= 2 max dt over the
instances whose world box the ray enters (restated in float64); any-hit answers must be equal."""
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from conftest import GOLDEN, ROOT, bits
from test_gpu_parity import ctx  # noqa: F401  (module-scoped context fixture)

MATS4 = ("matte", "glass", "metal", "plastic")
HERE = os.path.dirname(os.path.abspath(__file__))


def lattice(which, n_tris=None, size=None):
    """bench.workload_scene_kwargs restated: cfg5 = a 10 x 10 x 10 lattice of a 50 k-triangle plastic object (size 0.09,
    spacing 0.2), cfg5s = 5 x 5 x 2 of a 1 M-triangle one (size 0.25, spacing 0.4 / 0.8); every third instance plain,
    stretched (1.2, 0.8, 1) or mirrored (1, 1, -1.1).  n_tris / size replace the object's for smaller or non-overlapping
    variants."""
    kinds = [(1.0, 1.0, 1.0), (1.2, 0.8, 1.0), (1.0, 1.0, -1.1)]
    if which == "cfg5":
        inst = [dict(object=0, center=(-0.9 + 0.2 * (k % 10), -0.9 + 0.2 * ((k // 10) % 10), -0.9 + 0.2 * (k // 100)),
                     scale=kinds[k % 3]) for k in range(1000)]
        obj = dict(n_tris=50000, seed=77, material="plastic", size=0.09)
    else:
        inst = [dict(object=0, center=(-0.8 + 0.4 * (k % 5), -0.8 + 0.4 * ((k // 5) % 5), -0.4 + 0.8 * (k // 25)),
                     scale=kinds[k % 3]) for k in range(50)]
        obj = dict(n_tris=1000000, seed=77, material="plastic", size=0.25)
    if n_tris is not None:
        obj["n_tris"] = n_tris
    if size is not None:
        obj["size"] = size
    return dict(objects=(obj,), instances=tuple(inst))


def test_lattices_are_the_benchmarks():
    """The restatement above is bench.py's workload (no GPU needed)."""
    sys.path.insert(0, ROOT)
    import bench
    assert lattice("cfg5") == bench.workload_scene_kwargs("cfg5") == bench.workload_scene_kwargs("cfg5rgb")
    assert lattice("cfg5s") == bench.workload_scene_kwargs("cfg5s")


def make_scene(scenes, which, n_soup, n_tris, size=None):
    """The workload's scene: bench.py's 100 k-triangle soup (n_soup) with its five lights, four materials, the lattice."""
    return scenes.SceneArrays(n_soup, materials=MATS4, soup_version=1, **lattice(which, n_tris, size))


def ray_families(abi, arr, n, seed=5):
    """n rays in each of four families: from the bench camera (eye (0, 0, -4.5), fov 35, 16:9) over the film; from
    inside the lattice in random directions; the same with a finite tMax; inside rays with one or two zero direction
    components (-0.0 inside the mirrored instances)."""
    rng = np.random.default_rng(seed)
    rays = np.zeros(4 * n, dtype=abi.RAY_DTYPE)
    tan = np.tan(np.radians(35.0) / 2)
    cam = rays[:n]
    cam["o"] = (0.0, 0.0, -4.5)
    d = np.stack([rng.uniform(-16 / 9, 16 / 9, n) * tan, rng.uniform(-1, 1, n) * tan, np.ones(n)], 1)
    cam["d"] = (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)
    inside = rays[n:]
    inside["o"] = rng.uniform(-1.0, 1.0, (3 * n, 3)).astype(np.float32)
    inside["d"] = rng.normal(size=(3 * n, 3)).astype(np.float32)
    rays["t_max"] = np.inf
    rays["t_max"][2 * n:3 * n] = rng.uniform(0.02, 1.0, n).astype(np.float32)
    zero = rays[3 * n:]
    axis = np.arange(n) % 3
    zero["d"][np.arange(n), axis] = 0.0
    rows = np.arange(0, n, 4)
    zero["d"][rows, (axis[rows] + 1) % 3] = 0.0
    return rays


def oracle_parallel(o, fn, rays):
    """The oracle's trace entry points over chunks of rays on all cores (ctypes releases the GIL)."""
    chunks = np.array_split(np.arange(len(rays)), max(1, min(64, len(rays) // 2000)))
    with ThreadPoolExecutor(os.cpu_count()) as ex:
        parts = list(ex.map(lambda idx: getattr(o, fn)(rays[idx]), chunks))
    return np.concatenate(parts)


def trace_arm(scene, rays):
    h = scene.trace_closest(rays)
    return dict(triangle=h["triangle"], t=h["t"], b0=h["b0"], b1=h["b1"], occ=scene.trace_any(rays).astype(np.uint8))


def film_setup(scenes, abi):
    """128x72, 4 spp, depth 16, power light strategy: 40 tiles, several batches at B200PT_BATCH_PATHS = 7 tiles."""
    return scenes.RenderSetup(128, 72, 4, max_depth=16, strategy=abi.LIGHTS_POWER)


def render_arm(pkg, scene, setup):
    r = pkg.Render(scene, setup)
    try:
        r.render_tiles()
        return r.read_raw(), r.stats()
    finally:
        r.close()


def _load_with_lib(lib):
    """The package bound to another build of the library (the check build): what tests/conftest.py's hostcheck does."""
    import types
    sys.path.insert(0, ROOT)
    import __graft_entry__ as graft
    pkg = graft.load_package()
    if os.path.realpath(lib) == os.path.realpath(pkg.LIB_PATH):
        return pkg
    init = os.path.join(graft.PKG_DIR, "__init__.py")
    marker = 'LIB_PATH = os.path.join(_HERE, "libb200pt.so")'
    mod = types.ModuleType(graft.PKG_NAME + "_other")
    mod.__file__, mod.__package__ = init, graft.PKG_NAME
    exec(compile(open(init).read().replace(marker, "LIB_PATH = %r" % lib), init, "exec"), mod.__dict__)
    return mod


def child_main(spec_path):
    """The separate-pass arm: same scene, same rays, B200PT_NO_TRACE2=1 set by the parent; answers and film to an .npz file."""
    spec = json.load(open(spec_path))
    pkg = _load_with_lib(spec["lib"])
    from pbrt_v3_distributed_b200 import abi, scenes
    arr = make_scene(scenes, spec["which"], spec["n_soup"], spec["n_tris"])
    c = pkg.Context(0)
    scene = pkg.Scene(c, arr.desc(), keepalive=arr)
    out = trace_arm(scene, np.load(os.path.join(spec["dir"], "rays.npy")))
    film, st = render_arm(pkg, scene, film_setup(scenes, abi))
    np.savez(os.path.join(spec["dir"], "separate.npz"), film=film, stats=json.dumps(st), **out)
    scene.close()
    c.close()


def separate_pass(pkg, which, n_soup, n_tris, rays, tmp_path):
    """The child process of the separate-pass arm (it inherits B200PT_BATCH_PATHS)."""
    os.makedirs(str(tmp_path), exist_ok=True)
    np.save(os.path.join(str(tmp_path), "rays.npy"), rays)
    spec = os.path.join(str(tmp_path), "spec.json")
    json.dump(dict(which=which, n_soup=n_soup, n_tris=n_tris, dir=str(tmp_path), lib=pkg.LIB_PATH), open(spec, "w"))
    env = dict(os.environ, B200PT_NO_TRACE2="1")
    code = "import sys; sys.path[:0] = [%r, %r]; import test_zz_instances_gpu as T; T.child_main(%r)" % (HERE, ROOT, spec)
    r = subprocess.run([sys.executable, "-s", "-c", code], env=env, cwd=ROOT, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    z = np.load(os.path.join(str(tmp_path), "separate.npz"))
    return {k: z[k] for k in ("triangle", "t", "b0", "b1", "occ", "film")}, json.loads(str(z["stats"]))


def max_dt_of_entered_instances(arr, rays):
    """float64: for each ray, the largest Transform(Ray) origin offset dt (transform.h:251-264) over the instances whose
    world box (8 transformed corners of the object's bounds) the ray enters within [0, tMax]."""
    n = len(arr.instance_specs)
    w2i = np.array([np.array(arr._instances[k].world_to_instance, np.float64).reshape(4, 4) for k in range(n)])
    i2w = np.array([np.array(arr._instances[k].instance_to_world, np.float64).reshape(4, 4) for k in range(n)])
    first, count = arr.object_ranges[0]
    v = arr.vertices[first:first + count].reshape(-1, 3).astype(np.float64)
    lo, hi = v.min(0), v.max(0)
    corners = np.array([[(hi if c & (1 << a) else lo)[a] for a in range(3)] + [1.0] for c in range(8)])
    wc = np.einsum("kij,cj->kci", i2w, corners)[..., :3]
    blo, bhi = wc.min(1), wc.max(1)
    o = rays["o"].astype(np.float64)
    d = rays["d"].astype(np.float64)
    tmax = rays["t_max"].astype(np.float64)
    g3 = 3 * 2.0 ** -24 / (1 - 3 * 2.0 ** -24)
    with np.errstate(divide="ignore", invalid="ignore"):
        inv = 1 / d
        t0 = (blo[None] - o[:, None]) * inv[:, None]
        t1 = (bhi[None] - o[:, None]) * inv[:, None]
        tn = np.nan_to_num(np.minimum(t0, t1), nan=-np.inf).max(2)
        tf = np.nan_to_num(np.maximum(t0, t1), nan=np.inf).min(2)
    enters = (tn <= tf * (1 + 1e-6)) & (tf >= 0) & (tn <= tmax[:, None])
    terms = np.abs(w2i[None, :, :3, :3] * o[:, None, None, :]).sum(3) + np.abs(w2i[None, :, :3, 3])
    oe = g3 * terms
    dd = np.einsum("kij,rj->rki", w2i[:, :3, :3], d)
    dt = (np.abs(dd) * oe).sum(2) / np.maximum((dd * dd).sum(2), 1e-300)
    return np.where(enters, dt, 0).max(1)


def compare_with_oracle(what, arr, rays, got, want, occ_got, occ_want):
    assert np.array_equal(occ_got, occ_want), "%s: %d any-hit answers differ from the oracle" % (
        what, int((occ_got != occ_want).sum()))
    differ = (got["triangle"] != want["triangle"])
    hit = want["triangle"] >= 0
    for k in ("t", "b0", "b1"):
        differ |= hit & (bits(got[k]) != bits(want[k]))
    idx = np.nonzero(differ)[0]
    if len(idx):
        g, w = got["triangle"][idx], want["triangle"][idx]
        both = (g >= 0) & (w >= 0)
        obj = (g >= arr.n_toplevel) | (w >= arr.n_toplevel)
        dt = max_dt_of_entered_instances(arr, rays[idx])
        near = np.abs(got["t"][idx].astype(np.float64) - want["t"][idx].astype(np.float64)) <= 2 * dt
        bad = ~(both & obj & near)
        assert not bad.any(), "%s: %d rays disagree with the oracle beyond a near tie, first %d: device %s oracle %s" % (
            what, int(bad.sum()), int(idx[bad][0]), got[idx[bad][0]], want[idx[bad][0]])
    print("%s: %d rays, %d hits in instances, %d admissible near ties" % (
        what, len(rays), int((want["triangle"] >= arr.n_toplevel).sum()), len(idx)))
    assert len(idx) <= 1e-4 * len(rays)
    return len(idx)


def check_lattice(pkg, abi, scenes, ob, ctx, monkeypatch, tmp_path, which, n_soup=100000, n_tris=None, n_rays=250000):
    """(1) k_trace2 against the separate pass, bit for bit, rays and a 128x72 render of the lattice; (2) both against the
    oracle with the near-tie rule."""
    t_start = time.time()
    arr = make_scene(scenes, which, n_soup, n_tris)
    rays = ray_families(abi, arr, n_rays)
    monkeypatch.setenv("B200PT_BATCH_PATHS", str(7 * 256 * 4))
    scene = pkg.Scene(ctx, arr.desc(), keepalive=arr)
    try:
        two = trace_arm(scene, rays)
        film, st = render_arm(pkg, scene, film_setup(scenes, abi))
    finally:
        scene.close()
    sep, sst = separate_pass(pkg, which, n_soup, n_tris, rays, tmp_path)
    for k in ("triangle", "t", "b0", "b1", "occ"):
        same = bits(two[k]) == bits(sep[k]) if two[k].dtype == np.float32 else two[k] == sep[k]
        assert same.all(), "%s: %s of %d rays differs between k_trace2 and the separate pass, first ray %d" % (
            which, k, int((~same).sum()), int(np.nonzero(~same)[0][0]))
    assert np.array_equal(bits(film), bits(sep["film"])), "%s: the two traversal arms render different films" % which
    for k in ("camera_rays", "regular_rays", "shadow_rays", "stack_overflows"):
        assert st[k] == sst[k], (k, st[k], sst[k])
    assert st["stack_overflows"] == 0
    t0 = time.time()
    o = ob.Oracle(abi, arr)
    try:
        want = oracle_parallel(o, "trace_closest", rays)
        occ = oracle_parallel(o, "trace_any", rays)
    finally:
        o.close()
    print("%s: oracle %.1f s for %d rays" % (which, time.time() - t0, len(rays)))
    n = len(rays) // 4
    ties = {}
    for f, name in enumerate(("camera", "inside", "finite tMax", "zero components")):
        s = slice(f * n, (f + 1) * n)
        ties[name] = compare_with_oracle("%s %s" % (which, name), arr, rays[s],
                                         {k: two[k][s] for k in ("triangle", "t", "b0", "b1")}, want[s], two["occ"][s], occ[s])
    print("%s: near ties %s; %.1f s" % (which, ties, time.time() - t_start))


@pytest.mark.gpu
def test_cfg5_lattice_vs_separate_pass_and_oracle(pkg, abi, scenes, ob, ctx, monkeypatch, tmp_path):
    check_lattice(pkg, abi, scenes, ob, ctx, monkeypatch, tmp_path, "cfg5")


@pytest.mark.gpu
def test_cfg5s_lattice_vs_separate_pass_and_oracle(pkg, abi, scenes, ob, ctx, monkeypatch, tmp_path):
    check_lattice(pkg, abi, scenes, ob, ctx, monkeypatch, tmp_path, "cfg5s")


@pytest.mark.gpu
@pytest.mark.parametrize("spectral", [False, True])
def test_separated_lattice_renders_vs_oracle(pkg, abi, scenes, ob, ctx, monkeypatch, spectral, n_soup=100000, n_tris=50000,
                                             batch_tiles=7):
    """(3) The 1000-instance lattice with a smaller object (size 0.06: no two instance boxes overlap) and the top-level
    soup moved behind it (z in [1.5, 2.5]), so that no near tie can arise: 128x72, 4 spp, depth 16, power light
    strategy, several batches, RGB and 60 bins, raw film bit for bit against the oracle."""
    arr = make_scene(scenes, "cfg5", n_soup, n_tris, size=0.06)
    soup = slice(len(arr.light_quads) * 2, arr.n_toplevel)
    arr.vertices[soup, :, 2] = (arr.vertices[soup, :, 2] * np.float32(0.5) + np.float32(2.0)).astype(np.float32)
    tables = None
    if spectral:
        tables = json.load(open(os.path.join(GOLDEN, "spectral_tables.json")))
        arr.attach_spectral(tables)
    setup = film_setup(scenes, abi)
    spp = setup.sampler.samples_per_pixel
    monkeypatch.setenv("B200PT_BATCH_PATHS", str(batch_tiles * 256 * spp))
    o = ob.Oracle(abi, arr, spectral_tables=tables)
    scene = pkg.Scene(ctx, arr.desc(), keepalive=arr)
    r = pkg.Render(scene, setup)
    try:
        t0 = time.time()
        film, ost = o.render(setup)
        print("oracle %.1f s" % (time.time() - t0))
        r.render_tiles()
        raw = r.read_raw()
        st = r.stats()
        nbad = int((bits(raw) != bits(film)).sum())
        if nbad:
            ys, xs, _ = np.nonzero(bits(raw) != bits(film))
            print("first differing pixel", xs[0], ys[0], raw[ys[0], xs[0]], film[ys[0], xs[0]])
        assert nbad == 0, "%d of %d raw film values differ from the oracle" % (nbad, raw.size)
        assert -(-r.n_tiles // batch_tiles) > 1
        for k in ("camera_rays", "regular_rays", "shadow_rays"):
            assert st[k] == ost[k], (k, st[k], ost[k])
        assert st["stack_overflows"] == 0 and st["dimension_overflows"] == 0, st
    finally:
        r.close()
        scene.close()
        o.close()
