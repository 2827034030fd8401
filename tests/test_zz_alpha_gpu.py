"""Alpha masks (TriangleMesh::alphaMask / shadowAlphaMask, shapes/triangle.cpp:332-337, 531-570) inside the device's
traversal: float imagemap masks under the "uv" mapping (every wrap, EWA and trilinear settings, scale / delta, a
non-power-of-two map the host resamples), "float alpha" [0] and "float shadowalpha" [0], on meshes with and without
uvs, on an area light, on objects in rotated and mirrored instances next to spheres, under path (alpha, then
shadowalpha for shadow rays) and volpath (alpha only), in fog and with a cloud.  Every image of the drop-in binary is
compared bit for bit, and the ray counters exactly, with what the unmodified reference renders from the same .pbrt
file.  The masks are small PFMs generated from a seed."""
import os
import re
import sys

import numpy as np
import pytest

from conftest import ROOT, bits
import alpha_rays
import test_zz_infinite_gpu as I
import test_zz_textures_gpu as T

pytestmark = pytest.mark.gpu

REF, PLUGIN, PLUGIN_SPECTRAL, needs_binaries = I.REF, I.PLUGIN, I.PLUGIN_SPECTRAL, I.needs_binaries
REF_SPECTRAL = os.path.join(ROOT, "oracle", "_ref", "pbrt_ref_spectral")


def leaf(seed, w, h, zero=0.5):
    """A leaf-like mask: about `zero` of the texels exactly 0 (in blobs and scattered), the rest in (0, 1]."""
    rng = np.random.default_rng(seed)
    m = rng.uniform(0.05, 1.0, (h, w)).astype(np.float32)
    m[rng.uniform(size=(h, w)) < zero * 0.6] = 0
    m[h // 3:(2 * h) // 3, w // 4:w // 2] = 0
    return m


INSTANCES = dict(objects=(dict(n_tris=300, seed=5, material="plastic", size=0.45),),
                 instances=(dict(object=0, center=(0.0, 0.0, -2.2)),
                            dict(object=0, center=(1.0, 0.6, -1.8), rotate=(35, 0.3, 1, 0.2)),
                            dict(object=0, center=(-1.0, -0.6, -2.0), scale=(1.0, -1.2, 1.0), rotate=(-50, 1, 0, 0))))

# name: (scene arguments, film w, h, spp, maxdepth, strategy, write_pbrt extras)
CASES = {
    # leaf masks on a mesh with uvs (repeat, scaled and shifted) and on one without (clamp, the GetUVs defaults), EWA
    "leaf_uvs_spatial": (dict(n_tris=3000, materials=("matte", "plastic"), uvs=(0,), n_lights=2,
                              alphas={"matte": {"alpha": dict(map=leaf(1, 24, 10), uscale=3, vscale=2, udelta=0.25)},
                                      "plastic": {"alpha": dict(map=leaf(2, 16, 16), wrap="clamp")}}),
                         40, 32, 8, 5, "spatial", {}),
    # trilinear and anisotropy settings (a mask never reads them), black wrap, scale, power strategy
    "trilinear_black_power": (dict(n_tris=3000, materials=("matte", "metal", "glass"), uvs=(0, 1),
                                   alphas={"matte": {"alpha": dict(map=leaf(3, 32, 16), trilinear=True, wrap="black", uscale=1.6,
                                                                   vdelta=-0.3)},
                                           "metal": {"alpha": dict(map=leaf(4, 8, 8), maxanisotropy=2, scale=0.5, uscale=5)}}),
                              40, 32, 8, 6, "power", {}),
    # shadowalpha unlike alpha: path's shadow rays test both
    "shadowalpha_path": (dict(n_tris=3000, materials=("matte", "plastic"), uvs=(0, 1),
                              alphas={"matte": {"alpha": dict(map=leaf(5, 16, 16), uscale=2),
                                                "shadowalpha": dict(map=leaf(6, 16, 16, 0.8), wrap="clamp")},
                                      "plastic": {"shadowalpha": dict(map=leaf(7, 32, 32), uscale=3)}}),
                         40, 32, 8, 5, "uniform", {}),
    # the same under volpath, no medium: its shadow rays go through Tr (Intersect) and ignore shadowalpha
    "shadowalpha_volpath": (dict(n_tris=3000, materials=("matte", "plastic"), uvs=(0, 1),
                                 alphas={"matte": {"alpha": dict(map=leaf(5, 16, 16), uscale=2),
                                                   "shadowalpha": dict(map=leaf(6, 16, 16, 0.8), wrap="clamp")},
                                         "plastic": {"shadowalpha": dict(map=leaf(7, 32, 32), uscale=3)}}),
                            40, 32, 8, 5, "uniform", dict(integrator="volpath")),
    # ... and in fog
    "shadowalpha_volpath_fog": (dict(n_tris=3000, materials=("matte", "plastic"), uvs=(0, 1),
                                     alphas={"matte": {"alpha": dict(map=leaf(5, 16, 16), uscale=2),
                                                       "shadowalpha": dict(map=leaf(6, 16, 16, 0.8), wrap="clamp")},
                                             "plastic": {"shadowalpha": dict(map=leaf(7, 32, 32), uscale=3)}}),
                                40, 32, 8, 5, "uniform",
                                dict(integrator="volpath", medium=dict(sigma_a=(0.02, 0.03, 0.04), sigma_s=(0.05, 0.04, 0.03)))),
    # "float alpha" [0] (a ConstantTexture(0): the mesh is invisible) and "float shadowalpha" [0] (casts no shadow)
    "constant_zero": (dict(n_tris=3000, materials=("matte", "plastic", "metal"), alphas={"plastic": {"alpha": 0}, "metal": {"shadowalpha": 0}}),
                      40, 32, 8, 5, "uniform", {}),
    # a masked area light: sampled over its whole area (Shape::Sample ignores masks), seen through its holes
    "masked_light": (dict(n_tris=3000, materials=("matte", "plastic"), n_lights=2,
                          alphas={"light": {"alpha": dict(map=leaf(8, 8, 8), wrap="clamp")}, "matte": {"alpha": dict(map=leaf(9, 16, 16))}}),
                     40, 32, 8, 5, "spatial", {}),
    # masked objects in rotated and mirrored instances, next to spheres
    "instances_spheres": (dict(n_tris=2000, materials=("matte", "plastic"), n_lights=2,
                               spheres=[dict(center=(0.3, -0.2, 0.5), radius=0.45, material="matte"),
                                        dict(center=(-0.7, 0.4, 0.2), radius=0.35, material="plastic")],
                               alphas={"plastic": {"alpha": dict(map=leaf(10, 16, 16), uscale=2), "shadowalpha": dict(map=leaf(11, 8, 8))}},
                               **INSTANCES),
                          40, 32, 8, 5, "spatial", {}),
    # masked objects in instances without spheres: the two-level traversal kernel
    "instances_two_level": (dict(n_tris=2000, materials=("matte", "plastic"), n_lights=2,
                                 alphas={"plastic": {"alpha": dict(map=leaf(12, 16, 16), uscale=2), "shadowalpha": dict(map=leaf(13, 8, 8))},
                                         "matte": {"alpha": dict(map=leaf(14, 16, 16))}},
                                 **INSTANCES),
                            40, 32, 8, 5, "uniform", {}),
    # a cloud: the medium walk's segments meet masked triangles
    "volpath_cloud": (dict(n_tris=3000, materials=("matte", "plastic"), uvs=(0, 1),
                           spheres=[dict(center=(0.0, 0.0, -2.5), radius=0.8, boundary=dict(sigma_a=(0.3, 0.3, 0.3), sigma_s=(0.5, 0.5, 0.5)))],
                           alphas={"matte": {"alpha": dict(map=leaf(15, 16, 16), uscale=2)},
                                   "plastic": {"alpha": dict(map=leaf(16, 16, 16)), "shadowalpha": 0}}),
                      40, 32, 8, 5, "uniform", dict(integrator="volpath")),
    # image-textured materials seen through another mesh's cut-outs: camera differentials survive a rejected candidate
    "textures_behind_cutouts": (dict(n_tris=3000, materials=("matte", "plastic"), uvs=(0, 1),
                                     textures={"plastic": {"Kd": dict(map=T.rgb_map(51, 32, 16), uscale=3)}},
                                     alphas={"matte": {"alpha": dict(map=leaf(17, 16, 16, 0.7), uscale=2)}}),
                                40, 32, 8, 5, "spatial", {}),
}


def write_case(scenes, tmp_path, name, masks=True):
    kw, w, h, spp, depth, strat, extra = CASES[name]
    kw = dict(kw)
    if not masks:
        kw.pop("alphas")
    arr = scenes.SceneArrays(kw.pop("n_tris"), soup_version=1, **kw)
    return scenes.write_pbrt(str(tmp_path), name, arr, w, h, spp, max_depth=depth, strategy=strat, **extra)


def render(binary, path, out):
    r = I.run(binary, path, out)
    assert r.returncode == 0 and "Error" not in r.stderr, r.stdout + r.stderr
    return r


@needs_binaries
@pytest.mark.parametrize("name", sorted(CASES))
def test_dropin_alpha_vs_reference(scenes, tmp_path, name, plugin=PLUGIN):
    path = write_case(scenes, tmp_path, name)
    ref = render(REF, path, os.path.join(str(tmp_path), "ref.pfm"))
    got = render(plugin, path, os.path.join(str(tmp_path), "got.pfm"))
    img = scenes.read_pfm(os.path.join(str(tmp_path), "got.pfm"))
    I.assert_same(img, scenes.read_pfm(os.path.join(str(tmp_path), "ref.pfm")),
                  I.counters(got.stdout + got.stderr), I.counters(ref.stdout + ref.stderr), name)
    # the masks change the image: the case does exercise them
    bare = write_case(scenes, tmp_path / "bare", name, masks=False)
    render(plugin, bare, str(tmp_path / "bare" / "bare.pfm"))
    assert not np.array_equal(bits(img), bits(scenes.read_pfm(str(tmp_path / "bare" / "bare.pfm")))), name + ": the masks change nothing"


@pytest.mark.skipif(not (os.path.exists(REF_SPECTRAL) and os.path.exists(PLUGIN_SPECTRAL)),
                    reason="pbrt_ref_spectral / pbrt_b200_spectral are built where the reference sources exist")
def test_dropin_spectral_alpha_vs_reference(scenes, tmp_path):
    """The same traversal kernels under a SampledSpectrum host, against the 60-bin reference."""
    path = write_case(scenes, tmp_path, "shadowalpha_path")
    ref = render(REF_SPECTRAL, path, os.path.join(str(tmp_path), "ref.pfm"))
    got = render(PLUGIN_SPECTRAL, path, os.path.join(str(tmp_path), "got.pfm"))
    I.assert_same(scenes.read_pfm(os.path.join(str(tmp_path), "got.pfm")), scenes.read_pfm(os.path.join(str(tmp_path), "ref.pfm")),
                  I.counters(got.stdout + got.stderr), I.counters(ref.stdout + ref.stderr), "spectral")


@needs_binaries
def test_dropin_all_zero_mask_renders_as_without_the_mesh(scenes, tmp_path, plugin=PLUGIN):
    """Needs no reference: with uniform light sampling and area lights only, a mesh whose mask is 0 everywhere renders
    exactly the image, with the same ray counters, as the scene without that mesh."""
    arr = scenes.SceneArrays(3000, soup_version=1, materials=("matte", "plastic"), uvs=(1,), n_lights=2,
                             alphas={"plastic": {"alpha": dict(map=np.zeros((8, 8), np.float32))}})
    masked = scenes.write_pbrt(str(tmp_path), "masked", arr, 40, 32, 8, max_depth=5, strategy="uniform")
    text = open(masked).read()
    mesh = re.search(r'^Material "plastic".*\nShape "plymesh" "string filename" "masked_m1\.ply".*\n', text, re.M)
    assert mesh, text
    without = os.path.join(str(tmp_path), "without.pbrt")
    with open(without, "w") as f:
        f.write(text[:mesh.start()] + text[mesh.end():])
    a = render(plugin, masked, os.path.join(str(tmp_path), "a.pfm"))
    b = render(plugin, without, os.path.join(str(tmp_path), "b.pfm"))
    ia, ib = scenes.read_pfm(os.path.join(str(tmp_path), "a.pfm")), scenes.read_pfm(os.path.join(str(tmp_path), "b.pfm"))
    assert np.array_equal(bits(ia), bits(ib)) and ia.max() > 0
    assert I.counters(a.stdout + a.stderr) == I.counters(b.stdout + b.stderr)


def harness_render(pkg, abi, scenes, ctx, tmp_path, name, plugin):
    """The case through the Python harness: the host's dumped descriptors, its texture and alpha-mask tables."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from replay_dump import DumpScene
    path = write_case(scenes, tmp_path, name)
    dump = os.path.join(str(tmp_path), "scene.dump")
    r = I.run(plugin, path, os.path.join(str(tmp_path), "unused.pfm"), env=dict(B200PT_DUMP_SCENE=dump))
    assert r.returncode == 0, r.stdout + r.stderr
    masks, alpha, shadow = scenes.read_dump_alpha(dump, abi)
    assert masks and len(alpha) == len(shadow)
    ds = DumpScene(dump, abi, scenes)
    setup = ds.setup()
    scene = pkg.Scene(ctx, ds.desc(), keepalive=ds)
    mips, binds = scenes.read_dump_textures(dump, abi)
    ids = [scene.add_mipmap(m["levels"], m["wrap"], m["trilinear"], m["max_anisotropy"], m["weight_lut"]) for m in mips]
    for b in binds:
        scene.bind_texture(b["material"], b["slot"], ids[b["mipmap"]], b["su"], b["sv"], b["du"], b["dv"], b["remap"])
    mids = [scene.add_alpha_mask(m["texels"], m["wrap"], m["su"], m["sv"], m["du"], m["dv"]) for m in masks]
    assert mids == list(range(len(masks)))
    scene.set_alpha_masks(alpha, shadow)
    rend = pkg.Render(scene, setup)
    rend.render_tiles()
    rgb, st = rend.read_rgb(), rend.stats()
    rend.close()
    scene.close()
    return rgb, st, path


HARNESS_CASES = ["leaf_uvs_spatial", "shadowalpha_path", "textures_behind_cutouts"]


@needs_binaries
@pytest.mark.parametrize("name", HARNESS_CASES)
def test_harness_alpha_vs_reference(pkg, abi, scenes, tmp_path, name, plugin=PLUGIN):
    c = pkg.Context(0)
    try:
        rgb, st, path = harness_render(pkg, abi, scenes, c, tmp_path, name, plugin)
    finally:
        c.close()
    ref_run = I.run(REF, path, os.path.join(str(tmp_path), "ref.pfm"))
    ref = scenes.read_pfm(os.path.join(str(tmp_path), "ref.pfm"))
    cgot = {"Camera rays traced": st["camera_rays"], "Regular ray intersection tests": st["regular_rays"],
            "Shadow ray intersection tests": st["shadow_rays"] or None}
    I.assert_same(rgb, ref, cgot, I.counters(ref_run.stdout + ref_run.stderr), name)


@pytest.fixture(scope="module")
def ctx(pkg):
    c = pkg.Context(0)
    yield c
    c.close()


def _mask_scene(pkg, abi, scenes, ctx):
    """A soup whose plastic group carries a leaf mask (alpha) and a second one (shadowalpha), set through the C ABI."""
    arr = scenes.SceneArrays(4000, soup_version=1, materials=("matte", "plastic"), uvs=(1,))
    scene = pkg.Scene(ctx, arr.desc(), keepalive=arr)
    a = scene.add_alpha_mask(leaf(20, 32, 32), abi.WRAP_REPEAT, su=2.0, sv=3.0, du=0.1)
    s = scene.add_alpha_mask(leaf(21, 16, 16, 0.9), abi.WRAP_CLAMP)
    plastic = arr.material_id == 1
    scene.set_alpha_masks(np.where(plastic, a, -1), np.where(plastic, s, -1))
    return arr, scene


def test_trace_entry_points_apply_masks(pkg, abi, scenes, ctx):
    """b200pt_trace_closest / b200pt_trace_any answer Scene::Intersect / IntersectP with the masks: a masked scene
    occludes no ray the unmasked one does not, loses hits to the masks, and every closest hit it keeps on an unmasked
    triangle is one the plain traversal finds too when nothing masked lies in front."""
    arr = scenes.SceneArrays(4000, soup_version=1, materials=("matte", "plastic"), uvs=(1,))
    plain = pkg.Scene(ctx, arr.desc(), keepalive=arr)
    _, masked = _mask_scene(pkg, abi, scenes, ctx)
    rng = np.random.default_rng(3)
    rays = np.zeros(200000, dtype=abi.RAY_DTYPE)
    rays["o"] = rng.uniform(-2, 2, (len(rays), 3))
    rays["d"] = rng.normal(size=(len(rays), 3))
    rays["t_max"] = np.inf
    hp, hm = plain.trace_closest(rays), masked.trace_closest(rays)
    op, om = plain.trace_any(rays), masked.trace_any(rays)
    assert not (om & ~op).any()
    assert (op & ~om).sum() > 100, "no shadow ray passed through a mask"
    lost = (hp["triangle"] >= 0) & (hm["triangle"] != hp["triangle"])
    assert lost.sum() > 100, "no closest hit was rejected by a mask"
    plastic = arr.material_id == 1
    same = hp["triangle"] == hm["triangle"]
    # a hit the plain traversal finds on a matte triangle is kept exactly (nothing in front of it was closer)
    keep = (hp["triangle"] >= 0) & ~plastic[np.maximum(hp["triangle"], 0)]
    assert same[keep].all()
    assert np.array_equal(hp["t"][keep].view(np.uint32), hm["t"][keep].view(np.uint32))
    # the masked scene's hits lie no nearer than the plain ones
    both = (hp["triangle"] >= 0) & (hm["triangle"] >= 0)
    assert (hm["t"][both] >= hp["t"][both]).all()
    plain.close()
    masked.close()


def check_per_ray(pkg, abi, ctx, tmp_path):
    ref, hits, occ, bare = alpha_rays.compare(pkg, abi, ctx, str(tmp_path))
    assert len(ref) == len(hits) > 10 ** 6
    bad = np.flatnonzero(hits["triangle"] != ref["tri"])
    assert not len(bad), "closest-hit triangle differs from Triangle::Intersect at %d rays, first %s" % (len(bad), bad[:5])
    hit = ref["tri"] >= 0
    assert np.array_equal(hits["t"][hit].view(np.uint32), ref["t"][hit].view(np.uint32)), "closest-hit t differs"
    bad = np.flatnonzero(occ != ref["occ"])
    assert not len(bad), "occlusion differs from IntersectP at %d rays, first %s" % (len(bad), bad[:5])
    assert (bare["triangle"] != hits["triangle"]).sum() > 10 ** 5, "few closest hits were rejected by a mask"
    assert (occ == 0).sum() > 10 ** 4, "few shadow rays passed through the masks"


@pytest.mark.skipif(not os.path.exists(alpha_rays.PROBE), reason="alpha_probe is built where the reference sources exist")
def test_trace_entry_points_vs_reference_per_ray(pkg, abi, ctx, tmp_path):
    """b200pt_trace_closest / b200pt_trace_any against the reference's Triangle::Intersect / IntersectP with the same
    masks, ray by ray, bit for bit (alpha_rays.py)."""
    check_per_ray(pkg, abi, ctx, tmp_path)
