"""The drop-in boundary: pbrt_b200 = the reference's own CLI / parser / Film linked with
pbrt-v3-distributed_b200/host/gpupath.cpp (GpuPathIntegrator).  CPU: it must fail loudly
without a GPU (no CPU fallback).  GPU: an unmodified .pbrt file renders bit-identically to the
reference's PFM."""
import os
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, ROOT, bits

PLUGIN = os.path.join(ROOT, "oracle", "_ref", "plugin", "pbrt_b200")
needs_plugin = pytest.mark.skipif(not os.path.exists(PLUGIN), reason="pbrt_b200 is built where the reference sources exist")


def _scene(scenes, tmp_path, name="four", strategy="uniform", depth=5, materials=("matte", "glass", "metal", "plastic"),
           spp=8, sampler="sobol", **scene_kw):
    arr = scenes.SceneArrays(3000, materials=materials, soup_version=1, **scene_kw)
    return scenes.write_pbrt(str(tmp_path), "render_" + name, arr, 40, 32, spp, max_depth=depth, strategy=strategy,
                             sampler=sampler)


@needs_plugin
def test_plugin_fails_loudly_without_gpu(scenes, tmp_path):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    path = _scene(scenes, tmp_path)
    r = subprocess.run([PLUGIN, "--quiet", os.path.basename(path)], cwd=str(tmp_path), capture_output=True, text=True)
    assert "no usable CUDA device" in (r.stdout + r.stderr)
    assert not os.path.exists(os.path.join(str(tmp_path), "render_four.pfm")), "no image may be produced without a GPU"


def run_ranks(plugin, scenes, tmp_path, world, extra_env=None):
    """pbrt_b200 as `world` processes (B200PT_RANK / B200PT_WORLD_SIZE, tiles i mod world each): the ranks' raw film sums
    meet on rank 0, which alone writes the image; returns that image."""
    path = _scene(scenes, tmp_path)
    out = os.path.join(str(tmp_path), "render_four.pfm")
    procs = []
    for k in range(world):
        env = dict(os.environ, B200PT_RANK=str(k), B200PT_WORLD_SIZE=str(world), **(extra_env or {}))
        procs.append(subprocess.Popen([plugin, "--quiet", os.path.basename(path)], cwd=str(tmp_path), env=env,
                                      stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))
    logs = [p.communicate(timeout=600)[0] for p in procs]
    assert all(p.returncode == 0 for p in procs), "\n".join(logs)
    assert not [f for f in os.listdir(str(tmp_path)) if ".rank" in f], "the ranks' partial films must be consumed by rank 0"
    return scenes.read_pfm(out), logs


@needs_plugin
@pytest.mark.gpu
def test_dropin_two_ranks_one_image(scenes, tmp_path):
    """ADVICE r1 / SURVEY 8e: two pbrt_b200 processes shard the tiles of one film; rank 0 writes the one image, equal to
    the reference's.  (Both ranks share this box's GPU, so the merge goes through the file hand-over; with one GPU per
    rank and B200PT_NCCL_ID_FILE it is b200pt_film_reduce = one ncclReduce.)"""
    got, _ = run_ranks(PLUGIN, scenes, tmp_path, 2)
    ref = scenes.read_pfm(os.path.join(GOLDEN, "render_four.pfm"))
    assert np.array_equal(bits(got), bits(ref)), "the two ranks' merged image differs from the reference PFM"


@needs_plugin
@pytest.mark.gpu
def test_dropin_binary_matches_reference(scenes, tmp_path):
    path = _scene(scenes, tmp_path)
    r = subprocess.run([PLUGIN, "--quiet", os.path.basename(path)], cwd=str(tmp_path), capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    got = scenes.read_pfm(os.path.join(str(tmp_path), "render_four.pfm"))
    ref = scenes.read_pfm(os.path.join(GOLDEN, "render_four.pfm"))
    assert np.array_equal(bits(got), bits(ref)), "drop-in render differs from the reference PFM"
    # pbrt's default light sample strategy ("spatial") through the same binary
    path = _scene(scenes, tmp_path, "spatial", "spatial")
    r = subprocess.run([PLUGIN, "--quiet", os.path.basename(path)], cwd=str(tmp_path), capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    got = scenes.read_pfm(os.path.join(str(tmp_path), "render_spatial.pfm"))
    ref = scenes.read_pfm(os.path.join(GOLDEN, "render_spatial.pfm"))
    assert np.array_equal(bits(got), bits(ref)), "drop-in render (spatial light distribution) differs from the reference"
    # meshes with per-vertex shading normals / uvs and ReverseOrientation, read from PLY by the reference's own loader
    path = _scene(scenes, tmp_path, "normals_uv", "spatial", depth=6, shading_normals=(0, 2), uvs=(0, 3),
                  reverse_orientation=(3,))
    r = subprocess.run([PLUGIN, "--quiet", os.path.basename(path)], cwd=str(tmp_path), capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    got = scenes.read_pfm(os.path.join(str(tmp_path), "render_normals_uv.pfm"))
    ref = scenes.read_pfm(os.path.join(GOLDEN, "render_normals_uv.pfm"))
    assert np.array_equal(bits(got), bits(ref)), "drop-in render (shading normals / uvs) differs from the reference"
    # OrenNayar matte and rough glass parsed from the .pbrt file by the reference's own material factories
    path = _scene(scenes, tmp_path, "rough", "spatial", depth=8, materials=("matte_rough", "glass_rough", "metal", "plastic"))
    r = subprocess.run([PLUGIN, "--quiet", os.path.basename(path)], cwd=str(tmp_path), capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    got = scenes.read_pfm(os.path.join(str(tmp_path), "render_rough.pfm"))
    ref = scenes.read_pfm(os.path.join(GOLDEN, "render_rough.pfm"))
    assert np.array_equal(bits(got), bits(ref)), "drop-in render (OrenNayar / rough glass) differs from the reference"
    # pbrt's default sampler (Halton) with a non-power-of-two sample count
    path = _scene(scenes, tmp_path, "halton", "spatial", spp=6, sampler="halton")
    r = subprocess.run([PLUGIN, "--quiet", os.path.basename(path)], cwd=str(tmp_path), capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    got = scenes.read_pfm(os.path.join(str(tmp_path), "render_halton.pfm"))
    ref = scenes.read_pfm(os.path.join(GOLDEN, "render_halton.pfm"))
    assert np.array_equal(bits(got), bits(ref)), "drop-in render (Halton sampler) differs from the reference"
    # Sphere shapes (two of them area lights) written as `Translate` / `Scale` / `Shape "sphere"`
    from render_cases import EXTRA, RENDERS
    nt, mats, w, h, spp, depth, strat, nl = RENDERS["spheres"]
    arr = scenes.SceneArrays(nt, materials=mats, soup_version=1, n_lights=nl, **EXTRA["spheres"]["scene"])
    path = scenes.write_pbrt(str(tmp_path), "render_spheres", arr, w, h, spp, max_depth=depth, strategy=strat)
    r = subprocess.run([PLUGIN, "--quiet", os.path.basename(path)], cwd=str(tmp_path), capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    got = scenes.read_pfm(os.path.join(str(tmp_path), "render_spheres.pfm"))
    ref = scenes.read_pfm(os.path.join(GOLDEN, "render_spheres.pfm"))
    assert np.array_equal(bits(got), bits(ref)), "drop-in render (Sphere shapes) differs from the reference"
    # a Gaussian pixel filter (samples outside the film, 2-pixel tile aprons); golden from the 1-thread reference
    nt, mats, w, h, spp, depth, strat, nl = RENDERS["filter_gaussian"]
    arr = scenes.SceneArrays(nt, materials=mats, soup_version=1, n_lights=nl)
    path = scenes.write_pbrt(str(tmp_path), "render_filter_gaussian", arr, w, h, spp, max_depth=depth, strategy=strat,
                             pixel_filter="gaussian")
    r = subprocess.run([PLUGIN, "--quiet", os.path.basename(path)], cwd=str(tmp_path), capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    got = scenes.read_pfm(os.path.join(str(tmp_path), "render_filter_gaussian.pfm"))
    ref = scenes.read_pfm(os.path.join(GOLDEN, "render_filter_gaussian.pfm"))
    assert np.array_equal(bits(got), bits(ref)), "drop-in render (Gaussian pixel filter) differs from the reference"
    # object instancing: ObjectBegin / ObjectInstance blocks become TransformedPrimitives over per-object BVHAccels; the
    # rotated instances carry the matrices of pbrt's own Rotate
    for name in ("instances", "instances_affine"):
        nt, mats, w, h, spp, depth, strat, nl = RENDERS[name]
        arr = scenes.SceneArrays(nt, materials=mats, soup_version=1, n_lights=nl, **EXTRA[name]["scene"])
        path = scenes.write_pbrt(str(tmp_path), "render_" + name, arr, w, h, spp, max_depth=depth, strategy=strat)
        r = subprocess.run([PLUGIN, "--quiet", os.path.basename(path)], cwd=str(tmp_path), capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
        got = scenes.read_pfm(os.path.join(str(tmp_path), "render_%s.pfm" % name))
        ref = scenes.read_pfm(os.path.join(GOLDEN, "render_%s.pfm" % name))
        assert np.array_equal(bits(got), bits(ref)), "drop-in render (object instances, %s) differs from the reference" % name
    # delta lights and the mirror material, parsed by the reference's own factories
    for name in ("delta_lights", "mirror"):
        nt, mats, w, h, spp, depth, strat, nl = RENDERS[name]
        arr = scenes.SceneArrays(nt, materials=mats, soup_version=1, n_lights=nl, **EXTRA.get(name, {}).get("scene", {}))
        path = scenes.write_pbrt(str(tmp_path), "render_" + name, arr, w, h, spp, max_depth=depth, strategy=strat)
        r = subprocess.run([PLUGIN, "--quiet", os.path.basename(path)], cwd=str(tmp_path), capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
        got = scenes.read_pfm(os.path.join(str(tmp_path), "render_%s.pfm" % name))
        ref = scenes.read_pfm(os.path.join(GOLDEN, "render_%s.pfm" % name))
        assert np.array_equal(bits(got), bits(ref)), "drop-in render (%s) differs from the reference" % name


KILLEROO_DIR = os.path.join(ROOT, "oracle", "_ref", "scenes")


@needs_plugin
@pytest.mark.gpu
@pytest.mark.skipif(not os.path.exists(os.path.join(KILLEROO_DIR, "killeroo-cfg1-ref.pfm")),
                    reason="oracle/_ref/scenes is staged by `make -C oracle ref` where the reference sources exist")
@pytest.mark.parametrize("name,res", [("simple", 700), ("cfg1", 400)])
def test_killeroo_matches_reference(scenes, tmp_path, name, res):
    """BASELINE.json configs[0]: scenes/killeroo-simple.pbrt exactly as the reference ships it (700x700, 8 spp) and
    as BASELINE quotes it (400x400, 64 spp) -- Halton sampler, loop-subdivision meshes with shading normals,
    plastic, a Sphere area light -- through pbrt_b200 on the GPU vs the image the unmodified reference rendered
    from the same file."""
    import hashlib
    ref_path = os.path.join(KILLEROO_DIR, "killeroo-%s-ref.pfm" % name)
    want = open(os.path.join(GOLDEN, "killeroo_%s.sha256" % name)).read().split()[0]
    assert hashlib.sha256(open(ref_path, "rb").read()).hexdigest() == want, "staged reference image drifted"
    out = str(tmp_path / "killeroo-gpu.pfm")
    r = subprocess.run([PLUGIN, "--quiet", "--outfile", out, "killeroo-%s.pbrt" % name], cwd=KILLEROO_DIR,
                       capture_output=True, text=True)
    assert r.returncode == 0 and os.path.exists(out), r.stdout + r.stderr
    got, ref = scenes.read_pfm(out), scenes.read_pfm(ref_path)
    assert got.shape == ref.shape == (res, res, 3)
    diff = bits(got) != bits(ref)
    assert not diff.any(), "%d of %d components differ from the reference (max abs %.3g)" % (
        diff.sum(), diff.size, np.abs(got - ref).max())


# ---- SampledSpectrum host: pbrt_b200_spectral = the same drop-in linked with the reference built with
# `typedef SampledSpectrum Spectrum` (host/Makefile plugin_spectral, oracle/Makefile ref_spectral) ---------------------
PLUGIN_SPECTRAL = os.path.join(ROOT, "oracle", "_ref", "plugin", "pbrt_b200_spectral")
needs_spectral_plugin = pytest.mark.skipif(not os.path.exists(PLUGIN_SPECTRAL),
                                           reason="pbrt_b200_spectral is built where the reference sources exist")


def _read_spectral_trailer(path, abi):
    """The tables a SampledSpectrum host passes in b200pt_scene_desc, from a B200PT_DUMP_SCENE file (gpupath.cpp)."""
    import ctypes as C
    raw = open(path, "rb").read()
    hdr = np.frombuffer(raw, np.int64, 8)
    nt, nm, nl, nsph, has_n, has_uv = (int(x) for x in hdr[1:7])
    off = 64 + nt * (36 + 4 + 4 + 1 + 1) + (nt * 36 if has_n else 0) + (nt * 24 if has_uv else 0)
    mats = np.frombuffer(raw, np.uint8, nm * C.sizeof(abi.Material), off).reshape(nm, -1)
    off += nm * C.sizeof(abi.Material) + nl * C.sizeof(abi.AreaLight) + nsph * C.sizeof(abi.Sphere)
    off += C.sizeof(abi.CameraDesc) + 48 + C.sizeof(abi.IntegratorDesc) + 24  # film desc (48 B), six sampler ints
    ns = int(np.frombuffer(raw, np.int32, 1, off)[0])
    off += 4
    ms = np.frombuffer(raw, np.float32, nm * 5 * ns, off).reshape(nm, 5, ns)
    off += ms.nbytes
    ls = np.frombuffer(raw, np.float32, nl * ns, off).reshape(nl, ns)
    off += ls.nbytes
    cie = np.frombuffer(raw, np.float32, 3 * ns, off).reshape(3, ns)
    assert off + cie.nbytes == len(raw)
    return ns, mats, ms, ls, cie


@needs_spectral_plugin
def test_spectral_plugin_hands_over_the_hosts_spectra(abi, scenes, tmp_path):
    """CPU check of the host side: what gpupath.cpp (built against the SampledSpectrum reference) extracts from the
    parsed scene -- 60 bins per material spectrum and light, SampledSpectrum::X/Y/Z -- equals what the harness builds
    from the probe's fixtures (SceneArrays.attach_spectral), which the spectral oracle turns into the reference's image."""
    import json
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present: the GPU test renders through this binary")
    tables = json.load(open(os.path.join(GOLDEN, "spectral_tables.json")))
    arr = scenes.SceneArrays(3000, materials=("matte", "glass", "metal", "plastic"), soup_version=1).attach_spectral(tables)
    path = scenes.write_pbrt(str(tmp_path), "render_spectral_four", arr, 40, 32, 8, max_depth=5, strategy="uniform")
    dump = os.path.join(str(tmp_path), "scene.dump")
    r = subprocess.run([PLUGIN_SPECTRAL, "--quiet", os.path.basename(path)], cwd=str(tmp_path), capture_output=True,
                       text=True, env=dict(os.environ, B200PT_DUMP_SCENE=dump))
    assert "no usable CUDA device" in (r.stdout + r.stderr)
    ns, mats, ms, ls, cie = _read_spectral_trailer(dump, abi)
    assert ns == abi.SPECTRUM_SAMPLES
    assert np.array_equal(bits(cie), bits(arr.cie_xyz))
    assert len(ls) == arr.n_lights and all(np.array_equal(bits(row), bits(arr.light_spectra[0])) for row in ls)
    # the host numbers materials in the order it meets them (one per light quad, too): every one of its materials
    # must be one of the harness's, bin for bin, and every harness material must appear
    mine = [(int(m.type), arr.material_spectra[i]) for i, m in enumerate(arr._materials)]
    seen = set()
    for i in range(len(mats)):
        mtype = int(np.frombuffer(mats[i].tobytes(), np.int32, 1)[0])
        hit = [k for k, (t, rows) in enumerate(mine) if t == mtype and np.array_equal(bits(ms[i]), bits(rows))]
        assert hit, "host material %d (type %d) has spectra the fixtures do not hold" % (i, mtype)
        seen.update(hit)
    assert seen == set(range(len(mine)))
