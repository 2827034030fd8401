"""Synthetic workloads of BASELINE.json (`configs`) as plain arrays + descriptors.

The triangle soup is SURVEY.md Appendix A.3 verbatim (numpy default_rng(1234),
centres U[-1,1]^3, offsets U[-s,s]^3, unshared vertices).  `version` 0 is the
soup the CPU probes in BASELINE.md were timed on (s = N^-1/3, one emissive quad
at y=+3); version 1 (s = 0.5 N^-1/3, five inward-facing emissive quads) is the
better-lit variant SURVEY.md section 6 asks for before taking parity numbers.
Everything here is host-side description; nothing touches the device.

The same description can be written out as `.pbrt` + binary PLY
(`write_pbrt`) so the unmodified reference renders the identical scene.
"""
import ctypes as C
import os
import re
import struct

import numpy as np

from . import abi

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")

# default copper spectrum of MetalMaterial converted to RGB by the reference
# (materials/metal.cpp:82-118; values dumped by oracle/probe `consts`).
COPPER_ETA = [float.fromhex("0x1.9994b8p-3"), float.fromhex("0x1.d81b7ap-1"), float.fromhex("0x1.199178p+0")]
COPPER_K = [float.fromhex("0x1.f3cb18p+1"), float.fromhex("0x1.394c0cp+1"), float.fromhex("0x1.119e9ap+1")]


def soup_vertices(n, seed=1234, version=0):
    if n == 0:
        return np.zeros((0, 3, 3), np.float32)
    rng = np.random.default_rng(seed)
    c = rng.uniform(-1, 1, (n, 1, 3)).astype(np.float32)
    k = 1.0 if version == 0 else 0.5
    s = np.float32(k * n ** (-1 / 3))
    v = (c + rng.uniform(-s, s, (n, 3, 3)).astype(np.float32)).astype(np.float32)
    return np.ascontiguousarray(v)


def quad(p0, p1, p2, p3):
    """Two triangles (0 1 2) (0 2 3) as in the `trianglemesh` of Appendix A.4."""
    q = np.array([p0, p1, p2, p3], dtype=np.float32)
    return np.stack([q[[0, 1, 2]], q[[0, 2, 3]]])


def light_quads(version, n_lights=None):
    """Emissive quads, each wound so that Cross(p0-p2, p1-p2) faces the soup."""
    top = quad([-1.5, 3, -1.5], [1.5, 3, -1.5], [1.5, 3, 1.5], [-1.5, 3, 1.5])
    if n_lights is not None:  # Cfg 4: n_lights/2 1x1 quads on a grid at y=+3
        quads = []
        nq = n_lights // 2
        cols = 4
        for i in range(nq):
            cx = -2.25 + 1.5 * (i % cols)
            cz = -0.75 + 1.5 * (i // cols)
            quads.append(quad([cx - .5, 3, cz - .5], [cx + .5, 3, cz - .5], [cx + .5, 3, cz + .5],
                              [cx - .5, 3, cz + .5]))
        return quads
    if version == 0:
        return [top]
    bottom = quad([-1.5, -3, -1.5], [-1.5, -3, 1.5], [1.5, -3, 1.5], [1.5, -3, -1.5])
    left = quad([-3, -1.5, -1.5], [-3, 1.5, -1.5], [-3, 1.5, 1.5], [-3, -1.5, 1.5])
    right = quad([3, -1.5, -1.5], [3, -1.5, 1.5], [3, 1.5, 1.5], [3, 1.5, -1.5])
    back = quad([-1.5, -1.5, 3], [-1.5, 1.5, 3], [1.5, 1.5, 3], [1.5, -1.5, 3])
    return [top, bottom, left, right, back]


def default_materials(which):
    """Material table: matte Kd .5 / glass / metal(copper, roughness .01) /
    plastic(Kd=Ks=.25, roughness .1) with the factories' defaults
    (glass.cpp:94-110, metal.cpp:115-134, plastic.cpp:72-83)."""
    from . import host_oren_nayar, host_roughness_to_alpha  # C-ABI host helpers (same libm as the reference)
    mats = []
    for w in which:
        m = abi.Material()
        if w == "matte":
            m.type = abi.MAT_MATTE
            m.kd[:] = [0.5, 0.5, 0.5]
        elif w == "matte_rough":  # sigma = 30 degrees -> OrenNayar
            m.type = abi.MAT_MATTE
            m.kd[:] = [0.5, 0.5, 0.5]
            m.alpha_x, m.alpha_y = host_oren_nayar(30.0)
            m.variant = 1
        elif w == "glass_rough":  # uroughness .2, vroughness .1, remapped -> microfacet reflection + transmission
            m.type = abi.MAT_GLASS
            m.ks[:] = [1, 1, 1]
            m.kt[:] = [1, 1, 1]
            m.index = 1.5
            m.alpha_x = host_roughness_to_alpha(0.2)
            m.alpha_y = host_roughness_to_alpha(0.1)
            m.variant = 1
        elif w == "black":
            m.type = abi.MAT_MATTE
            m.kd[:] = [0, 0, 0]
        elif w == "mirror":  # MirrorMaterial, Kr 0.9 (mirror.cpp:58-64): the specular family's variant 2
            m.type = abi.MAT_GLASS
            m.ks[:] = [0.9, 0.9, 0.9]
            m.index = 1.0
            m.variant = 2
        elif w == "glass":
            m.type = abi.MAT_GLASS
            m.ks[:] = [1, 1, 1]
            m.kt[:] = [1, 1, 1]
            m.index = 1.5
        elif w == "metal":
            m.type = abi.MAT_METAL
            m.eta[:] = COPPER_ETA
            m.k[:] = COPPER_K
            a = host_roughness_to_alpha(0.01)
            m.alpha_x = a
            m.alpha_y = a
        elif w == "plastic":
            m.type = abi.MAT_PLASTIC
            m.kd[:] = [0.25, 0.25, 0.25]
            m.ks[:] = [0.25, 0.25, 0.25]
            a = host_roughness_to_alpha(0.1)
            m.alpha_x = a
            m.alpha_y = a
        else:
            raise ValueError(w)
        mats.append(m)
    return mats


PBRT_MATERIAL = {
    "matte": 'Material "matte" "rgb Kd" [0.5 0.5 0.5]',
    "black": 'Material "matte" "rgb Kd" [0 0 0]',
    "glass": 'Material "glass"',
    "mirror": 'Material "mirror"',
    "matte_rough": 'Material "matte" "rgb Kd" [0.5 0.5 0.5] "float sigma" [30]',
    "glass_rough": 'Material "glass" "float uroughness" [0.2] "float vroughness" [0.1]',
    "metal": 'Material "metal"',
    "plastic": 'Material "plastic"',
}


class SceneArrays:
    """Flattened scene in the layout b200pt_scene_desc wants."""

    def __init__(self, n_tris, materials=("matte",), soup_version=1, seed=1234, light_L=40.0,
                 n_lights=None, two_sided=False, reverse_orientation=(), shading_normals=(), uvs=(), spheres=(),
                 objects=(), instances=(), delta_lights=(), infinite_lights=(), textures=None, alphas=None):
        """spheres: dicts {center, radius, material (a name in `materials` or "black"), emit (radiance or
        None), scale (sx, sy, sz) or None, reverse_orientation} -- written as `Translate` + `Scale` +
        `Shape "sphere"` by write_pbrt, after the meshes."""
        self.material_names = list(materials) + ["black"]
        soup = soup_vertices(n_tris, seed, soup_version)
        quads = light_quads(soup_version, n_lights)
        light_tris = np.concatenate(quads) if quads else np.zeros((0, 3, 3), np.float32)
        nl = len(light_tris)
        # primitive order == .pbrt order (write_pbrt): lights first, then one
        # plymesh per material holding triangles m::len(materials)
        nm = len(materials)
        parts, mids = [light_tris], [np.full(nl, nm, np.int32)]
        self.ply_parts = []
        for m in range(nm):
            part = np.ascontiguousarray(soup[m::nm])
            parts.append(part)
            mids.append(np.full(len(part), m, np.int32))
            self.ply_parts.append(part)
        self.vertices = np.ascontiguousarray(np.concatenate(parts).astype(np.float32))
        self.material_id = np.ascontiguousarray(np.concatenate(mids))
        self.light_id = np.full(len(self.vertices), -1, np.int32)
        self.light_id[:nl] = np.arange(nl, dtype=np.int32)
        self.flip = np.zeros(len(self.vertices), np.uint8)
        # "ReverseOrientation" on the plymesh of material m (identity CTM: no handedness swap)
        self.reverse_orientation = tuple(reverse_orientation)
        for m in self.reverse_orientation:
            self.flip[self.material_id == m] = 1
        # optional per-vertex shading normals / uvs on the plymesh of material m (deterministic, seed + 7):
        # un-normalised perturbed face normals and random uvs, to exercise triangle.cpp:293-413
        self.shading_normals, self.uv_meshes = tuple(shading_normals), tuple(uvs)
        self.normals = self.uvs = self.vertex_flags = None
        if self.shading_normals or self.uv_meshes:
            r2 = np.random.default_rng(seed + 7)
            v = self.vertices
            fn = np.cross(v[:, 1] - v[:, 0], v[:, 2] - v[:, 0])
            fn /= np.maximum(np.linalg.norm(fn, axis=1, keepdims=True), 1e-20)
            self.normals = np.ascontiguousarray((fn[:, None, :] + r2.uniform(-0.4, 0.4, v.shape)).astype(np.float32))
            self.uvs = np.ascontiguousarray(r2.uniform(0, 1, (len(v), 3, 2)).astype(np.float32))
            self.vertex_flags = np.zeros(len(v), np.uint8)
            for m in self.shading_normals:
                self.vertex_flags[self.material_id == m] |= 1
            for m in self.uv_meshes:
                self.vertex_flags[self.material_id == m] |= 2
        self.light_quads = quads
        self.light_L = float(light_L)
        self.two_sided = bool(two_sided)
        self._materials = None
        # object instancing: objects = dicts {n_tris, seed, material, size}; each is a small soup in its own space
        # (written as ObjectBegin/ObjectEnd at the identity CTM); instances = dicts {object, center, scale, rotate,
        # order} (instance_steps)
        self.n_toplevel = len(self.vertices)
        self.object_specs = [dict(o) for o in objects]
        self.instance_specs = [dict(i) for i in instances]
        self.object_ranges, self.object_parts = [], []
        for o in self.object_specs:
            part = np.ascontiguousarray(soup_vertices(o["n_tris"], o.get("seed", 5), 1) * np.float32(o.get("size", 0.3)))
            self.object_ranges.append((len(self.vertices), len(part)))
            self.object_parts.append(part)
            mid = self.material_names.index(o.get("material", "matte"))
            self.vertices = np.ascontiguousarray(np.concatenate([self.vertices, part]))
            self.material_id = np.ascontiguousarray(np.concatenate([self.material_id, np.full(len(part), mid, np.int32)]))
            self.light_id = np.ascontiguousarray(np.concatenate([self.light_id, np.full(len(part), -1, np.int32)]))
            self.flip = np.ascontiguousarray(np.concatenate([self.flip, np.zeros(len(part), np.uint8)]))
        assert not (self.object_specs and (self.shading_normals or self.uv_meshes)), "objects + per-vertex data: not wired"
        self._instances = (abi.Instance * max(len(self.instance_specs), 1))()
        for k, ins in enumerate(self.instance_specs):
            first, count = self.object_ranges[ins["object"]]
            rec = self._instances[k]
            rec.first_triangle, rec.n_triangles = first, count
            m, minv = ctm(instance_steps(ins))
            rec.instance_to_world[:] = m.reshape(-1).tolist()
            rec.world_to_instance[:] = minv.reshape(-1).tolist()
            rec.is_identity = int(np.array_equal(m, np.eye(4)))  # Transform::IsIdentity (transform.h:148-155)
        self.sphere_specs = [dict(s) for s in spheres]
        n_sl = sum(1 for s in self.sphere_specs if s.get("emit"))
        # delta lights: dicts {kind: "point"|"spot"|"distant", from_, to, I or L, coneangle, conedelta}; they follow
        # the emissive quads in the .pbrt file, hence in Scene::lights
        self.delta_specs = [dict(x) for x in delta_lights]
        # infinite lights: dicts {L (rgb or scalar), scale (rgb or scalar), map (array [h][w][3], written as <name>_sky<k>.pfm
        # and named by "string mapname") or None, steps: [(op, args)] of the light's transform}; they follow the delta lights
        self.infinite_specs = [dict(x) for x in infinite_lights]
        # image textures: {material name: {pbrt parameter ("Kd", "roughness", ...): texture spec, "params": extra material
        # parameters}} with texture spec {map: [h][w][3] texels (written as a PFM), wrap, trilinear, maxanisotropy, scale,
        # gamma, uscale, vscale, udelta, vdelta}; write_pbrt declares them as imagemap textures under the "uv" mapping.  The
        # descriptors here keep the materials' constants: the texture tables come from the host (read_dump_textures)
        self.texture_specs = {k: dict(v) for k, v in (textures or {}).items()}
        # alpha masks: {material name (its meshes and objects) or "light" (the area-light quads): {"alpha" / "shadowalpha":
        # 0 (written as "float alpha" [0]) or a mask spec {map: [h][w] texels (written as a PFM), wrap, trilinear,
        # maxanisotropy, scale, uscale, vscale, udelta, vdelta}}}; write_pbrt declares the maps as float imagemap textures
        # under the "uv" mapping.  The descriptors here carry no masks: their tables come from the host.
        self.alpha_specs = {k: dict(v) for k, v in (alphas or {}).items()}
        self._lights = (abi.AreaLight * max(nl + len(self.delta_specs) + len(self.infinite_specs) + n_sl, 1))()
        for i in range(nl):
            self._lights[i].triangle = i
            self._lights[i].lemit[:] = [light_L] * 3
            self._lights[i].two_sided = int(two_sided)
            self._lights[i].sphere = -1
        for dl in self.delta_specs:
            from . import host_spot_light
            rec = self._lights[nl]
            nl += 1
            rec.triangle, rec.sphere = -1, -1
            val = dl.get("I", dl.get("L", 1.0))
            rec.lemit[:] = [val] * 3 if np.isscalar(val) else list(val)
            f_, t_ = dl.get("from_", (0, 0, 0)), dl.get("to", (0, 0, 1))
            if dl["kind"] == "point":  # CreatePointLight, point.cpp:82-92
                rec.kind = abi.LIGHT_POINT
                rec.position[:] = [np.float32(v) for v in f_]
            elif dl["kind"] == "spot":
                host_spot_light(rec, f_, t_, dl.get("coneangle", 30.0), dl.get("conedelta", 5.0))
            else:  # CreateDistantLight, distant.cpp:87-96: wLight = Normalize(from - to)
                rec.kind = abi.LIGHT_DISTANT
                f32 = np.float32
                dvec = [f32(f32(a) - f32(b)) for a, b in zip(f_, t_)]
                ln = np.sqrt(f32(f32(f32(dvec[0] * dvec[0]) + f32(dvec[1] * dvec[1])) + f32(dvec[2] * dvec[2])))
                inv = f32(1) / f32(ln)  # Vector3::operator/ multiplies by the reciprocal (geometry.h:132-137)
                rec.position[:] = [f32(v * inv) for v in dvec]
        for il in self.infinite_specs:  # CreateInfiniteLight (infinite.cpp:180-191): WorldToLight = Inverse(CTM)
            rec = self._lights[nl]
            nl += 1
            rec.triangle, rec.sphere, rec.kind = -1, -1, abi.LIGHT_INFINITE
            _, minv = ctm(il.get("steps", ()))
            rec.world_to_light[:] = minv.reshape(-1).tolist()
        self._spheres = (abi.Sphere * max(len(self.sphere_specs), 1))()
        for k, sp in enumerate(self.sphere_specs):
            m, minv = sphere_transform(sp["center"], sp.get("scale"))
            rec = self._spheres[k]
            rec.object_to_world[:] = m.reshape(-1).tolist()
            rec.world_to_object[:] = minv.reshape(-1).tolist()
            rec.radius = sp["radius"]
            rec.material_id = self.material_names.index(sp.get("material", "black"))
            rec.reverse_orientation = int(bool(sp.get("reverse_orientation")))
            sc = sp.get("scale") or (1, 1, 1)
            rec.transform_swaps_handedness = int(sc[0] * sc[1] * sc[2] < 0)  # Transform::SwapsHandedness
            if any(k in sp for k in ("zmin", "zmax", "phimax")):  # partial sphere: the Sphere ctor's members
                from . import host_sphere_params
                r_ = sp["radius"]
                zp = host_sphere_params(r_, sp.get("zmin", -r_), sp.get("zmax", r_), sp.get("phimax", 360.0))
                rec.z_min, rec.z_max, rec.theta_min, rec.theta_max, rec.phi_max = zp
            rec.light_id = -1
            if sp.get("emit"):
                li = nl
                nl += 1
                rec.light_id = li
                self._lights[li].triangle = -1
                self._lights[li].sphere = k
                self._lights[li].lemit[:] = [sp["emit"]] * 3
                self._lights[li].two_sided = int(bool(sp.get("two_sided")))
        self.n_lights = nl

    @property
    def n_triangles(self):
        return len(self.vertices)

    def attach_spectral(self, tables):
        """Describe the scene the way a SampledSpectrum build of the host would (b200pt_scene_desc::n_spectrum_samples
        = 60).  `tables` is tests/golden/spectral_tables.json: the 60-bin spectra that build holds for the RGB triples /
        constant spectra of this harness (dumped from the reference by oracle/probe, never computed here) and its
        SampledSpectrum::X / Y / Z."""
        f32 = np.float32
        lut = {tuple(np.array([float.fromhex(x) for x in rgb], f32).view(np.uint32).tolist()):
               np.array([float.fromhex(x) for x in spec], f32) for rgb, spec in tables["spectra"]}

        def look(rgb, what):
            key = tuple(np.array(list(rgb), f32).view(np.uint32).tolist())
            if key not in lut:
                raise KeyError("no SampledSpectrum fixture for %s = %s" % (what, list(rgb)))
            return lut[key]
        if self._materials is None:
            mats = default_materials(self.material_names)
            self._materials = (abi.Material * len(mats))(*mats)
        used = {abi.MAT_MATTE: ("kd",), abi.MAT_PLASTIC: ("kd", "ks"), abi.MAT_METAL: ("eta", "k"), abi.MAT_GLASS: ("ks", "kt")}
        order = ("kd", "ks", "kt", "eta", "k")
        ms = np.zeros((len(self._materials), len(order), abi.SPECTRUM_SAMPLES), f32)
        for i, m in enumerate(self._materials):
            for name in used[m.type]:
                if m.type == abi.MAT_GLASS and m.variant == 2 and name == "kt":
                    continue  # MirrorMaterial has no Kt
                ms[i, order.index(name)] = look(getattr(m, name), "material %d %s" % (i, name))
        n = max(self.n_lights, 1)
        ls = np.zeros((n, abi.SPECTRUM_SAMPLES), f32)
        for i in range(self.n_lights):
            ls[i] = look(self._lights[i].lemit, "light %d" % i)
        self.material_spectra, self.light_spectra = ms, ls
        self.cie_xyz = np.array([[float.fromhex(x) for x in tables[k]] for k in ("cie_x", "cie_y", "cie_z")], f32)
        return self

    def desc(self):
        if self._materials is None:
            mats = default_materials(self.material_names)
            self._materials = (abi.Material * len(mats))(*mats)
        d = abi.SceneDesc()
        if getattr(self, "cie_xyz", None) is not None:
            d.n_spectrum_samples = abi.SPECTRUM_SAMPLES
            d.material_spectra = abi.ptr(self.material_spectra)
            d.light_spectra = abi.ptr(self.light_spectra)
            d.cie_xyz = abi.ptr(self.cie_xyz)
        d.n_triangles = self.n_triangles
        d.vertices = abi.ptr(self.vertices)
        d.material_id = abi.ptr(self.material_id)
        d.light_id = abi.ptr(self.light_id)
        d.flip_normal = abi.ptr(self.flip)
        d.n_materials = len(self._materials)
        d.materials = C.cast(self._materials, C.POINTER(abi.Material))
        d.n_lights = self.n_lights
        d.lights = C.cast(self._lights, C.POINTER(abi.AreaLight))
        d.normals = abi.ptr(self.normals)
        d.uvs = abi.ptr(self.uvs)
        d.vertex_flags = abi.ptr(self.vertex_flags)
        d.n_spheres = len(self.sphere_specs)
        d.spheres = C.cast(self._spheres, C.POINTER(abi.Sphere))
        d.n_instances = len(getattr(self, "instance_specs", ()))
        if d.n_instances:
            d.instances = C.cast(self._instances, C.POINTER(abi.Instance))
            d.n_toplevel_triangles = self.n_toplevel
        return d


def _mat_mul(a, b):
    """Matrix4x4::Mul (transform.cpp:98-106): float sums in index order."""
    f = np.float32
    r = np.zeros((4, 4), f)
    for i in range(4):
        for j in range(4):
            r[i, j] = f(f(f(a[i, 0] * b[0, j]) + f(a[i, 1] * b[1, j])) + f(a[i, 2] * b[2, j])) + f(a[i, 3] * b[3, j])
    return r


def _libm_float(name):
    """sinf / cosf of the host libm: what std::sin / std::cos of a float call in the reference."""
    import ctypes.util
    fn = getattr(C.CDLL(ctypes.util.find_library("m")), name)
    fn.restype, fn.argtypes = C.c_float, [C.c_float]
    return lambda x: np.float32(fn(float(x)))


def step_transform(op, args):
    """(m, mInv) of one CTM statement: Translate / Scale / Rotate (transform.cpp:141-153, :178-201).  Rotate restates
    Normalize (geometry.h:984-986), Radians (pbrt.h:320) and the float sin / cos of the host libm; its inverse is the
    transpose."""
    f = np.float32
    m = np.eye(4, dtype=f)
    minv = np.eye(4, dtype=f)
    if op == "Translate":
        m[:3, 3] = [f(c) for c in args]
        minv[:3, 3] = [-f(c) for c in args]
    elif op == "Scale":
        for a in range(3):
            m[a, a] = f(args[a])
            minv[a, a] = f(1) / f(args[a])
    elif op == "Rotate":
        v = [f(c) for c in args[1:]]
        inv = f(1) / np.sqrt(f(f(f(v[0] * v[0]) + f(v[1] * v[1])) + f(v[2] * v[2])))
        x, y, z = (f(c * inv) for c in v)
        theta = f(f(f(3.14159265358979323846) / f(180)) * f(args[0]))
        s, c = _libm_float("sinf")(theta), _libm_float("cosf")(theta)
        omc = f(1 - c)
        m[:3, :3] = [[f(f(x * x) + f(f(1 - f(x * x)) * c)), f(f(f(x * y) * omc) - f(z * s)), f(f(f(x * z) * omc) + f(y * s))],
                     [f(f(f(x * y) * omc) + f(z * s)), f(f(y * y) + f(f(1 - f(y * y)) * c)), f(f(f(y * z) * omc) - f(x * s))],
                     [f(f(f(x * z) * omc) - f(y * s)), f(f(f(y * z) * omc) + f(x * s)), f(f(z * z) + f(f(1 - f(z * z)) * c))]]
        minv = np.ascontiguousarray(m.T)
    else:
        raise ValueError(op)
    return m, minv


def ctm(steps):
    """CTM pbrt builds from CTM statements inside an attribute block at identity (api.cpp pbrtTranslate / pbrtScale /
    pbrtRotate: ctm = ctm * T; Transform::operator*, transform.cpp:222-225: the inverse multiplies in reverse order)."""
    m = np.eye(4, dtype=np.float32)
    minv = np.eye(4, dtype=np.float32)
    for op, args in steps:
        t, ti = step_transform(op, args)
        m, minv = _mat_mul(m, t), _mat_mul(ti, minv)
    return m, minv


def sphere_transform(center, scale=None):
    """CTM of `Translate c` [+ `Scale s`]."""
    return ctm([("Translate", center)] + ([("Scale", scale)] if scale else []))


def instance_steps(ins):
    """The CTM statements of an instance spec, in the spec's `order` (default "TSR"): Translate `center`, Scale `scale`,
    Rotate `rotate` = (degrees, ax, ay, az).  "TSR" gives the linear part S R (not orthogonal under a non-uniform
    scale), "TRS" R S.  An instance with neither scale nor rotation nor offset has no statement (the identity)."""
    c, sc, rot = tuple(ins.get("center", (0, 0, 0))), ins.get("scale"), ins.get("rotate")
    have = {"T": ("Translate", c) if c != (0, 0, 0) or sc or rot else None,
            "S": ("Scale", tuple(sc)) if sc else None, "R": ("Rotate", tuple(rot)) if rot else None}
    return [have[k] for k in ins.get("order", "TSR") if have[k]]


def write_ply(path, tris, normals=None, uvs=None):
    n = len(tris)
    cols = [np.asarray(tris, np.float32).reshape(3 * n, 3)]
    props = "property float x\nproperty float y\nproperty float z\n"
    if normals is not None:
        cols.append(np.asarray(normals, np.float32).reshape(3 * n, 3))
        props += "property float nx\nproperty float ny\nproperty float nz\n"
    if uvs is not None:
        cols.append(np.asarray(uvs, np.float32).reshape(3 * n, 2))
        props += "property float u\nproperty float v\n"
    with open(path, "wb") as f:
        f.write(("ply\nformat binary_little_endian 1.0\nelement vertex %d\n%selement face %d\n"
                 "property list uchar int vertex_indices\nend_header\n" % (3 * n, props, n)).encode())
        f.write(np.ascontiguousarray(np.concatenate(cols, axis=1), dtype="<f4").tobytes())
        rec = np.zeros(n, dtype=[("c", "u1"), ("i", "<i4", 3)])
        rec["c"] = 3
        rec["i"] = np.arange(3 * n, dtype=np.int32).reshape(n, 3)
        f.write(rec.tobytes())


TEXTURE_FLOAT_PARAMS = ("roughness", "uroughness", "vroughness")


def _texture_lines(scene, name, dirname):
    """The Texture statements of scene.texture_specs (and their PFMs); {material: material statement} for textured ones."""
    lines, mats = [], {}
    for mat, params in sorted(getattr(scene, "texture_specs", {}).items()):
        stmt = PBRT_MATERIAL[mat]
        for param, t in sorted((k, v) for k, v in params.items() if k != "params"):
            tex = "%s_%s" % (mat, param)
            pfm = "%s_tex_%s.pfm" % (name, tex)
            write_pfm(os.path.join(dirname, pfm), np.asarray(t["map"], np.float32))
            line = 'Texture "%s" "%s" "imagemap" "string filename" "%s"' % (tex, "float" if param in TEXTURE_FLOAT_PARAMS else "spectrum", pfm)
            for key, kind in (("wrap", "string"), ("trilinear", "bool"), ("maxanisotropy", "float"), ("scale", "float"),
                              ("gamma", "bool"), ("uscale", "float"), ("vscale", "float"), ("udelta", "float"), ("vdelta", "float")):
                if key in t:
                    v = t[key]
                    line += ' "%s %s" [%s]' % (kind, key, ('"%s"' % v) if kind == "string" else
                                               ('"true"' if v else '"false"') if kind == "bool" else "%.9g" % v)
            lines.append(line)
            stmt = re.sub(r' "\w+ %s" \[[^\]]*\]' % param, "", stmt) + ' "texture %s" "%s"' % (param, tex)
        if params.get("params"):
            stmt += " " + params["params"]
        mats[mat] = stmt
    return lines, mats


def _alpha_lines(scene, name, dirname):
    """The Texture statements of scene.alpha_specs (and their PFMs); {group: shape parameters naming its masks}."""
    lines, params = [], {}
    for group, kinds in sorted(getattr(scene, "alpha_specs", {}).items()):
        p = ""
        for kind, t in sorted(kinds.items()):
            if not isinstance(t, dict):
                p += ' "float %s" [%.9g]' % (kind, t)
                continue
            tex = "%s_%s" % (group, kind)
            pfm = "%s_alpha_%s.pfm" % (name, tex)
            m = np.asarray(t["map"], np.float32)
            write_pfm(os.path.join(dirname, pfm), np.repeat(m[:, :, None], 3, axis=2) if m.ndim == 2 else m)
            line = 'Texture "%s" "float" "imagemap" "string filename" "%s"' % (tex, pfm)
            for key, k2 in (("wrap", "string"), ("trilinear", "bool"), ("maxanisotropy", "float"), ("scale", "float"),
                            ("uscale", "float"), ("vscale", "float"), ("udelta", "float"), ("vdelta", "float")):
                if key in t:
                    v = t[key]
                    line += ' "%s %s" [%s]' % (k2, key, ('"%s"' % v) if k2 == "string" else
                                               ('"true"' if v else '"false"') if k2 == "bool" else "%.9g" % v)
            lines.append(line)
            p += ' "texture %s" "%s"' % (kind, tex)
        params[group] = p
    return lines, params


def write_pbrt(dirname, name, scene, xres, yres, spp, max_depth=5, strategy="uniform", pixel_bounds=None,
               eye=(0, 0, -4.5), look=(0, 0, 0), up=(0, 1, 0), fov=35.0, lens_radius=0.0, focal_distance=1e6,
               crop_window=None, film_scale=1.0, max_sample_luminance=None, sampler="sobol", pixel_filter=None,
               integrator="path", medium=None):
    """Appendix A.4 wrapper: the reference-readable twin of `scene`.  medium = dict(sigma_a=(r, g, b), sigma_s=(r, g, b),
    g=...): a homogeneous medium that fills the scene -- the camera starts in it and no surface is a medium transition
    (media/homogeneous.cpp, api.cpp:763-800, :892-898); meant for integrator="volpath"."""
    os.makedirs(dirname, exist_ok=True)
    lines = []
    if medium:
        lines += ['MakeNamedMedium "fog" "string type" "homogeneous" "rgb sigma_a" [%.9g %.9g %.9g] "rgb sigma_s" [%.9g %.9g %.9g] '
                  '"float g" [%.9g] "float scale" [1]' % (tuple(medium["sigma_a"]) + tuple(medium["sigma_s"]) + (medium.get("g", 0.0),)),
                  'MediumInterface "" "fog"']
    lines += ["LookAt %g %g %g  %g %g %g  %g %g %g" % (*eye, *look, *up),
             'Camera "perspective" "float fov" [%g]' % fov +
             (' "float lensradius" [%.9g] "float focaldistance" [%.9g]' % (lens_radius, focal_distance)
              if lens_radius > 0 else ""),
             'Film "image" "integer xresolution" [%d] "integer yresolution" [%d] "string filename" "%s.pfm"'
             % (xres, yres, name) +
             (' "float cropwindow" [%.9g %.9g %.9g %.9g]' % tuple(crop_window) if crop_window else "") +
             (' "float scale" [%.9g]' % film_scale if film_scale != 1.0 else "") +
             (' "float maxsampleluminance" [%.9g]' % max_sample_luminance if max_sample_luminance else ""),
             'Sampler "%s" "integer pixelsamples" [%d]' % (sampler, spp)]
    if pixel_filter:
        lines.append(FilterTables().get(pixel_filter)[0])
    integ = 'Integrator "%s" "integer maxdepth" [%d] "string lightsamplestrategy" "%s"' % (integrator, max_depth, strategy)
    if pixel_bounds is not None:
        integ += ' "integer pixelbounds" [%d %d %d %d]' % (pixel_bounds[0], pixel_bounds[2], pixel_bounds[1],
                                                          pixel_bounds[3])
    lines += [integ, "WorldBegin"]
    if medium:
        lines.append('MediumInterface "fog" "fog"')
    tex_lines, tex_mats = _texture_lines(scene, name, dirname)
    lines += tex_lines
    material = lambda m: tex_mats.get(m, PBRT_MATERIAL[m])
    alpha_lines, alpha_params = _alpha_lines(scene, name, dirname)
    lines += alpha_lines
    for q in scene.light_quads:
        # quad() stores (p0 p1 p2)(p0 p2 p3); recover the 4 corners
        pts = [q[0][0], q[0][1], q[0][2], q[1][2]]
        flat = " ".join("%.9g" % v for p in pts for v in p)
        lines += ["AttributeBegin",
                  '  AreaLightSource "diffuse" "rgb L" [%g %g %g]%s' %
                  (scene.light_L, scene.light_L, scene.light_L,
                   ' "bool twosided" "true"' if scene.two_sided else ""),
                  '  Material "matte" "rgb Kd" [0 0 0]',
                  '  Shape "trianglemesh" "integer indices" [0 1 2 0 2 3] "point P" [%s]' % flat + alpha_params.get("light", ""),
                  "AttributeEnd"]
    for dl in getattr(scene, "delta_specs", ()):
        val = dl.get("I", dl.get("L", 1.0))
        rgb = "%.9g %.9g %.9g" % ((val,) * 3 if np.isscalar(val) else tuple(val))
        f_, t_ = dl.get("from_", (0, 0, 0)), dl.get("to", (0, 0, 1))
        if dl["kind"] == "point":
            lines.append('LightSource "point" "rgb I" [%s] "point from" [%.9g %.9g %.9g]' % ((rgb,) + tuple(f_)))
        elif dl["kind"] == "spot":
            lines.append('LightSource "spot" "rgb I" [%s] "point from" [%.9g %.9g %.9g] "point to" [%.9g %.9g %.9g] '
                         '"float coneangle" [%.9g] "float conedeltaangle" [%.9g]'
                         % ((rgb,) + tuple(f_) + tuple(t_) + (dl.get("coneangle", 30.0), dl.get("conedelta", 5.0))))
        else:
            lines.append('LightSource "distant" "rgb L" [%s] "point from" [%.9g %.9g %.9g] "point to" [%.9g %.9g %.9g]'
                         % ((rgb,) + tuple(f_) + tuple(t_)))
    for k, il in enumerate(getattr(scene, "infinite_specs", ())):
        rgb3 = lambda v: "%.9g %.9g %.9g" % ((v,) * 3 if np.isscalar(v) else tuple(v))
        light = 'LightSource "infinite" "rgb L" [%s]' % rgb3(il.get("L", 1.0))
        if "scale" in il:
            light += ' "rgb scale" [%s]' % rgb3(il["scale"])
        if il.get("map") is not None:
            sky = "%s_sky%d.pfm" % (name, k)
            write_pfm(os.path.join(dirname, sky), np.asarray(il["map"], np.float32))
            light += ' "string mapname" "%s"' % sky
        lines += ["AttributeBegin"] + ["  %s %s" % (op, " ".join("%.9g" % v for v in args)) for op, args in il.get("steps", ())]
        lines += ["  " + light, "AttributeEnd"]
    for m, part in enumerate(scene.ply_parts):
        ply = "%s_m%d.ply" % (name, m)
        sel = scene.material_id == m
        write_ply(os.path.join(dirname, ply), part,
                  scene.normals[sel] if m in scene.shading_normals else None,
                  scene.uvs[sel] if m in scene.uv_meshes else None)
        if m in scene.reverse_orientation:
            lines += ["AttributeBegin", "ReverseOrientation"]
        lines += [material(scene.material_names[m]),
                  'Shape "plymesh" "string filename" "%s"' % ply + alpha_params.get(scene.material_names[m], "")]
        if m in scene.reverse_orientation:
            lines += ["AttributeEnd"]
    for k, (o, part) in enumerate(zip(getattr(scene, "object_specs", ()), getattr(scene, "object_parts", ()))):
        ply = "%s_obj%d.ply" % (name, k)
        write_ply(os.path.join(dirname, ply), part)
        lines += ['ObjectBegin "obj%d"' % k, "  " + material(o.get("material", "matte")),
                  '  Shape "plymesh" "string filename" "%s"' % ply + alpha_params.get(o.get("material", "matte"), ""), "ObjectEnd"]
    for ins in getattr(scene, "instance_specs", ()):
        lines.append("AttributeBegin")
        lines += ["  %s %s" % (op, " ".join("%.9g" % v for v in args)) for op, args in instance_steps(ins)]
        lines += ['  ObjectInstance "obj%d"' % ins["object"], "AttributeEnd"]
    for sp in getattr(scene, "sphere_specs", ()):
        lines.append("AttributeBegin")
        if sp.get("emit"):
            lines.append('  AreaLightSource "diffuse" "rgb L" [%g %g %g]%s' %
                         (sp["emit"], sp["emit"], sp["emit"], ' "bool twosided" "true"' if sp.get("two_sided") else ""))
        mat = sp.get("material", "black")
        if sp.get("boundary"):  # a null-material sphere that bounds a homogeneous medium (oracle groundwork only)
            b = sp["boundary"]
            lines += ['  MakeNamedMedium "cloud%d" "string type" "homogeneous" "rgb sigma_a" [%.9g %.9g %.9g] "rgb sigma_s" '
                      '[%.9g %.9g %.9g] "float g" [%.9g] "float scale" [1]' % ((len(lines),) + tuple(b["sigma_a"]) + tuple(b["sigma_s"]) + (b.get("g", 0.0),)),
                      '  MediumInterface "cloud%d" "%s"' % (len(lines), "fog" if medium else ""), '  Material ""']
        else:
            lines.append("  " + ('Material "matte" "rgb Kd" [0 0 0]' if mat == "black" else material(mat)))
        lines.append("  Translate %.9g %.9g %.9g" % tuple(sp["center"]))
        if sp.get("scale"):
            lines.append("  Scale %.9g %.9g %.9g" % tuple(sp["scale"]))
        if sp.get("reverse_orientation"):
            lines.append("  ReverseOrientation")
        lines.append('  Shape "sphere" "float radius" [%.9g]' % sp["radius"] +
                     "".join(' "float %s" [%.9g]' % (k, sp[k]) for k in ("zmin", "zmax", "phimax") if k in sp))
        lines.append("AttributeEnd")
    lines.append("WorldEnd")
    path = os.path.join(dirname, name + ".pbrt")
    with open(path, "w") as f:
        f.write("\n".join(lines) + "\n")
    return path


def read_dump_infinite(path, abi):
    """{light index: tables for Scene.set_infinite_light} of the InfiniteAreaLights an RGBSpectrum host wrote to its
    B200PT_DUMP_SCENE file (host/gpupath.cpp appends them after the descriptors)."""
    return _read_dump_tail(path, abi)[0]


def read_dump_alpha(path, abi):
    """(masks, alpha ids, shadowalpha ids) of the alpha masks an RGBSpectrum host wrote to its B200PT_DUMP_SCENE file
    (behind the texture tables): masks are dicts {texels ([h][w] array, None for a constant 0), wrap, su, sv, du, dv}
    for Scene.add_alpha_mask, the ids one per triangle for Scene.set_alpha_masks; ([], None, None) without masks."""
    return _read_dump_tail(path, abi)[2]


def read_dump_textures(path, abi):
    """(mipmaps, binds) of the image textures an RGBSpectrum host wrote to its B200PT_DUMP_SCENE file (behind the infinite
    lights' tables): mipmaps are dicts {levels ([h][w][3] or [h][w] arrays), wrap, trilinear, max_anisotropy, weight_lut}
    for Scene.add_mipmap, binds are dicts {material, slot, mipmap, su, sv, du, dv, remap} in the host's material order."""
    return _read_dump_tail(path, abi)[1]


TEXTURE_MARKER = -2  # host/gpupath.cpp: the image textures' tables follow the infinite lights' behind this int32
ALPHA_MARKER = -3  # ... and the alpha masks' tables follow those behind this one


def _read_dump_tail(path, abi):
    raw = open(path, "rb").read()
    hdr = np.frombuffer(raw, np.int64, 8)
    nt, nm, nl, nsph, has_n, has_uv = (int(x) for x in hdr[1:7])
    off = 64 + nt * (36 + 4 + 4 + 1 + 1) + (nt * 36 if has_n else 0) + (nt * 24 if has_uv else 0)
    off += nm * C.sizeof(abi.Material) + nl * C.sizeof(abi.AreaLight) + nsph * C.sizeof(abi.Sphere)
    off += C.sizeof(abi.CameraDesc) + 48 + C.sizeof(abi.IntegratorDesc) + 24  # film desc (48 B), six sampler ints
    if int(np.frombuffer(raw, np.int32, 1, off)[0]) != 0:
        raise ValueError("%s: not an RGBSpectrum host's dump" % path)
    off += 4
    out = {}

    def take(n, shape=None):
        nonlocal off
        a = np.frombuffer(raw, np.float32, n, off).copy()
        off += 4 * n
        return a.reshape(shape) if shape else a

    def ints(n):
        nonlocal off
        a = [int(x) for x in np.frombuffer(raw, np.int32, n, off)]
        off += 4 * n
        return a
    marker = lambda: int(np.frombuffer(raw, np.int32, 1, off)[0]) if off < len(raw) else None
    while off < len(raw) and marker() not in (TEXTURE_MARKER, ALPHA_MARKER):
        light, w, h, nu, nv = ints(5)
        out[light] = dict(texels=take(w * h * 3, (h, w, 3)), light_to_world=take(16), cond_func=take(nv * nu, (nv, nu)),
                          cond_cdf=take(nv * (nu + 1), (nv, nu + 1)), cond_func_int=take(nv), marg_func=take(nv),
                          marg_cdf=take(nv + 1), marg_func_int=take(1)[0], power_rgb=take(3))
    mips, binds = [], []
    if marker() == TEXTURE_MARKER:
        _, nmip, nbind = ints(3)
        for _ in range(nmip):
            nlev, ch, wrap, tri = ints(4)
            aniso = float(take(1)[0])
            lut = take(128)
            levels = []
            for _ in range(nlev):
                w, h = ints(2)
                levels.append(take(w * h * ch, (h, w, 3) if ch == 3 else (h, w)))
            mips.append(dict(levels=levels, wrap=wrap, trilinear=tri, max_anisotropy=aniso, weight_lut=lut))
        for _ in range(nbind):
            mat, slot, mip = ints(3)
            su, sv, du, dv = (float(x) for x in take(4))
            binds.append(dict(material=mat, slot=slot, mipmap=mip, su=su, sv=sv, du=du, dv=dv, remap=ints(1)[0]))
    masks, alpha, shadow = [], None, None
    if marker() == ALPHA_MARKER:
        _, nmask = ints(2)
        for _ in range(nmask):
            w, h, wrap = ints(3)
            su, sv, du, dv = (float(x) for x in take(4))
            masks.append(dict(texels=take(w * h, (h, w)) if w else None, wrap=wrap, su=su, sv=sv, du=du, dv=dv))
        alpha, shadow = np.array(ints(nt), np.int32), np.array(ints(nt), np.int32)
    if off != len(raw):
        raise ValueError("%s: truncated infinite-light, texture or alpha-mask tables" % path)
    return out, (mips, binds), (masks, alpha, shadow)


def read_pfm(path):
    with open(path, "rb") as f:
        tag = f.readline().strip()
        w, h = map(int, f.readline().split())
        scale = float(f.readline())
        nc = 3 if tag == b"PF" else 1
        data = np.frombuffer(f.read(), dtype="<f4" if scale < 0 else ">f4").reshape(h, w, nc)
    return np.ascontiguousarray(data[::-1]).astype(np.float32)


def write_pfm(path, rgb):
    h, w, _ = rgb.shape
    with open(path, "wb") as f:
        f.write(b"PF\n%d %d\n-1.000000\n" % (w, h))
        f.write(np.ascontiguousarray(rgb[::-1], dtype="<f4").tobytes())


class SobolTables:
    """tests/golden/sobol_tables.bin: the Joe-Kuo generator matrices pbrt uses
    (first 256 of its 1024 dimensions) + the (0,2)-net index maps, dumped from
    the reference's own tables by oracle/probe `tables`.  A pbrt host passes
    its in-memory tables instead (see INTEGRATION.md)."""

    def __init__(self, path=None):
        path = path or os.path.join(GOLDEN_DIR, "sobol_tables.bin")
        raw = open(path, "rb").read()
        magic, nd, msize, nrows = struct.unpack_from("<4I", raw, 0)
        assert magic == 0x32424F53 and msize == 52
        off = 16
        self.n_dims = nd
        self.matrices32 = np.frombuffer(raw, "<u4", nd * 52, off).copy()
        off += nd * 52 * 4
        self.vdc = np.frombuffer(raw, "<u8", nrows * 52, off).reshape(nrows, 52).copy()
        off += nrows * 52 * 8
        self.vdc_inv = np.frombuffer(raw, "<u8", nrows * 52, off).reshape(nrows, 52).copy()


class HaltonTables:
    """tests/golden/halton_perms.bin: HaltonSampler::radicalInversePermutations for the first
    n_dims prime bases, dumped from the reference by oracle/probe `haltonperms` (the table is the
    output of pbrt's PCG32 shuffle with the default seed; a pbrt host passes its own copy)."""

    def __init__(self, path=None):
        path = path or os.path.join(GOLDEN_DIR, "halton_perms.bin")
        raw = open(path, "rb").read()
        magic, nd, count, _ = struct.unpack_from("<4I", raw, 0)
        assert magic == 0x544C4148
        self.n_dims = nd
        self.perms = np.frombuffer(raw, "<u2", count, 16).copy()


class FilterTables:
    """tests/golden/filter_tables.json: radius and Film::filterTable (16x16 weights, film.cpp:68-77) of a few
    PixelFilter configurations, dumped from the reference by oracle/probe `filtertable`.  A pbrt host passes the
    table of its own Film."""

    def __init__(self, path=None):
        import json
        self.entries = json.load(open(path or os.path.join(GOLDEN_DIR, "filter_tables.json")))

    def get(self, key):
        e = self.entries[key]
        radius = [float.fromhex(v) for v in e["radius"]]
        table = np.array([float.fromhex(v) for v in e["table"]], np.float32)
        return e["pbrt"], radius, table


def rank_tiles(n_tiles, rank, world):
    """Image-space decomposition used for multi-GPU runs (SURVEY 8e): tile i -> rank i mod N.
    Interleaving balances sky / geometry tiles; every rank keeps the FULL-film sampler so the
    union of the shards is sample-identical to a single-GPU render."""
    return np.arange(n_tiles, dtype=np.int32)[rank::world]


def round_up_pow2(v):
    return 1 << (int(v) - 1).bit_length()


class RenderSetup:
    """camera + film + sampler + integrator descriptors for a full-film render
    with the default box filter (sample bounds == cropped pixel bounds)."""

    def __init__(self, xres, yres, spp, max_depth=5, strategy=abi.LIGHTS_UNIFORM, pixel_bounds=None,
                 eye=(0, 0, -4.5), look=(0, 0, 0), up=(0, 1, 0), fov=35.0, tables=None, camera=None,
                 lens_radius=0.0, focal_distance=1e6, crop_window=None, film_scale=1.0, max_sample_luminance=None,
                 sampler="sobol", pixel_filter=None, integrator="path", medium=None, spectral_tables=None,
                 boundaries=None):
        from . import host_perspective_camera
        self.xres, self.yres = xres, yres
        self.sampler_name = sampler
        self.tables = tables or (HaltonTables() if sampler == "halton" else SobolTables())
        self.camera = camera if camera is not None else host_perspective_camera(eye, look, up, fov, xres, yres)
        if lens_radius > 0:
            self.camera.lens_radius = lens_radius
            self.camera.focal_distance = focal_distance
        self.film = abi.FilmDesc()
        self.film.full_resolution[:] = [xres, yres]
        cb = [0, 0, xres, yres]
        if crop_window:  # Film ctor, film.cpp:54-58: ceil(res * crop) in float
            f32 = np.float32
            cw = [f32(c) for c in crop_window]  # x0 x1 y0 y1
            cb = [int(np.ceil(f32(xres) * cw[0])), int(np.ceil(f32(yres) * cw[2])),
                  int(np.ceil(f32(xres) * cw[1])), int(np.ceil(f32(yres) * cw[3]))]
        self.crop = cb
        self.film.cropped_bounds[:] = cb
        self.film.filter_radius[:] = [0.5, 0.5]
        self.pixel_filter = pixel_filter
        sb = list(cb)
        if pixel_filter:  # a key of tests/golden/filter_tables.json
            _, radius, self._filter_table = FilterTables().get(pixel_filter)
            self.film.filter_radius[:] = radius
            self.film.filter_table = abi.ptr(self._filter_table)
            # Film::GetSampleBounds, film.cpp:80-86
            f32 = np.float32
            sb = [int(np.floor(f32(cb[0]) + f32(0.5) - f32(radius[0]))), int(np.floor(f32(cb[1]) + f32(0.5) - f32(radius[1]))),
                  int(np.ceil(f32(cb[2]) - f32(0.5) + f32(radius[0]))), int(np.ceil(f32(cb[3]) - f32(0.5) + f32(radius[1])))]
        self.sample_bounds = sb
        self.film.scale = film_scale
        self.film.max_sample_luminance = max_sample_luminance if max_sample_luminance else float("inf")
        self.sampler = abi.SamplerDesc()
        # Film::GetSampleBounds; with the box filter of radius 0.5 == the cropped pixel bounds (film.cpp:80-86)
        self.sampler.sample_bounds[:] = sb
        self.sampler.n_dimensions = self.tables.n_dims
        if sampler == "halton":  # halton.cpp:65-93: any sample count
            self.sampler.type = abi.SAMPLER_HALTON
            self.sampler.samples_per_pixel = spp
            self.sampler.halton_permutations = abi.ptr(self.tables.perms)
        else:
            self.sampler.samples_per_pixel = round_up_pow2(spp)
            self._sobol_tables(sb)
        self.integrator = abi.IntegratorDesc()
        self.integrator.max_depth = max_depth
        self.integrator.rr_threshold = 1.0
        self.integrator.light_strategy = strategy
        self.integrator.pixel_bounds[:] = pixel_bounds or sb
        # integrator="volpath": VolPathIntegrator; medium = dict(sigma_a=, sigma_s=, g=): homogeneous, around everything
        self.integrator.volumetric = 1 if integrator == "volpath" else 0
        if medium:
            self.integrator.medium.present = 1
            self.integrator.medium.sigma_a[:] = list(medium["sigma_a"])
            self.integrator.medium.sigma_s[:] = list(medium["sigma_s"])
            self.integrator.medium.g = medium.get("g", 0.0)
            if spectral_tables is not None:  # a SampledSpectrum host: the medium's 60-bin spectra (fixtures of the probe)
                f32 = np.float32
                lut = {tuple(np.array([float.fromhex(x) for x in rgb], f32).view(np.uint32).tolist()):
                       np.array([float.fromhex(x) for x in spec], f32) for rgb, spec in spectral_tables["spectra"]}
                self._medium_spectra = np.stack([lut[tuple(np.array(list(medium[k]), f32).view(np.uint32).tolist())]
                                                 for k in ("sigma_a", "sigma_s")])
                self.integrator.medium.spectra = abi.ptr(self._medium_spectra)
        # boundaries = the scene's sphere specs (SceneArrays.sphere_specs): those with a `boundary` entry are null-material
        # surfaces around a homogeneous medium (MediumInterface "inside" "outside" + Material "")
        specs = [(k, sp["boundary"]) for k, sp in enumerate(boundaries or ()) if sp.get("boundary")]
        if specs:
            self._bounded = (abi.Medium * len(specs))()
            self._sphere_medium = np.full(len(boundaries), -1, np.int32)
            for j, (k, b) in enumerate(specs):
                self._bounded[j].present = 1
                self._bounded[j].sigma_a[:] = list(b["sigma_a"])
                self._bounded[j].sigma_s[:] = list(b["sigma_s"])
                self._bounded[j].g = b.get("g", 0.0)
                self._sphere_medium[k] = j
            self.integrator.n_bounded_media = len(specs)
            self.integrator.bounded_media = C.cast(self._bounded, C.c_void_p)
            self.integrator.sphere_medium = abi.ptr(self._sphere_medium)

    def _sobol_tables(self, cb):
        res = round_up_pow2(max(cb[2] - cb[0], cb[3] - cb[1]))
        m = res.bit_length() - 1
        self._vdc = np.ascontiguousarray(self.tables.vdc[max(m - 1, 0)])
        self._vdc_inv = np.ascontiguousarray(self.tables.vdc_inv[max(m - 1, 0)])
        self.sampler.matrices32 = abi.ptr(self.tables.matrices32)
        self.sampler.vdc = abi.ptr(self._vdc)
        self.sampler.vdc_inv = abi.ptr(self._vdc_inv)

    @property
    def n_tiles(self):
        sb = self.sample_bounds
        return ((sb[2] - sb[0] + 15) // 16) * ((sb[3] - sb[1] + 15) // 16)
