"""pbrt-v3-distributed_b200: H100-native hot path of pbrt-v3-distributed.

Host-side Python mirror of the C ABI in include/b200pt.h (ctypes).  The product
is libb200pt.so (hand-written sm_90a CUDA + host C++); this module only loads
it and wraps handles.  There is no CPU fallback: if the library is missing the
import fails loudly, and every compute call fails if no CUDA device is usable.

The directory name contains '-', so the package is imported through
`__graft_entry__.load_package()` under the module name
`pbrt_v3_distributed_b200`.
"""
import ctypes as C
import os

import numpy as np

from . import abi

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libb200pt.so")
# profiles/ A/B runs load an experimental build of the same sources (make VARIANT=<name> EXTRA=-D...) instead
if os.environ.get("B200PT_LIB_VARIANT"):
    LIB_PATH = os.path.join(_HERE, "_variants", os.environ["B200PT_LIB_VARIANT"], "libb200pt.so")

if not os.path.exists(LIB_PATH):
    raise ImportError("libb200pt.so is not built (run `python -c 'import __graft_entry__ as g; g.build()'`); "
                      "there is no CPU fallback")

lib = C.CDLL(LIB_PATH)

_vp, _i32, _i64, _u64 = C.c_void_p, C.c_int32, C.c_int64, C.c_uint64
_SIGNATURES = {
    "b200pt_abi_version": (C.c_int, []),
    "b200pt_last_error": (C.c_char_p, []),
    "b200pt_ctx_create": (C.c_int, [C.c_int, C.POINTER(_vp)]),
    "b200pt_ctx_destroy": (None, [_vp]),
    "b200pt_ctx_synchronize": (C.c_int, [_vp]),
    "b200pt_ctx_stream": (_u64, [_vp]),
    "b200pt_ctx_set_option": (C.c_int, [_vp, C.c_char_p, C.c_int64]),
    "b200pt_scene_create": (C.c_int, [_vp, C.POINTER(abi.SceneDesc), C.POINTER(_vp)]),
    "b200pt_scene_destroy": (None, [_vp]),
    "b200pt_scene_upload": (C.c_int, [_vp, C.POINTER(_u64)]),
    "b200pt_scene_info": (C.c_int, [_vp, C.POINTER(_u64), C.POINTER(_u64), C.POINTER(_u64)]),
    "b200pt_scene_set_infinite_light": (C.c_int, [_vp, _i32, C.POINTER(abi.InfiniteLight)]),
    "b200pt_scene_add_mipmap": (C.c_int, [_vp, C.POINTER(abi.Mipmap), C.POINTER(_i32)]),
    "b200pt_scene_bind_texture": (C.c_int, [_vp, _i32, _i32, _i32, C.c_float, C.c_float, C.c_float, C.c_float, _i32]),
    "b200pt_scene_add_alpha_mask": (C.c_int, [_vp, C.POINTER(abi.AlphaMask), C.POINTER(_i32)]),
    "b200pt_scene_set_alpha_masks": (C.c_int, [_vp, _vp, _vp]),
    "b200pt_trace_closest": (C.c_int, [_vp, _vp, _vp, _i64]),
    "b200pt_trace_any": (C.c_int, [_vp, _vp, _vp, _i64]),
    "b200pt_trace_closest_dev": (C.c_int, [_vp, _u64, _u64, _i64]),
    "b200pt_trace_any_dev": (C.c_int, [_vp, _u64, _u64, _i64]),
    "b200pt_render_create": (C.c_int, [_vp, C.POINTER(abi.CameraDesc), C.POINTER(abi.FilmDesc),
                                       C.POINTER(abi.SamplerDesc), C.POINTER(abi.IntegratorDesc),
                                       C.POINTER(_vp)]),
    "b200pt_render_destroy": (None, [_vp]),
    "b200pt_render_tile_counts": (C.c_int, [_vp, C.POINTER(_i32), C.POINTER(_i32)]),
    "b200pt_film_clear": (C.c_int, [_vp]),
    "b200pt_render_tiles": (C.c_int, [_vp, _vp, _i64]),
    "b200pt_film_device_buffer": (C.c_int, [_vp, C.POINTER(_u64), C.POINTER(_u64)]),
    "b200pt_film_read_raw": (C.c_int, [_vp, _vp]),
    "b200pt_film_read_rgb": (C.c_int, [_vp, _vp]),
    "b200pt_comm_create": (C.c_int, [_vp, C.c_int, C.c_int, C.c_char_p, C.POINTER(_vp)]),
    "b200pt_comm_from_nccl": (C.c_int, [_vp, _vp, C.c_int, C.c_int, C.POINTER(_vp)]),
    "b200pt_comm_destroy": (None, [_vp]),
    "b200pt_film_reduce": (C.c_int, [_vp, _vp, C.c_int]),
    "b200pt_debug_sobol": (C.c_int, [_vp, _i32, _i32, _i64, _i32, _i32, _vp]),
    "b200pt_debug_camera_rays": (C.c_int, [_vp, _i32, _i32, _i32, _vp]),
    "b200pt_debug_pixel_samples": (C.c_int, [_vp, _i32, _i32, _vp]),
    "b200pt_render_set_option": (C.c_int, [_vp, C.c_char_p, C.c_int]),
    "b200pt_get_stats": (C.c_int, [_vp, C.POINTER(abi.Stats)]),
    "b200pt_reset_stats": (C.c_int, [_vp]),
    "b200pt_host_perspective_camera": (C.c_int, [C.POINTER(C.c_float), C.POINTER(C.c_float),
                                                 C.POINTER(C.c_float), C.c_float, _i32, _i32,
                                                 C.POINTER(abi.CameraDesc)]),
    "b200pt_host_roughness_to_alpha": (C.c_float, [C.c_float]),
    "b200pt_host_oren_nayar": (None, [C.c_float, C.POINTER(C.c_float), C.POINTER(C.c_float)]),
    "b200pt_host_spot_light": (None, [C.POINTER(C.c_float), C.POINTER(C.c_float), C.c_float, C.c_float, _vp]),
    "b200pt_host_sphere_params": (None, [C.c_float, C.c_float, C.c_float, C.c_float, C.POINTER(C.c_float)]),
}
EXPORTED_SYMBOLS = sorted(_SIGNATURES)


def _bind():
    missing = []
    for name, (res, args) in _SIGNATURES.items():
        try:
            fn = getattr(lib, name)
        except AttributeError:
            missing.append(name)
            continue
        fn.restype = res
        fn.argtypes = args
    return missing


MISSING_SYMBOLS = _bind()


class B200ptError(RuntimeError):
    pass


def _check(rc):
    if rc != 0:
        raise B200ptError("b200pt error %d: %s" % (rc, lib.b200pt_last_error().decode()))


def host_perspective_camera(eye, look, up, fov, xres, yres):
    out = abi.CameraDesc()
    f3 = C.c_float * 3
    _check(lib.b200pt_host_perspective_camera(f3(*eye), f3(*look), f3(*up), fov, xres, yres, C.byref(out)))
    return out


def host_roughness_to_alpha(r):
    return float(lib.b200pt_host_roughness_to_alpha(r))


def host_spot_light(light, from_, to, coneangle, conedelta):
    """Fills the spot-light fields of an abi.AreaLight like CreateSpotLight does."""
    f = (C.c_float * 3)(*from_)
    t = (C.c_float * 3)(*to)
    lib.b200pt_host_spot_light(f, t, coneangle, conedelta, C.byref(light))


def host_sphere_params(radius, zmin, zmax, phimax_degrees):
    out = (C.c_float * 5)()
    lib.b200pt_host_sphere_params(radius, zmin, zmax, phimax_degrees, out)
    return list(out)


def host_oren_nayar(sigma_degrees):
    a, b = C.c_float(), C.c_float()
    lib.b200pt_host_oren_nayar(sigma_degrees, C.byref(a), C.byref(b))
    return a.value, b.value


class Context:
    def __init__(self, device=0):
        self.h = _vp()
        _check(lib.b200pt_ctx_create(device, C.byref(self.h)))

    def synchronize(self):
        _check(lib.b200pt_ctx_synchronize(self.h))

    def set_option(self, key, value):
        _check(lib.b200pt_ctx_set_option(self.h, key.encode(), int(value)))

    @property
    def stream(self):
        return int(lib.b200pt_ctx_stream(self.h))

    def close(self):
        if self.h:
            lib.b200pt_ctx_destroy(self.h)
            self.h = _vp()


class Scene:
    """Device-resident triangles + 8-wide compressed BVH (b200pt_scene_create)."""

    def __init__(self, ctx, desc, keepalive=None):
        self.ctx = ctx
        self._keep = keepalive
        self.h = _vp()
        self.n_triangles = int(desc.n_triangles)
        _check(lib.b200pt_scene_create(ctx.h, C.byref(desc), C.byref(self.h)))

    def upload(self):
        n = _u64()
        _check(lib.b200pt_scene_upload(self.h, C.byref(n)))
        return n.value

    def info(self):
        a, b, c = _u64(), _u64(), _u64()
        _check(lib.b200pt_scene_info(self.h, C.byref(a), C.byref(b), C.byref(c)))
        return {"node_bytes": a.value, "tri_bytes": b.value, "n_nodes": c.value}

    def set_infinite_light(self, light, tables):
        """b200pt_scene_set_infinite_light: `tables` is a dict of the host's InfiniteAreaLight data -- texels [h][w][3],
        light_to_world (16), cond_func [nv][nu], cond_cdf [nv][nu+1], cond_func_int [nv], marg_func [nv],
        marg_cdf [nv+1], marg_func_int, power_rgb (3).  The library copies them."""
        f32 = lambda k: np.ascontiguousarray(tables[k], dtype=np.float32)
        arrs = {k: f32(k) for k in ("texels", "cond_func", "cond_cdf", "cond_func_int", "marg_func", "marg_cdf")}
        rec = abi.InfiniteLight()
        rec.height, rec.width = arrs["texels"].shape[:2]
        rec.nv, rec.nu = arrs["cond_func"].shape
        for k, a in arrs.items():
            setattr(rec, k, a.ctypes.data)
        rec.light_to_world[:] = [float(v) for v in f32("light_to_world").reshape(-1)]
        rec.marg_func_int = float(np.float32(tables["marg_func_int"]))
        rec.power_rgb[:] = [float(v) for v in f32("power_rgb")]
        _check(lib.b200pt_scene_set_infinite_light(self.h, int(light), C.byref(rec)))

    def add_mipmap(self, levels, wrap, trilinear, max_anisotropy, weight_lut):
        """b200pt_scene_add_mipmap: `levels` are the pyramid's texel arrays, [h][w][3] (spectrum) or [h][w] (float);
        returns the MIPMap's id.  The library copies the texels."""
        arrs = [np.ascontiguousarray(a, dtype=np.float32) for a in levels]
        rec = abi.Mipmap()
        rec.n_levels = len(arrs)
        rec.channels = 3 if arrs[0].ndim == 3 else 1
        for i, a in enumerate(arrs[:abi.MIPMAP_MAX_LEVELS]):
            rec.height[i], rec.width[i] = a.shape[:2]
            rec.texels[i] = a.ctypes.data
        rec.wrap, rec.trilinear, rec.max_anisotropy = int(wrap), int(trilinear), float(max_anisotropy)
        rec.weight_lut[:] = [float(v) for v in np.asarray(weight_lut, dtype=np.float32)]
        out = _i32()
        _check(lib.b200pt_scene_add_mipmap(self.h, C.byref(rec), C.byref(out)))
        return out.value

    def bind_texture(self, material, slot, mipmap, su=1.0, sv=1.0, du=0.0, dv=0.0, remap_roughness=False):
        """b200pt_scene_bind_texture: MIPMap `mipmap` under UVMapping2D(su, sv, du, dv) on parameter `slot` (abi.TEX_*)
        of material `material`."""
        _check(lib.b200pt_scene_bind_texture(self.h, int(material), int(slot), int(mipmap), su, sv, du, dv,
                                             1 if remap_roughness else 0))

    def add_alpha_mask(self, texels=None, wrap=abi.WRAP_REPEAT, su=1.0, sv=1.0, du=0.0, dv=0.0):
        """b200pt_scene_add_alpha_mask: `texels` is level 0 of the mask's MIPMap, [h][w]; None is ConstantTexture(0).
        Returns the mask's id.  The library copies the texels."""
        rec = abi.AlphaMask()
        arr = None
        if texels is not None:
            arr = np.ascontiguousarray(texels, dtype=np.float32)
            if arr.ndim != 2:
                raise ValueError("an alpha mask is one float channel, [h][w]")
            rec.height, rec.width = arr.shape
            rec.texels = arr.ctypes.data
        rec.wrap, rec.su, rec.sv, rec.du, rec.dv = int(wrap), su, sv, du, dv
        out = _i32()
        _check(lib.b200pt_scene_add_alpha_mask(self.h, C.byref(rec), C.byref(out)))
        return out.value

    def set_alpha_masks(self, alpha=None, shadow_alpha=None):
        """b200pt_scene_set_alpha_masks: per triangle of the scene's numbering, the alpha / shadowalpha mask id or -1
        (None: no mask of that kind).  Before the scene's first trace or render."""
        arrs = []
        for a in (alpha, shadow_alpha):
            if a is not None:
                a = np.ascontiguousarray(a, dtype=np.int32)
                if a.shape != (self.n_triangles,):
                    raise ValueError("set_alpha_masks: %s ids for %d triangles" % (a.shape, self.n_triangles))
            arrs.append(a)
        _check(lib.b200pt_scene_set_alpha_masks(self.h, abi.ptr(arrs[0]), abi.ptr(arrs[1])))

    def trace_closest(self, rays):
        rays = np.ascontiguousarray(rays, dtype=abi.RAY_DTYPE)
        hits = np.zeros(len(rays), dtype=abi.HIT_DTYPE)
        _check(lib.b200pt_trace_closest(self.h, abi.ptr(rays), abi.ptr(hits), len(rays)))
        return hits

    def trace_any(self, rays):
        rays = np.ascontiguousarray(rays, dtype=abi.RAY_DTYPE)
        occ = np.zeros(len(rays), dtype=np.uint8)
        _check(lib.b200pt_trace_any(self.h, abi.ptr(rays), abi.ptr(occ), len(rays)))
        return occ

    def trace_closest_dev(self, rays_ptr, hits_ptr, n):
        _check(lib.b200pt_trace_closest_dev(self.h, rays_ptr, hits_ptr, n))

    def trace_any_dev(self, rays_ptr, occ_ptr, n):
        _check(lib.b200pt_trace_any_dev(self.h, rays_ptr, occ_ptr, n))

    def close(self):
        if self.h:
            lib.b200pt_scene_destroy(self.h)
            self.h = _vp()


class Comm:
    """NCCL communicator for the film merge of a multi-process render (b200pt_comm_create: rank 0 publishes the
    NCCL id through `id_file`, a path every rank can reach)."""

    def __init__(self, ctx, rank, world_size, id_file):
        self.h = _vp()
        _check(lib.b200pt_comm_create(ctx.h, rank, world_size, os.fsencode(id_file), C.byref(self.h)))

    def close(self):
        if self.h:
            lib.b200pt_comm_destroy(self.h)
            self.h = _vp()


class Render:
    """SamplerIntegrator::Render replacement bound to a scene (b200pt_render_create)."""

    def __init__(self, scene, setup):
        self.scene = scene
        self.setup = setup
        self.h = _vp()
        _check(lib.b200pt_render_create(scene.h, C.byref(setup.camera), C.byref(setup.film),
                                        C.byref(setup.sampler), C.byref(setup.integrator), C.byref(self.h)))
        nx, ny = _i32(), _i32()
        _check(lib.b200pt_render_tile_counts(self.h, C.byref(nx), C.byref(ny)))
        self.tiles_x, self.tiles_y = nx.value, ny.value
        cb = setup.film.cropped_bounds
        self.width, self.height = cb[2] - cb[0], cb[3] - cb[1]

    @property
    def n_tiles(self):
        return self.tiles_x * self.tiles_y

    def clear(self):
        _check(lib.b200pt_film_clear(self.h))

    def render_tiles(self, tiles=None, n=None):
        if tiles is None:
            _check(lib.b200pt_render_tiles(self.h, None, self.n_tiles if n is None else n))
        else:
            t = np.ascontiguousarray(tiles, dtype=np.int32)
            _check(lib.b200pt_render_tiles(self.h, abi.ptr(t), len(t)))

    def film_device_buffer(self):
        p, n = _u64(), _u64()
        _check(lib.b200pt_film_device_buffer(self.h, C.byref(p), C.byref(n)))
        return p.value, n.value

    def film_reduce(self, comm, root=0):
        """Adds every rank's raw film sums into `root`'s film (one ncclReduce, b200pt_film_reduce)."""
        _check(lib.b200pt_film_reduce(self.h, comm.h, root))

    def read_raw(self):
        out = np.zeros((self.height, self.width, 4), np.float32)
        _check(lib.b200pt_film_read_raw(self.h, abi.ptr(out)))
        return out

    def read_rgb(self):
        out = np.zeros((self.height, self.width, 3), np.float32)
        _check(lib.b200pt_film_read_rgb(self.h, abi.ptr(out)))
        return out

    def debug_sobol(self, px, py, sample, dim0, n):
        out = np.zeros(n, np.float32)
        _check(lib.b200pt_debug_sobol(self.h, px, py, sample, dim0, n, abi.ptr(out)))
        return out

    def debug_camera_rays(self, px, py, n):
        out = np.zeros(n, dtype=abi.RAY_DTYPE)
        _check(lib.b200pt_debug_camera_rays(self.h, px, py, n, abi.ptr(out)))
        return out

    def debug_pixel_samples(self, px, py):
        out = np.zeros((self.setup.sampler.samples_per_pixel, 3), np.float32)
        _check(lib.b200pt_debug_pixel_samples(self.h, px, py, abi.ptr(out)))
        return out

    def set_option(self, name, value):
        _check(lib.b200pt_render_set_option(self.h, name.encode(), int(value)))

    def stats(self):
        s = abi.Stats()
        _check(lib.b200pt_get_stats(self.h, C.byref(s)))
        return {k: getattr(s, k) for k, _ in abi.Stats._fields_}

    def reset_stats(self):
        _check(lib.b200pt_reset_stats(self.h))

    def close(self):
        if self.h:
            lib.b200pt_render_destroy(self.h)
            self.h = _vp()
