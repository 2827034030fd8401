"""Per-ray comparison of the alpha masks with the reference's own Triangle::Intersect / IntersectP (oracle/_ref/alpha_probe:
CreateTriangleMesh + ImageTexture<Float, Float> + UVMapping2D inside a BVHAccel).  Quads facing +z carry masks with
every wrap, scale / delta, non-power-of-two maps (the reference resamples them; the library gets the reference's own
level 0), uvs and the GetUVs defaults, uv seams, shadowalpha unlike alpha and masked degenerate triangles.  Rays run
along +z: some at random, most aimed at texel centres and texel edges (where a bilinear weight is exactly 0 next to a
nonzero texel), each with its neighbouring floats."""
import ctypes as C
import os
import subprocess

import numpy as np

from conftest import ROOT

PROBE = os.path.join(ROOT, "oracle", "_ref", "alpha_probe")


def mask(seed, w, h):
    """Zero blocks of 3 x 3 texels (where a bilinear lookup is exactly 0 inside) and scattered single zeros (where it is
    0 only at the texel's centre, with the neighbours' weights exactly 0)."""
    rng = np.random.default_rng(seed)
    m = rng.uniform(0.05, 1.0, (h, w)).astype(np.float32)
    m[rng.uniform(size=(h, w)) < 0.2] = 0
    blocks = (rng.uniform(size=((h + 2) // 3, (w + 2) // 3)) < 0.5).repeat(3, 0).repeat(3, 1)[:h, :w]
    m[blocks] = 0
    return m


def quad(z, x0, y0, x1, y1, u0=0.0, v0=0.0, u1=1.0, v1=1.0):
    """Two triangles at depth z over [x0, x1] x [y0, y1]; uv linear in x, y from (u0, v0) to (u1, v1)."""
    p = np.array([[x0, y0, z], [x1, y0, z], [x1, y1, z], [x0, y1, z]], np.float32)
    t = np.array([[u0, v0], [u1, v0], [u1, v1], [u0, v1]], np.float32)
    return np.stack([p[[0, 1, 2]], p[[0, 2, 3]]]), np.stack([t[[0, 1, 2]], t[[0, 2, 3]]])


# groups: (quad args, uvs?, alpha spec, shadowalpha spec); spec None, 0 or (map, wrap, su, sv, du, dv)
GROUPS = [
    (dict(z=0.0, x0=-1, y0=-1, x1=1, y1=1), True, (mask(1, 12, 10), "repeat", 2.5, 1.5, 0.1, -0.2), None),
    (dict(z=1.0, x0=-1, y0=-1, x1=1, y1=1, u0=-0.3, u1=1.4), True, (mask(2, 8, 8), "clamp", 1.3, 1.0, 0.0, 0.05),
     (mask(3, 16, 4), "black", 1.0, 2.0, -0.1, 0.0)),
    # a uv seam: u runs across 1.0 (repeat) and the mask's edge columns differ
    (dict(z=2.0, x0=-1, y0=-1, x1=1, y1=1, u0=0.8, u1=1.2, v0=-0.5, v1=0.5), True, (mask(4, 16, 16), "repeat", 1.0, 1.0, 0.0, 0.0),
     (mask(5, 6, 6), "repeat", 3.0, 3.0, 0.0, 0.0)),
    # the GetUVs defaults (0,0) (1,0) (1,1), shadowalpha a constant 0
    (dict(z=3.0, x0=-1, y0=-1, x1=1, y1=1), False, (mask(6, 32, 16), "black", 1.0, 1.0, 0.0, 0.0), 0),
    (dict(z=4.0, x0=-1, y0=-1, x1=1, y1=1), True, None, None),  # a backstop without masks
]


def build(tmp):
    """(triangles [n][3][3], uvs [n][3][2], vertex flags, alpha ids, shadow ids, masks for add_alpha_mask, probe request)."""
    tris, uvs, flags, groups = [], [], [], []
    for g in GROUPS:
        p, t = quad(**g[0])
        groups.append((len(tris), len(p)))
        tris += list(p)
        uvs += list(t)
        flags += [2 if g[1] else 0] * len(p)
    # masked degenerate triangles (zero geometric normal) in front of everything, with and without uvs
    first_deg = len(tris)
    for k in range(4):
        x = -0.5 + 0.3 * k
        tris.append(np.array([[x, -1, -0.5], [x, 0, -0.5], [x, 1, -0.5]], np.float32))
        uvs.append(np.array([[0, 0], [0.5, 0.5], [1, 1]], np.float32))
        flags.append(2 if k % 2 else 0)
    tris, uvs = np.array(tris, np.float32), np.array(uvs, np.float32)
    n = len(tris)
    tris.tofile(os.path.join(tmp, "tris.f32"))
    uvs.tofile(os.path.join(tmp, "uvs.f32"))
    masks, alpha, shadow = [], np.full(n, -1, np.int32), np.full(n, -1, np.int32)
    lines = ["tris tris.f32", "uvs uvs.f32", "rays rays.bin"]

    def spec(s, ids, lo, cnt):
        if s is None:
            return "none - 0 0 0 0 0"
        ids[lo:lo + cnt] = len(masks)
        if isinstance(s, (int, float)):
            masks.append(dict(texels=None, wrap=0, su=1.0, sv=1.0, du=0.0, dv=0.0))
            return "zero - 0 0 0 0 0"
        m, wrap, su, sv, du, dv = s
        f = "mask%d.pfm" % len(masks)
        with open(os.path.join(tmp, f), "wb") as fh:  # the grey image as RGB: y() of equal channels
            fh.write(b"PF\n%d %d\n-1\n" % (m.shape[1], m.shape[0]))
            fh.write(np.ascontiguousarray(np.repeat(m[::-1, :, None], 3, axis=2), "<f4").tobytes())
        masks.append(dict(texels="level0", wrap={"repeat": 0, "black": 1, "clamp": 2}[wrap], su=su, sv=sv, du=du, dv=dv))
        return "map %s %s %.9g %.9g %.9g %.9g" % (f, wrap, su, sv, du, dv)

    for (lo, cnt), g in zip(groups, GROUPS):
        lines.append("group %d %d %s %s %s" % (lo, cnt, "uv" if g[1] else "nouv", spec(g[2], alpha, lo, cnt), spec(g[3], shadow, lo, cnt)))
    lines.append("group %d 2 nouv %s %s" % (first_deg, spec(GROUPS[0][2], alpha, first_deg, 2), spec(0, shadow, first_deg, 2)))
    lines.append("group %d 2 uv %s %s" % (first_deg + 2, spec(GROUPS[1][2], alpha, first_deg + 2, 2), spec(None, shadow, first_deg + 2, 2)))
    with open(os.path.join(tmp, "request.txt"), "w") as fh:
        fh.write("\n".join(lines) + "\n")
    return tris, uvs, np.array(flags, np.uint8), alpha, shadow, masks


def rays(abi, n_random=1000000):
    """Rays along +z: random ones, and ones at the x, y where a quad's st lands on texel centres and texel edges of its
    masks (the quads map x linearly to u), each with its two float neighbours in x and y."""
    rng = np.random.default_rng(9)
    xs, ys = [rng.uniform(-1, 1, n_random).astype(np.float32)], [rng.uniform(-1, 1, n_random).astype(np.float32)]
    for g in GROUPS:
        q = g[0]
        u0, u1, v0, v1 = q.get("u0", 0.0), q.get("u1", 1.0), q.get("v0", 0.0), q.get("v1", 1.0)
        for s in (g[2], g[3]):
            if not isinstance(s, tuple):
                continue
            m, _, su, sv, du, dv = s
            W, H = 1 << int(np.ceil(np.log2(m.shape[1]))), 1 << int(np.ceil(np.log2(m.shape[0])))
            # st * size - 0.5 integer: texel centres; + 0.5: the edge between two texels
            ks = np.arange(-2 * W, 2 * W + 1) / 2.0
            kt = np.arange(-2 * H, 2 * H + 1) / 2.0
            u = ((ks + 0.5) / W - du) / su
            v = ((kt + 0.5) / H - dv) / sv
            x = -1 + 2 * (u - u0) / (u1 - u0)
            y = -1 + 2 * (v - v0) / (v1 - v0)
            x, y = x[np.abs(x) < 1], y[np.abs(y) < 1]
            gx, gy = np.meshgrid(x.astype(np.float32), y.astype(np.float32))
            gx, gy = gx.ravel(), gy.ravel()
            for dx in (-1, 0, 1):
                for dy in (-1, 0, 1):
                    xs.append(gx + dx * np.spacing(gx))
                    ys.append(gy + dy * np.spacing(gy))
    x, y = np.concatenate(xs), np.concatenate(ys)
    # not along a quad's diagonal x == y: both triangles there give the same t, and which one the reference reports
    # follows its BVH's order, not the masks (DESIGN.md, ties)
    keep = np.abs(x - y) > 1e-4
    x, y = x[keep], y[keep]
    r = np.zeros(len(x), dtype=abi.RAY_DTYPE)
    r["o"][:, 0], r["o"][:, 1], r["o"][:, 2] = x, y, -2.0
    r["d"][:, 2] = 1.0
    r["d"][:, :2] = rng.normal(0, 1e-3, (len(x), 2)).astype(np.float32) * (rng.uniform(size=(len(x), 1)) < 0.3)
    r["t_max"] = np.where(rng.uniform(size=len(x)) < 0.2, np.float32(4.5), np.float32(np.inf))
    return r


def reference(tmp, r):
    r.tofile(os.path.join(tmp, "rays.bin"))
    p = subprocess.run([PROBE, "request.txt", "out.bin", "levels.bin"], cwd=tmp, capture_output=True, text=True)
    assert p.returncode == 0, p.stdout + p.stderr
    out = np.fromfile(os.path.join(tmp, "out.bin"), dtype=[("tri", "<i4"), ("t", "<f4"), ("occ", "<i4")])
    raw = open(os.path.join(tmp, "levels.bin"), "rb").read()
    levels, off = [], 0
    while off < len(raw):
        w, h = np.frombuffer(raw, np.int32, 2, off)
        levels.append(np.frombuffer(raw, np.float32, w * h, off + 8).reshape(h, w).copy())
        off += 8 + 4 * w * h
    return out, levels


def compare(pkg, abi, ctx, tmp):
    """Runs both sides; returns (reference answers, closest hits, occlusion, closest hits without masks)."""
    tris, uvs, flags, alpha, shadow, masks = build(tmp)
    r = rays(abi)
    ref, levels = reference(tmp, r)
    n = len(tris)
    mat = (abi.Material * 1)()
    mat[0].type = abi.MAT_MATTE
    keep = dict(tris=np.ascontiguousarray(tris), uvs=np.ascontiguousarray(uvs), flags=flags, mid=np.zeros(n, np.int32),
                lid=np.full(n, -1, np.int32), flip=np.zeros(n, np.uint8), mat=mat)
    d = abi.SceneDesc()
    d.n_triangles = n
    d.vertices, d.uvs, d.vertex_flags = abi.ptr(keep["tris"]), abi.ptr(keep["uvs"]), abi.ptr(flags)
    d.material_id, d.light_id, d.flip_normal = abi.ptr(keep["mid"]), abi.ptr(keep["lid"]), abi.ptr(keep["flip"])
    d.n_materials, d.materials = 1, C.cast(mat, C.POINTER(abi.Material))
    plain = pkg.Scene(ctx, d, keepalive=keep)
    scene = pkg.Scene(ctx, d, keepalive=keep)
    it = iter(levels)
    for m in masks:
        assert scene.add_alpha_mask(next(it) if m["texels"] is not None else None, m["wrap"], m["su"], m["sv"], m["du"], m["dv"]) >= 0
    scene.set_alpha_masks(alpha, shadow)
    hits, occ, bare = scene.trace_closest(r), scene.trace_any(r), plain.trace_closest(r)
    plain.close()
    scene.close()
    return ref, hits, occ, bare
