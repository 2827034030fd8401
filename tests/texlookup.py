"""Shared by tests/test_texlookup.py (host-compiled half) and tests/test_zz_texlookup_gpu.py (device): the texture and sky
functions of pt_texture.cuh and ComputeDifferentials, run by the devmath harness (tests/devmath/devmath.cu) and compared
bit for bit with the reference's own MIPMap, InfiniteAreaLight, SurfaceInteraction and TrowbridgeReitzDistribution,
called by oracle/_ref/ref_probe.  The input sets: structured edges of every branch, then stratified random points.

ref_probe exists only where the reference sources were built.  Elsewhere the tables the reference built (MIPMap pyramids
and weightLut, InfiniteAreaLight's Lmap level 0, Distribution2D tables and matrices) come from tests/golden/
texlookup_tables.npz, which `python tests/texlookup.py` regenerates and tests/test_texlookup.py checks against ref_probe,
and the expected answers are the host-compiled build's, which tests/test_texlookup.py pins to the reference's."""
import ctypes as C
import hashlib
import os
import struct
import subprocess

import numpy as np

from conftest import ROOT

PROBE = os.path.join(ROOT, "oracle", "_ref", "ref_probe")
GOLDEN = os.path.join(ROOT, "tests", "golden", "texlookup_tables.npz")
EWA, WIDTH, SAMPLE, PDF, LE, DIFF, ROUGH = range(7)
IN_WORDS = {EWA: 6, WIDTH: 3, SAMPLE: 2, PDF: 3, LE: 3, DIFF: 24, ROUGH: 1}
OUT_WORDS = {EWA: 3, WIDTH: 3, SAMPLE: 10, PDF: 1, LE: 3, DIFF: 4, ROUGH: 1}
ON_HOST, ON_DEVICE = 0, 1
REPEAT, BLACK, CLAMP = 0, 1, 2  # ImageWrap, B200PT_WRAP_*
MAX_LEVELS = 16
EWA_MAX_TEXELS = 4096  # the harness refuses larger EWA footprints (devmath.cu)
F32 = np.float32


class Report(C.Structure):
    _fields_ = [("checked", C.c_uint64), ("mismatches", C.c_uint64), ("n_first", C.c_int32), ("pad", C.c_int32),
                ("input", C.c_uint64 * 16), ("got", C.c_uint64 * 16), ("want", C.c_uint64 * 16)]

    def describe(self, words=1):
        rows = ["query %d word %d: got 0x%08x, expected 0x%08x" % (self.input[i] // words, self.input[i] % words,
                                                                 self.got[i], self.want[i]) for i in range(self.n_first)]
        return "%d of %d words differ; first: %s" % (self.mismatches, self.checked, "; ".join(rows))


class MipDesc(C.Structure):  # dm_mipmap
    _fields_ = [("channels", C.c_int32), ("levels", C.c_int32), ("wrap", C.c_int32), ("trilinear", C.c_int32),
                ("max_aniso", C.c_float), ("w", C.c_int32 * MAX_LEVELS), ("h", C.c_int32 * MAX_LEVELS),
                ("texels", C.c_void_p), ("weight_lut", C.c_float * 128)]


class SkyDesc(C.Structure):  # dm_sky
    _fields_ = [("w", C.c_int32), ("h", C.c_int32), ("nu", C.c_int32), ("nv", C.c_int32), ("texels", C.c_void_p),
                ("cond_func", C.c_void_p), ("cond_cdf", C.c_void_p), ("cond_func_int", C.c_void_p),
                ("marg_func", C.c_void_p), ("marg_cdf", C.c_void_p), ("marg_func_int", C.c_float),
                ("light_to_world", C.c_float * 16), ("world_to_light", C.c_float * 16), ("two_world_radius", C.c_float),
                ("ref_p", C.c_float * 3)]


def bind(path):
    lib = C.CDLL(path)
    vp, u64, rp = C.c_void_p, C.c_uint64, C.POINTER(Report)
    lib.dm_mip_footprint.argtypes = [C.POINTER(MipDesc), vp, u64, vp]
    lib.dm_check_mip.argtypes = [C.POINTER(MipDesc), C.c_int, vp, u64, vp, C.c_int, rp, vp]
    lib.dm_check_sky.argtypes = [C.POINTER(SkyDesc), C.c_int, vp, u64, vp, C.c_int, rp, vp]
    lib.dm_check_geom.argtypes = [C.c_int, vp, u64, vp, C.c_int, rp, vp]
    return lib


def f32(x):
    return np.asarray(x, dtype=F32)


def nxt(x, toward):
    return F32(np.nextafter(F32(x), F32(toward)))


def run_probe(args, tmp):
    r = subprocess.run([PROBE] + [str(a) for a in args], capture_output=True, cwd=tmp)
    assert r.returncode == 0, r.stderr.decode()[-2000:]
    return r.stdout


def ptr(a):
    return a.ctypes.data


def have_probe():
    return os.path.exists(PROBE)


_golden = {}


def golden(key):
    if not _golden:
        with np.load(GOLDEN) as z:
            _golden.update({k: z[k] for k in z.files})
    return _golden[key]


def mip_key(texels, wrap):
    return hashlib.sha1(np.ascontiguousarray(texels, F32).tobytes() + str(texels.shape + (wrap,)).encode()).hexdigest()[:20]


# ---------------------------------------------------------------------------------------------------- MIPMap
class Mip:
    """A MIPMap the reference built (pyramid, weightLut) and its answers to the queries given."""

    def __init__(self, tmp, texels, wrap, trilinear, max_aniso, ewa_q, width_q, tag="m"):
        texels = np.ascontiguousarray(texels, F32)
        h, w = texels.shape[:2]
        ch = 1 if texels.ndim == 2 else texels.shape[2]
        ewa_q = np.ascontiguousarray(ewa_q, F32).reshape(-1, 6)
        width_q = np.ascontiguousarray(width_q, F32).reshape(-1, 3)
        self.ewa_q, self.width_q, self.ch = ewa_q, width_q, ch
        if not have_probe():  # the reference's pyramid as committed; the answers come from the host-compiled build
            key = mip_key(texels, wrap)
            dims, levels = golden("mipdims/" + key), golden("mip/" + key)
            lv = lambda h: texels.ravel() if h == "input" else golden("lvl/" + h)  # a power-of-two map's level 0: its texels
            self.pyramid = np.ascontiguousarray(np.concatenate([lv(h) for h in levels]))
            self._desc(dims, golden("lut"), wrap, trilinear, max_aniso)
            self.ewa = self.width = None
            return
        req, out = os.path.join(tmp, tag + ".req"), os.path.join(tmp, tag + ".out")
        with open(req, "wb") as f:
            f.write(np.array([ch, w, h, wrap, int(trilinear), len(ewa_q), len(width_q), 0], np.int32).tobytes())
            f.write(f32([max_aniso]).tobytes() + texels.tobytes() + ewa_q.tobytes() + width_q.tobytes())
        run_probe(["mipmap", req, out], tmp)
        b = open(out, "rb").read()
        levels = struct.unpack_from("<i", b, 0)[0]
        dims = np.frombuffer(b, np.int32, 2 * levels, 4).reshape(levels, 2)
        at = 4 + 8 * levels
        n = int((dims[:, 0].astype(np.int64) * dims[:, 1]).sum()) * ch
        self.pyramid = np.frombuffer(b, F32, n, at).copy()
        at += 4 * n
        lut = np.frombuffer(b, F32, 128, at)
        at += 512
        self.ewa = np.frombuffer(b, F32, len(ewa_q) * ch, at).reshape(-1, ch)
        at += 4 * self.ewa.size
        self.width = np.frombuffer(b, F32, len(width_q) * ch, at).reshape(-1, ch)
        self.lut = lut.copy()
        self._desc(dims, lut, wrap, trilinear, max_aniso)

    def _desc(self, dims, lut, wrap, trilinear, max_aniso):
        self.dims = np.asarray(dims, np.int32)
        d = MipDesc()
        d.channels, d.levels, d.wrap, d.trilinear, d.max_aniso = self.ch, len(dims), wrap, int(trilinear), max_aniso
        for i in range(len(dims)):
            d.w[i], d.h[i] = int(dims[i][0]), int(dims[i][1])
        d.texels = ptr(self.pyramid)
        d.weight_lut[:] = [float(v) for v in lut]
        self.desc = d

    def want(self, fam, dm=None):
        """The reference's answers (3 words per query), or the host-compiled build's where ref_probe is not built."""
        a = self.ewa if fam == EWA else self.width
        if a is None:
            q = self.ewa_q if fam == EWA else self.width_q
            out = np.zeros(3 * len(q), np.uint32)
            assert dm.dm_check_mip(C.byref(self.desc), fam, ptr(q), len(q), ptr(out), ON_HOST, C.byref(Report()),
                                   ptr(out)) == 0
            return out
        return np.ascontiguousarray(np.repeat(a, 3 // a.shape[1], axis=1)).view(np.uint32)

    def check(self, dm, fam, where, rep, want=None, got=None):
        q = self.ewa_q if fam == EWA else self.width_q
        want = self.want(fam, dm) if want is None else want
        return dm.dm_check_mip(C.byref(self.desc), fam, ptr(q), len(q), ptr(want), where, C.byref(rep),
                               None if got is None else ptr(got))


def pyramid_dims(w, h):
    """The levels MIPMap's constructor makes: resolution rounded up to powers of two, halved down to 1 x 1."""
    up = lambda v: 1 << (v - 1).bit_length()
    w, h = up(w), up(h)
    levels = 1 + max(w, h).bit_length() - 1
    return [(max(1, w >> i), max(1, h >> i)) for i in range(levels)]


def footprints(dm, w, h, max_aniso, q):
    """Texels each EWA query scans, from the harness's own bound (the texel values do not enter it)."""
    dims = pyramid_dims(w, h)
    d = MipDesc()
    d.channels, d.levels, d.max_aniso = 1, len(dims), max_aniso
    for i, (a, b) in enumerate(dims):
        d.w[i], d.h[i] = a, b
    zeros = np.zeros(sum(a * b for a, b in dims), F32)
    d.texels = ptr(zeros)
    q = np.ascontiguousarray(q, F32)
    out = np.zeros(len(q), np.uint64)
    assert dm.dm_mip_footprint(C.byref(d), ptr(q), len(q), ptr(out)) == 0
    return out


def mip_texels(w, h, ch, seed, huge=False):
    """Texels in [-0.2, 1.6) with a black block (huge: values near 1e37, whose EWA sums overflow)."""
    rng = np.random.default_rng(seed)
    shape = (h, w) if ch == 1 else (h, w, ch)
    if huge:
        return (rng.uniform(0.5, 3.0, shape) * 1e37).astype(F32)
    t = rng.uniform(-0.2, 1.6, shape).astype(F32)
    t[h // 4:(h + 1) // 2, w // 4:(w + 1) // 2] = 0
    return t


def st_edges(w, h):
    """s (or t) values: +-0, 1 and 1 - ulp, [-3, 4) landmarks, texel centres and edges of the first and last texels and
    near-2^30 / size (|st * size| < 2^30)."""
    one_m = float(nxt(1, 0))
    big = float(F32((2 ** 30 - 2 ** 7) / max(pyramid_dims(w, h)[0])))
    vals = [0.0, -0.0, 1.0, one_m, -1.0, -3.0, 3.999, 0.5, 2.0 ** -149, -2.0 ** -24, big, -big, 1.0 + 2 ** -23]
    for n in pyramid_dims(w, h)[0]:
        for k in (0, 1, n - 1, n, -1):
            vals += [(k + 0.5) / n, k / n, float(nxt(k / n, -1)), float(nxt((k + 0.5) / n, 2))]
    a = np.unique(f32(vals).view(np.uint32))  # by bits: +0 and -0 both stay
    return a.view(F32).tolist()


def dst_edges(levels, max_aniso):
    """(dst0, dst1) pairs at the lookup's branch edges."""
    out = []
    a = max_aniso
    out += [(0, 0, 0, 0), (0.01, 0.02, 0, 0), (0, 0, 0.01, -0.02), (-0.0, 0.0, 0.0, -0.0)]  # both / one zero
    for k in (2.0 ** -10, 2.0 ** -4, 0.1, 0.5):  # equal lengths: the swap's tie
        out += [(k, 0, 0, k), (0, k, k, 0), (0.6 * k, 0.8 * k, -0.8 * k, 0.6 * k), (3 * k / 5, 4 * k / 5, 4 * k / 5, 3 * k / 5)]
    for e in range(0, 31, 3):  # major / minor at maxAnisotropy and +-1 ulp from it
        m = F32(2.0 ** -e)
        M = F32(m * a)
        for MM in (M, nxt(M, 0), nxt(M, np.inf)):
            out += [(MM, 0, 0, m), (0, m, MM, 0), (MM * 0.6, MM * 0.8, -m * 0.8, m * 0.6)]
    for L in range(-31, 3):  # minor lengths 2^-30 .. 2: lod < 0, on a level, exactly Levels() - 1 (minor 1) and above
        for frac in (1.0, 1.5, float(nxt(1, 0)), float(nxt(1, 2))):
            m = F32(frac * 2.0 ** L)
            out += [(m, 0, 0, m), (2 * m, 0, 0, m), (0, m, m * min(a, 4.0), 0)]
    for e in range(levels + 1):  # lod exactly on every level
        m = F32(2.0 ** (e - (levels - 1)))
        out += [(m, 0, 0, m), (m * 0.6, m * 0.8, m * 0.8, -m * 0.6)]
    for c in (1.0, -1.0, 0.5, 3.0):  # collinear pairs
        out += [(0.01, 0.02, 0.01 * c, 0.02 * c), (0.3, -0.1, 0.3 * c, -0.1 * c)]
    return f32(out)


def random_ewa(n, seed):
    """Stratified s, t in [-3, 4); minor length log-uniform in [2^-30, 2], eccentricity in [1, 128), random rotation and
    order."""
    rng = np.random.default_rng(seed)
    s = (np.arange(n) + rng.uniform(0, 1, n)) / n * 7 - 3
    t = rng.permutation((np.arange(n) + rng.uniform(0, 1, n)) / n * 7 - 3)
    minor = 2.0 ** rng.uniform(-30, 1, n)
    major = minor * 2.0 ** rng.uniform(0, 7, n)
    th = rng.uniform(0, 2 * np.pi, n)
    d0 = np.stack([major * np.cos(th), major * np.sin(th)], 1)
    d1 = np.stack([-minor * np.sin(th), minor * np.cos(th)], 1)
    sw = rng.uniform(0, 1, n) < 0.5
    d0[sw], d1[sw] = d1[sw].copy(), d0[sw].copy()
    return f32(np.concatenate([s[:, None], t[:, None], d0, d1], 1))


def ewa_queries(dm, w, h, max_aniso, n_random, seed):
    """Structured st x dst edges, then random queries; those whose footprint the harness would refuse are dropped (the
    structured ones are small by construction, so only random ones with a long major axis at lod 0 go)."""
    levels = len(pyramid_dims(w, h))
    st = st_edges(w, h)
    d = dst_edges(levels, max_aniso)
    rng = np.random.default_rng(seed + 1)
    rows = []
    for i, s in enumerate(st):
        for j, t in enumerate(st[::3]):
            rows.append([s, t] + list(d[(i * 7 + j) % len(d)]))
    mid = [[0.3, 0.7], [0.5, 0.5], [float(F32(0.5 / w)), float(F32(0.5 / h))], [-2.25, 3.5]]
    for dd in d:
        for s, t in mid:
            rows.append([s, t] + list(dd))
    q = np.concatenate([f32(rows), random_ewa(n_random, seed)])
    fp = footprints(dm, w, h, max_aniso, q)
    keep = fp <= EWA_MAX_TEXELS
    assert keep[:len(rows)].mean() > 0.95, "structured EWA queries should fit the footprint bound"
    return q[keep]


def width_queries(w, h, n_random, seed):
    """Widths 0, negative, the 1e-8 floor and +-1 ulp, both level cut-offs (2^-(Levels() - 1) and 1) +-1 ulp, every level,
    then random log-uniform widths, over st edges and random st."""
    levels = len(pyramid_dims(w, h))
    ws = [0.0, -1.0, 1e-8, nxt(1e-8, 0), nxt(1e-8, 1), 1.0, nxt(1, 0), nxt(1, 2), 4.0]
    c = 2.0 ** -(levels - 1)
    ws += [c, nxt(c, 0), nxt(c, 1)] + [2.0 ** (e - (levels - 1)) * f for e in range(levels) for f in (1, 1.25)]
    st = st_edges(w, h)
    rows = [[s, t, wd] for i, s in enumerate(st) for t in st[i % 3::5] for wd in ws[i % 4::4]]
    rows += [[s, 0.375, wd] for s in st[::2] for wd in ws]
    rng = np.random.default_rng(seed)
    s = (np.arange(n_random) + rng.uniform(0, 1, n_random)) / n_random * 7 - 3
    t = rng.uniform(-3, 4, n_random)
    wd = 2.0 ** rng.uniform(-32, 2, n_random)
    return np.concatenate([f32(rows), f32(np.stack([s, t, wd], 1))])


MIP_MAPS = [(1, 1), (1, 16), (16, 1), (2, 2), (8, 4), (64, 64), (256, 64), (24, 10), (3, 5), (1000, 1)]
MIP_HUGE = (8, 8)  # values near 1e37
# maxanisotropy below 1 scales the minor axis up even when the two are equally long: the only setting where the swap
# of equally long differentials shows
MIP_FILTERS = [("ewa", 1.0), ("ewa", 8.0), ("ewa", 64.0), ("ewa", 0.5), ("trilinear", 8.0)]


def mip_cases():
    out = []
    for (w, h) in MIP_MAPS + [MIP_HUGE]:
        for ch in (3, 1):
            out.append((w, h, ch, (w, h) == MIP_HUGE))
    return out


def run_mip_case(dm, tmp, w, h, ch, huge, where, n_random, n_width):
    """Every wrap x filter for one map and channel count: n_random random EWA queries per wrap and filter, n_width random
    Lookup(st, width) queries per wrap.  Returns [(name, fam, report)] and the query count."""
    tex = mip_texels(w, h, ch, seed=w * 131 + h * 7 + ch, huge=huge)
    res, nq = [], 0
    wq = width_queries(w, h, n_width, seed=w + h)
    for wrap in (REPEAT, BLACK, CLAMP):
        for k, (filt, aniso) in enumerate(MIP_FILTERS):
            tri = filt == "trilinear"
            eq = ewa_queries(dm, w, h, aniso, n_random, seed=1000 * wrap + 10 * k + w)
            m = Mip(tmp, tex, wrap, tri, aniso, eq, wq if k == 0 else np.zeros((0, 3), F32))
            name = "%dx%d ch%d wrap%d %s aniso%g" % (w, h, ch, wrap, filt, aniso)
            for fam in ((EWA, WIDTH) if k == 0 else (EWA,)):
                rep = Report()
                rc = m.check(dm, fam, where, rep)
                assert rc == 0, "%s: harness returned %d" % (name, rc)
                res.append(("%s %s" % (name, "width" if fam == WIDTH else "lookup"), fam, rep))
                nq += len(m.ewa_q if fam == EWA else m.width_q)
    return res, nq


# ---------------------------------------------------------------------------------------------------- sky
def write_pfm(path, rgb):
    """rgb [h][w][3]; PFM stores the bottom row first."""
    h, w = rgb.shape[:2]
    with open(path, "wb") as f:
        f.write(b"PF\n%d %d\n-1\n" % (w, h))
        f.write(np.ascontiguousarray(rgb[::-1], "<f4").tobytes())


def sky_map(name):
    rng = np.random.default_rng(len(name))
    if name == "constant":
        return f32([[[0.7, 1.3, 2.1]]])
    if name == "8x4":
        return rng.uniform(0, 3, (4, 8, 3)).astype(F32)
    if name in ("24x10", "24x10-dist"):  # resampled to 32 x 16
        return rng.uniform(0, 3, (10, 24, 3)).astype(F32)
    if name == "top-black":
        m = rng.uniform(0.1, 2, (8, 16, 3)).astype(F32)
        m[:4] = 0
        return m
    if name == "hot-texel":
        m = np.zeros((8, 16, 3), F32)
        m[5, 11] = (4000, 2500, 900)
        return m
    if name == "black":
        return np.zeros((4, 8, 3), F32)
    raise KeyError(name)


def sky_distribution(name):
    """The image whose Distribution2D replaces the light's own, or an empty one (keep the light's).  Every map's
    distribution is 2 x its power-of-two resolution, where (offset + du) / n equals (offset + du) * (1 / n); "24x10-dist"
    samples a 24 x 10 map through a 23 x 11 distribution with a black row and column."""
    if name != "24x10-dist":
        return np.zeros((0, 0), F32)
    img = np.random.default_rng(9).uniform(0, 2, (11, 23)).astype(F32)
    img[4] = 0
    img[:, 7] = 0
    return img


SKY_MAPS = ["constant", "8x4", "24x10", "24x10-dist", "top-black", "hot-texel", "black"]


def rotation(axis, deg):
    a = np.asarray(axis, float)
    a /= np.linalg.norm(a)
    c, s = np.cos(np.radians(deg)), np.sin(np.radians(deg))
    x, y, z = a
    return np.array([[c + x * x * (1 - c), x * y * (1 - c) - z * s, x * z * (1 - c) + y * s],
                     [y * x * (1 - c) + z * s, c + y * y * (1 - c), y * z * (1 - c) - x * s],
                     [z * x * (1 - c) - y * s, z * y * (1 - c) + x * s, c + z * z * (1 - c)]])


def sky_xform(name):
    m = np.eye(4)
    if name == "oblique":
        m[:3, :3] = rotation((1, 2, 3), 37)
    elif name == "mirror-scale":
        m[:3, :3] = np.diag([-1.0, 2.0, 0.5]) @ rotation((0.2, -1, 0.4), 71)
        m[:3, 3] = (3, -1, 0.5)
    return f32(m)


SKY_XFORMS = ["identity", "oblique", "mirror-scale"]
REF_P = (0.25, -1.5, 2.0)
WORLD_RADIUS = 13.375


class Sky:
    """An InfiniteAreaLight the reference built (level 0 of Lmap, Distribution2D tables, matrices) and its answers."""

    def __init__(self, tmp, mapname, xform, u=(), w=(), d=(), tag="s"):
        u, w, d = (np.ascontiguousarray(np.reshape(f32(a), (-1, k))) for a, k in ((u, 2), (w, 3), (d, 3)))
        self.u, self.w, self.d = u, w, d
        if not have_probe():  # the reference's tables as committed; the answers come from the host-compiled build
            g = lambda f: np.ascontiguousarray(golden("sky/%s/%s" % (mapname, f)))
            W, H, nu, nv = (int(v) for v in g("dims"))
            self.texels, self.cond_func, self.cond_cdf, self.cond_func_int = g("texels"), g("cond_func"), g("cond_cdf"), g("cond_func_int")
            self.marg_func, self.marg_cdf, self.marg_func_int = g("marg_func"), g("marg_cdf"), g("marg_func_int")[0]
            self.l2w, self.w2l = golden("xform/%s/l2w" % xform), golden("xform/%s/w2l" % xform)
            self.sample = self.pdf = self.le = None
            self._desc(W, H, nu, nv)
            return
        pfm = os.path.join(tmp, "sky_%s.pfm" % mapname)
        if not os.path.exists(pfm):
            write_pfm(pfm, sky_map(mapname))
        dist = sky_distribution(mapname)
        req, out = os.path.join(tmp, tag + ".req"), os.path.join(tmp, tag + ".out")
        with open(req, "wb") as f:
            nv, nu = dist.shape
            f.write(np.array([len(u), len(w), len(d), nu, nv, 0], np.int32).tobytes())
            f.write(sky_xform(xform).tobytes() + f32([WORLD_RADIUS]).tobytes() + f32(REF_P).tobytes() + dist.tobytes())
            f.write(u.tobytes() + w.tobytes() + d.tobytes())
        run_probe(["infinite", pfm, req, out], tmp)
        b = open(out, "rb").read()
        W, H, nu, nv = struct.unpack_from("<4i", b, 0)
        at = 16

        def take(n):
            nonlocal at
            a = np.frombuffer(b, F32, n, at).copy()
            at += 4 * n
            return a
        self.texels = take(W * H * 3)
        self.cond_func, self.cond_cdf, self.cond_func_int = take(nu * nv), take((nu + 1) * nv), take(nv)
        self.marg_func, self.marg_cdf = take(nv), take(nv + 1)
        self.marg_func_int = take(1)[0]
        self.l2w, self.w2l = take(16), take(16)
        self.sample, self.pdf, self.le = take(len(u) * 10).view(np.uint32), take(len(w)).view(np.uint32), take(len(d) * 3).view(np.uint32)
        assert at == len(b)
        self._desc(W, H, nu, nv)

    def _desc(self, W, H, nu, nv):
        self.nu, self.nv = nu, nv
        s = SkyDesc()
        s.w, s.h, s.nu, s.nv = W, H, nu, nv
        s.texels, s.cond_func, s.cond_cdf = ptr(self.texels), ptr(self.cond_func), ptr(self.cond_cdf)
        s.cond_func_int, s.marg_func, s.marg_cdf = ptr(self.cond_func_int), ptr(self.marg_func), ptr(self.marg_cdf)
        s.marg_func_int = float(self.marg_func_int)
        s.light_to_world[:] = self.l2w.tolist()
        s.world_to_light[:] = self.w2l.tolist()
        s.two_world_radius = float(F32(2) * F32(WORLD_RADIUS))
        s.ref_p[:] = list(REF_P)
        self.desc = s

    def answers(self, fam, dm=None):
        """The reference's answers, or the host-compiled build's where ref_probe is not built."""
        q, a = {SAMPLE: (self.u, self.sample), PDF: (self.w, self.pdf), LE: (self.d, self.le)}[fam]
        if a is None:
            a = np.zeros(OUT_WORDS[fam] * len(q), np.uint32)
            assert dm.dm_check_sky(C.byref(self.desc), fam, ptr(q), len(q), ptr(a), ON_HOST, C.byref(Report()), ptr(a)) == 0
        return a

    def check(self, dm, fam, where, rep, want=None, got=None):
        q = {SAMPLE: self.u, PDF: self.w, LE: self.d}[fam]
        want = self.answers(fam, dm) if want is None else want
        return dm.dm_check_sky(C.byref(self.desc), fam, ptr(q), len(q), ptr(want), where, C.byref(rep),
                               None if got is None else ptr(got))

    def cdf_us(self):
        """Every u equal to a CDF entry and 1 ulp below it: the marginal's against u0 = 0.5, every row's with a u1 inside
        that row's marginal interval (rows no u1 reaches included: u1 = their cdf entry)."""
        out = []
        for c in self.marg_cdf:
            for cc in (c, nxt(c, 0)):
                out += [(0.5, cc), (0.0, cc), (float(nxt(1, 0)), cc)]
        cdf = self.cond_cdf.reshape(self.nv, self.nu + 1)
        for v in range(self.nv):
            lo, hi = self.marg_cdf[v], self.marg_cdf[v + 1]
            u1 = float(F32(0.5 * (lo + hi))) if hi > lo else float(lo)
            for c in cdf[v]:
                for cc in (c, nxt(c, 0)):
                    out.append((cc, u1))
        return f32(out)


def axis():
    from test_zz_devmath_gpu import axis as devmath_axis
    return devmath_axis()


def grid(ax_u, ax_v):
    return f32(np.stack([np.tile(ax_u, len(ax_v)), np.repeat(ax_v, len(ax_u))], 1))


def sky_dirs(n_random, seed):
    """Random directions, the poles and 1 ulp off them, (x < 0, +-0, z) on atan2's seam, unnormalised ones (w.z > 1)."""
    rng = np.random.default_rng(seed)
    v = rng.normal(size=(n_random, 3))
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    scale = 2.0 ** rng.uniform(-10, 10, (n_random, 1))
    v[n_random // 2:] *= scale[n_random // 2:]
    e = []
    one_m = float(nxt(1, 0))
    for z in (1.0, -1.0):
        e += [(0, 0, z), (-0.0, 0, z), (0, -0.0, z), (2.0 ** -24, 0, z * one_m), (0, 2.0 ** -12, z), (-2.0 ** -12, -0.0, z),
              (2.0 ** -149, 0, z), (0, 0, z * one_m), (0, 0, z * float(nxt(1, 2)))]
    for z in (0.9, 0.3, 0.0, -0.0, -0.5, -0.99):
        for y in (0.0, -0.0, 2.0 ** -149, -2.0 ** -149):
            e += [(-1.0, y, z), (-0.25, y, z), (1.0, y, z)]
    e += [(0, 0, 2), (0.3, 0.2, 5), (0, 0, -7), (1e-3, 2e-3, 1.5), (3, -4, 12), (1e4, 1e4, -1e4), (1e-20, -1e-20, 1e-20)]
    return np.concatenate([f32(e), f32(v)])


def sky_runs(dm, tmp, mapname, xform, where, grid_u, n_dirs, chunk=1 << 21):
    """Sample_Li at the CDF entries and the grid (in chunks), Pdf_Li and Le at sky_dirs and at every wi returned."""
    base = Sky(tmp, mapname, xform)
    res = []

    def one(u, d):
        sky = Sky(tmp, mapname, xform, u=u, w=d, d=d)
        for fam in (SAMPLE, PDF, LE) if len(d) else (SAMPLE,):
            rep = Report()
            assert sky.check(dm, fam, where, rep) == 0
            res.append(("%s %s %s" % (mapname, xform, {SAMPLE: "Sample_Li", PDF: "Pdf_Li", LE: "Le"}[fam]), fam, rep))
        if len(u):  # the returned directions, fed back in
            wi = np.ascontiguousarray(sky.answers(SAMPLE, dm).view(F32).reshape(-1, 10)[:, :3])
            ray_d = wi[np.any(wi != 0, axis=1)]  # a sample of pdf 0 leaves wi (0, 0, 0), no ray direction
            fb = Sky(tmp, mapname, xform, w=wi, d=ray_d)
            for fam in (PDF, LE) if len(ray_d) else (PDF,):
                rep = Report()
                assert fb.check(dm, fam, where, rep) == 0
                res.append(("%s %s %s(wi)" % (mapname, xform, "Pdf_Li" if fam == PDF else "Le"), fam, rep))
            return sky
    one(base.cdf_us(), sky_dirs(n_dirs, seed=len(mapname)))
    for s in range(0, len(grid_u), chunk):
        one(grid_u[s:s + chunk], np.zeros((0, 3), F32))
    return res


# ---------------------------------------------------------------------------------------------------- differentials
def diff_cases(n_random, seed):
    """{p, n, dpdu, dpdv, rxOrigin, rxDirection, ryOrigin, ryDirection}: normals on the dominant-axis ties, axis-aligned
    and with -0 components; determinants at 1e-10 +-1 ulp; rays parallel to the plane (tx inf) and zero directions from
    the plane (tx NaN); p near 10^4; then random frames and rays."""
    rng = np.random.default_rng(seed)
    rows = []
    a, b = 0.6, 0.5291502622129182  # 2 a^2 + b^2 = 1
    normals = [(a, a, b), (a, -a, b), (-a, a, -b), (b, a, a), (b, -a, a), (a, b, a), (-a, b, -a), (0.57735, 0.57735, 0.57735),
               (1, 0, 0), (0, 1, 0), (0, 0, 1), (-1, 0, 0), (0, -1, 0), (0, 0, -1), (-0.0, 0, 1), (1, -0.0, -0.0),
               (0, -0.0, -1), (-0.0, 1, -0.0), (0.6, 0.8, 0), (0, 0.6, -0.8), (0.8, 0, 0.6)]
    for n in normals:
        for k in range(6):
            p = rng.uniform(-2, 2, 3)
            dpdu, dpdv = rng.uniform(-1, 1, 3), rng.uniform(-1, 1, 3)
            o = p + np.asarray(n) * rng.uniform(0.5, 3) + rng.uniform(-0.5, 0.5, 3)
            dx, dy = p - o + rng.uniform(-0.05, 0.05, 3), p - o + rng.uniform(-0.05, 0.05, 3)
            rows.append(np.concatenate([p, n, dpdu, dpdv, o, dx, o + rng.uniform(-0.01, 0.01, 3), dy]))
    # determinants at 1e-10 +-1 ulp (and -1e-10): n = z, so dims (x, y); det = A00 * A11 exactly
    t = F32(1e-10)
    for det in (t, nxt(t, 0), nxt(t, 1), -t, nxt(-t, 0), F32(0)):
        for a11 in (1.0, -1.0, 0.5):
            for n in ((0, 0, 1), (0, 1, 0), (1, 0, 0)):
                ax = int(np.argmax(np.abs(n)))
                d0, d1 = [i for i in range(3) if i != ax]
                dpdu, dpdv = np.zeros(3), np.zeros(3)
                dpdu[d0], dpdv[d1] = float(det) / a11, a11  # exact: det = A00 * A11
                dpdu[ax], dpdv[ax] = 0.25, -0.5
                p = np.array([0.3, -0.2, 0.1])
                o = p + 2 * np.asarray(n, float)
                rows.append(np.concatenate([p, n, dpdu, dpdv, o + (0.01, 0.02, 0), p - o + (0.003, -0.001, 0.002),
                                            o + (-0.02, 0.01, 0.005), p - o + (-0.002, 0.004, 0.001)]))
    # parallel rays (tx inf), zero directions from the plane (tx NaN), from off the plane (tx inf)
    p, n = np.array([0.5, 0.25, 1.0]), np.array([0.0, 0.0, 1.0])
    dpdu, dpdv = np.array([1.0, 0.2, 0]), np.array([-0.1, 1.0, 0])
    good_o, good_d = np.array([0.4, 0.3, 3.0]), np.array([0.1, -0.05, -2.0])
    for bad_o, bad_d in (((0.1, 0.2, 2.0), (1.0, 0.5, 0.0)), ((0.1, 0.2, 1.0), (0.0, 0.0, 0.0)), ((0.1, 0.2, 2.0), (0, 0, 0)),
                         ((0.1, 0.2, 1.0), (1.0, -1.0, 0.0)), ((0.1, 0.2, 2.0), (0.0, 0.0, -0.0))):
        rows.append(np.concatenate([p, n, dpdu, dpdv, bad_o, bad_d, good_o, good_d]))
        rows.append(np.concatenate([p, n, dpdu, dpdv, good_o, good_d, bad_o, bad_d]))
    # p near 10^4: cancellation in px - p
    for k in range(64):
        p = 1e4 + rng.uniform(-3, 3, 3)
        n = rng.normal(size=3)
        n /= np.linalg.norm(n)
        o = p + n * rng.uniform(1, 50) + rng.uniform(-1, 1, 3)
        rows.append(np.concatenate([p, n, rng.uniform(-1, 1, 3), rng.uniform(-1, 1, 3), o, p - o + rng.uniform(-1e-3, 1e-3, 3),
                                    o + rng.uniform(-1e-3, 1e-3, 3), p - o + rng.uniform(-1e-3, 1e-3, 3)]))
    # random: frames, normals, ray differentials around the hit; every fourth with p near 10^4
    n = n_random
    p = rng.uniform(-10, 10, (n, 3))
    p[::4] += 1e4
    nn = rng.normal(size=(n, 3))
    nn /= np.linalg.norm(nn, axis=1, keepdims=True)
    o = p + nn * rng.uniform(0.1, 20, (n, 1)) + rng.uniform(-2, 2, (n, 3))
    dx = p - o + rng.uniform(-0.1, 0.1, (n, 3))
    dy = p - o + rng.uniform(-0.1, 0.1, (n, 3))
    ox = o + rng.uniform(-0.01, 0.01, (n, 3))
    oy = o + rng.uniform(-0.01, 0.01, (n, 3))
    rnd = np.concatenate([p, nn, rng.uniform(-2, 2, (n, 3)), rng.uniform(-2, 2, (n, 3)), ox, dx, oy, dy], 1)
    return np.ascontiguousarray(np.concatenate([f32(rows), f32(rnd)]))


def probe_diff(tmp, q, dm=None):
    """ComputeDifferentials' answers: the reference's, or the host-compiled build's where ref_probe is not built."""
    if not have_probe():
        out = np.zeros(4 * len(q), np.uint32)
        assert check_geom(dm, DIFF, q, out, ON_HOST, Report(), out) == 0
        return out
    req, out = os.path.join(tmp, "diff.req"), os.path.join(tmp, "diff.out")
    q.tofile(req)
    run_probe(["differentials", req, out], tmp)
    return np.fromfile(out, np.uint32)


def check_geom(dm, fam, q, want, where, rep, got=None):
    q = np.ascontiguousarray(q, F32)
    return dm.dm_check_geom(fam, ptr(q), len(q) // IN_WORDS[fam] if q.ndim == 1 else len(q), ptr(want), where,
                            C.byref(rep), None if got is None else ptr(got))


# ---------------------------------------------------------------------------------------------------- roughness
def bits_of(x):
    return int(np.array([x], F32).view(np.uint32)[0])


def roughness_ranges(full):
    """[lo, hi) bit ranges: every float in [2^-10, 2) (full) or a strided sample of it; 0, subnormals, -0 and negatives,
    large values, inf and NaN."""
    lo, hi = bits_of(2.0 ** -10), bits_of(2.0)
    main = [(lo, hi)] if full else [(s, s + 4096) for s in range(lo, hi, (hi - lo) // 64)]
    edges = [(0, 1 << 14), (0x00800000 - 4096, 0x00800000 + 4096), (0x80000000, 0x80000000 + (1 << 14)),
             (bits_of(-1.0) - 4096, bits_of(-1.0) + 4096), (bits_of(1e-3) - 4096, bits_of(1e-3) + 4096),
             (bits_of(2.0), bits_of(2.0) + 4096), (0x7f7ff000, 0x7f800002), (0x7fc00000, 0x7fc00002),
             (0xff800000, 0xff800002), (0xffc00000, 0xffc00001)]
    return main + edges


def roughness_chunks(ranges, chunk=1 << 24, dm=None):
    """(inputs, reference answers) in chunks, the answers streamed from the probe (where it is not built: the
    host-compiled build's)."""
    if not have_probe():
        for lo, hi in ranges:
            for s in range(lo, hi, chunk):
                x = np.arange(s, min(hi, s + chunk), dtype=np.uint64).astype(np.uint32).view(F32)
                want = np.zeros(len(x), np.uint32)
                assert check_geom(dm, ROUGH, x, want, ON_HOST, Report(), want) == 0
                yield x, want
        return
    for lo, hi in ranges:
        p = subprocess.Popen([PROBE, "roughness", str(lo), str(hi)], stdout=subprocess.PIPE)
        for s in range(lo, hi, chunk):
            m = min(chunk, hi - s)
            want = np.frombuffer(p.stdout.read(4 * m), np.uint32)
            assert len(want) == m
            yield np.arange(s, s + m, dtype=np.uint64).astype(np.uint32).view(F32), want
        assert p.stdout.read() == b"" and p.wait() == 0


# ---------------------------------------------------------------------------------------------------- golden tables
def build_golden(tmp):
    """The tables the reference builds for every MIPMap (per map, channel count and wrap) and sky of the input sets, as
    arrays: MIPMap levels stored once per distinct content, none for a level 0 equal to the map's texels."""
    assert have_probe(), "regenerating the tables needs %s" % PROBE
    out = {}
    none6, none3 = np.zeros((0, 6), F32), np.zeros((0, 3), F32)
    for (w, h, ch, huge) in mip_cases():
        tex = mip_texels(w, h, ch, seed=w * 131 + h * 7 + ch, huge=huge)
        for wrap in (REPEAT, BLACK, CLAMP):
            m = Mip(tmp, tex, wrap, False, 8.0, none6, none3)
            key, at, names = mip_key(tex, wrap), 0, []
            for lw, lh in m.dims:
                lv = m.pyramid[at:at + lw * lh * ch]
                at += lw * lh * ch
                if np.array_equal(lv.view(np.uint32), tex.ravel().view(np.uint32)):
                    name = "input"
                else:
                    name = hashlib.sha1(lv.tobytes() + str((int(lw), int(lh), ch)).encode()).hexdigest()[:20]
                    out["lvl/" + name] = lv
                names.append(name)
            out["mip/" + key], out["mipdims/" + key], out["lut"] = np.array(names), m.dims, m.lut
    for name in SKY_MAPS:
        for x in SKY_XFORMS:
            s = Sky(tmp, name, x)
            out["xform/%s/l2w" % x], out["xform/%s/w2l" % x] = s.l2w, s.w2l
        out["sky/%s/dims" % name] = np.array([s.desc.w, s.desc.h, s.nu, s.nv], np.int32)
        for f in ("texels", "cond_func", "cond_cdf", "cond_func_int", "marg_func", "marg_cdf"):
            out["sky/%s/%s" % (name, f)] = getattr(s, f)
        out["sky/%s/marg_func_int" % name] = f32([s.marg_func_int])
    return out


if __name__ == "__main__":  # regenerates tests/golden/texlookup_tables.npz with oracle/_ref/ref_probe
    import sys
    import tempfile
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    with tempfile.TemporaryDirectory() as d:
        np.savez_compressed(GOLDEN, **build_golden(d))
    print(GOLDEN, os.path.getsize(GOLDEN))
