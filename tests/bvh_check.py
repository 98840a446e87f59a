"""Independent float64 checker of a BVH8 built by the library (or by the host emulation in tests/emu).

It reads the node and record arrays as embree_b200/csrc/rt_core.cuh:31-57 documents them (DESIGN section 3) and recomputes
everything it compares against from the scene's input buffers, with its own float64 arithmetic.  It calls no decode or
bounds routine of the library or the emulator.

Node8 (96 bytes, 24 words):  w0..w2 grid origin p (fp32), w3 = ex | ey << 8 | ez << 16 | imask << 24, w4 child_base,
w5 tri_base, bytes 24..47 the 24-bit leaf mask of slot s at byte 24 + 3 s, bytes 48..95 the planes qlo_x[8] qlo_y[8]
qlo_z[8] qhi_x[8] qhi_y[8] qhi_z[8].  A plane q of axis a decodes to p_a + q * 2^(e_a - 127).

Validity rules (a primitive that fails them is in no leaf), restated from the reference:
  triangles  kernels/common/scene_triangle_mesh.h:194-215 (indices in range, every coordinate inside +-FLT_LARGE)
  quads      kernels/common/scene_quad_mesh.h:186-203 (all four vertices)
  lines      kernels/common/scene_line_segments.h:427-441 (both vertices, radii >= 0)
  cubics     kernels/common/scene_curves.h:498-533, 661-691 (control points, tangents, and the box itself: isvalid(b))
  points     kernels/common/scene_points.h:146-199 (centre and radius, radius >= 0)
FLT_LARGE is common/math/constants.h:21.

`check_bvh` raises BVHCheckError naming the violated invariant and the node / slot / record.
"""
from fractions import Fraction

import numpy as np

FLT_LARGE = np.float32(1.844e18)
MAX_LEAF = 3          # rt_core.cuh kMaxLeafTris
STACK = 64            # rt_core.cuh kStackSize
INVALID = 0xFFFFFFFF
TRIANGLE, ROUND_LINEAR, FLAT_LINEAR, FLAT_CUBIC, ROUND_CUBIC, SPHERE, DISC, ORIENTED_DISC = range(8)
CUBIC_MARGIN = 1e-6   # cubic boxes: primref_gen's relative margins (1.2e-6 / 2.4e-7 + 4 ulp) cover the fp32 curve evaluation


class BVHCheckError(AssertionError):
    pass


def strided(buf, offset, stride, count, ncomp, dtype=np.float32):
    """`count` items of `ncomp` values of `dtype` at byte `offset` + i * `stride` of the byte buffer `buf`."""
    b = np.frombuffer(np.ascontiguousarray(buf).view(np.uint8).tobytes(), np.uint8)
    isz = np.dtype(dtype).itemsize
    rows = offset + stride * np.arange(count)[:, None] + isz * np.arange(ncomp)[None, :]
    take = b[(rows[..., None] + np.arange(isz)).reshape(-1)]
    return take.view(dtype).reshape(count, ncomp)


class Geom:
    """One geometry as the scene saw it (buffers already read through their strides / offsets).

    verts: float32 [nverts, 3] (triangles, quads) or [nverts, 4] (curves, points: xyz + radius); idx: uint32 [n, 3] / [n, 4] /
    [n] (first vertex of each curve); xfm: 12 floats of an instance's local-to-world columns, or None."""

    def __init__(self, kind, geomID, verts, idx=None, mask=0xFFFFFFFF, quad=False, basis=0, tess=4, tangents=None, normals=None,
                 flags=None, xfm=None, instID=INVALID):
        self.kind, self.geomID, self.mask, self.quad = kind, geomID, mask & 0xFFFFFFFF, quad
        self.verts = np.asarray(verts, np.float32)
        self.idx = None if idx is None else np.asarray(idx, np.uint32)
        self.basis, self.tess, self.tangents, self.normals, self.flags = basis, tess, tangents, normals, flags
        self.hermite = tangents is not None and kind in (FLAT_CUBIC, ROUND_CUBIC)
        self.xfm = None if xfm is None else np.asarray(xfm, np.float32).reshape(12)
        self.instID = instID

    def nprims(self):
        if self.kind >= SPHERE:
            return len(self.verts)
        n = len(self.idx)
        return {TRIANGLE: 2 * n if self.quad else n, FLAT_CUBIC: n * self.tess, ROUND_CUBIC: 7 * n}.get(self.kind, n)


def _inside(x):
    """(x > -FLT_LARGE) & (x < FLT_LARGE) on fp32 values, all along the last axis (NaN fails)"""
    x = np.asarray(x, np.float32)
    return ((x > -FLT_LARGE) & (x < FLT_LARGE)).all(axis=-1)


def _xfm64(g, p):
    """float64 local-to-world transform of points p[..., 3].  Each product of two fp32 values is exact in float64; the sum of four
    is rounded once or twice, 1e-16 relative, far below the 1e-6 relative widening primref_gen gives instanced boxes."""
    m = g.xfm.astype(np.float64)
    p = p.astype(np.float64)
    return p[..., 0:1] * m[0:3] + p[..., 1:2] * m[3:6] + p[..., 2:3] * m[6:9] + m[9:12]


def _basis(basis, u):
    """position and derivative weights [..., 4] of the cubic basis at u (float64 polynomials)"""
    u = np.asarray(u, np.float64)
    s = 1.0 - u
    if basis == 0:
        c = [s ** 3, 3 * u * s * s, 3 * u * u * s, u ** 3]
        d = [-3 * s * s, 3 * s * s - 6 * u * s, 6 * u * s - 3 * u * u, 3 * u * u]
    elif basis == 1:
        c = [s ** 3 / 6, (3 * u ** 3 - 6 * u * u + 4) / 6, (-3 * u ** 3 + 3 * u * u + 3 * u + 1) / 6, u ** 3 / 6]
        d = [-s * s / 2, 1.5 * u * u - 2 * u, -1.5 * u * u + u + 0.5, u * u / 2]
    else:
        c = [(-u ** 3 + 2 * u * u - u) / 2, (3 * u ** 3 - 5 * u * u + 2) / 2, (-3 * u ** 3 + 4 * u * u + u) / 2, (u ** 3 - u * u) / 2]
        d = [(-3 * u * u + 4 * u - 1) / 2, (9 * u * u - 10 * u) / 2, (-9 * u * u + 8 * u + 1) / 2, (3 * u * u - 2 * u) / 2]
    return np.stack(c, -1), np.stack(d, -1)


class Prims:
    """The BVH primitives of one geometry: validity, exact world extent, allowed slack, expected record words."""

    def __init__(self, n):
        self.valid = np.zeros(n, bool)
        self.maybe = np.zeros(n, bool)          # validity undecidable from the exact box (cubic box within 1e-5 of FLT_LARGE)
        self.lo = np.full((n, 3), np.inf)
        self.hi = np.full((n, 3), -np.inf)
        self.slack = np.zeros((n, 3))
        self.rec = np.zeros((n, 12), np.uint32)   # word 7 (geomID or descriptor index) is filled in by the checker


def _f32bits(x):
    return np.asarray(x, np.float32).view(np.uint32)


def primitives(g, robust):
    n = g.nprims()
    P = Prims(n)
    V = g.verts
    nv = len(V)
    if n == 0:
        return P
    if g.kind == TRIANGLE:
        if g.quad:
            q = g.idx.reshape(-1, 4)
            okq = (q < nv).all(1)
            qs = np.where(q < nv, q, 0)
            vq = V[qs]                                                    # [Q, 4, 3]
            okq &= _inside(vq.reshape(len(q), 12))
            tri = np.empty((2 * len(q), 3), np.int64)
            tri[0::2] = qs[:, [0, 1, 3]]
            tri[1::2] = qs[:, [2, 1, 3]]
            ok = np.repeat(okq, 2)
            lp = np.arange(2 * len(q), dtype=np.uint32)
            prim_word = (lp >> 1) | ((lp & 1) << 31)
        else:
            t = g.idx.reshape(-1, 3)
            ok = (t < nv).all(1)
            tri = np.where(t < nv, t, 0).astype(np.int64)
            ok &= _inside(V[tri].reshape(len(t), 9))
            prim_word = np.arange(len(t), dtype=np.uint32)
        v = V[tri]                                                        # [P, 3, 3] object space
        w = v.astype(np.float64) if g.xfm is None else _xfm64(g, v)
        if g.xfm is not None:
            ok &= np.isfinite(w).all((1, 2)) & (np.abs(w) < float(FLT_LARGE)).all((1, 2))
        P.valid = ok
        P.lo, P.hi = w.min(1), w.max(1)
        e1 = v[:, 1] if robust else v[:, 0] - v[:, 1]                    # fp32 subtraction, rounded to nearest as leaf_pack does
        e2 = v[:, 2] if robust else v[:, 2] - v[:, 0]
        P.rec[:, 0:3] = _f32bits(v[:, 0])
        P.rec[:, 3] = prim_word
        P.rec[:, 4:7] = _f32bits(e1)
        P.rec[:, 8:11] = _f32bits(e2)
        P.rec[:, 11] = g.mask
    elif g.kind in (ROUND_LINEAR, FLAT_LINEAR):
        vid = g.idx.reshape(-1).astype(np.int64)
        ok = vid + 1 < nv
        a = V[np.where(ok, vid, 0)]
        b = V[np.where(ok, vid + 1, 0)]
        ok &= _inside(np.concatenate([a, b], 1)) & (np.minimum(a[:, 3], b[:, 3]) >= 0)
        r = np.maximum(a[:, 3], b[:, 3]).astype(np.float64)[:, None]
        P.valid = ok
        P.lo = np.minimum(a[:, :3], b[:, :3]).astype(np.float64) - r
        P.hi = np.maximum(a[:, :3], b[:, :3]).astype(np.float64) + r
        if g.flags is not None:
            fl = np.asarray(g.flags, np.uint32) & 3
        else:   # derived from the index buffer as the library (and scene_line_segments.cpp:209-232) does
            right = np.zeros(len(vid), bool)
            right[:-1] = vid[1:] == vid[:-1] + 1
            left = np.zeros(len(vid), bool)
            left[1:] = right[:-1]
            fl = left.astype(np.uint32) | (right.astype(np.uint32) << 1)
        P.rec[:, 0:3] = _f32bits(a[:, :3])
        P.rec[:, 3] = np.arange(n, dtype=np.uint32)
        P.rec[:, 4:7] = _f32bits(b[:, :3])
        P.rec[:, 8] = _f32bits(a[:, 3])
        P.rec[:, 9] = _f32bits(b[:, 3])
        P.rec[:, 10] = (vid.astype(np.uint32) & 0x3FFFFFFF) | (fl << 30)
        P.rec[:, 11] = g.mask
    elif g.kind >= SPHERE:
        c = V
        ok = _inside(c) & (c[:, 3] >= 0)
        r = c[:, 3].astype(np.float64)[:, None]
        P.valid = ok
        P.lo, P.hi = c[:, :3].astype(np.float64) - r, c[:, :3].astype(np.float64) + r
        P.rec[:, 0:3] = _f32bits(c[:, :3])
        P.rec[:, 3] = np.arange(n, dtype=np.uint32)
        if g.kind == ORIENTED_DISC:
            P.rec[:, 4:7] = _f32bits(np.asarray(g.normals, np.float32).reshape(-1, 3))
        P.rec[:, 8] = _f32bits(c[:, 3])
        P.rec[:, 11] = g.mask
    else:
        _cubic_prims(g, P)
    if g.xfm is not None and g.kind != TRIANGLE:      # instanced curves / points: the 8 transformed corners of the object box
        lo, hi = P.lo, P.hi
        corners = np.stack([np.stack([(hi if (c & 4) else lo)[:, 0], (hi if (c & 2) else lo)[:, 1], (hi if (c & 1) else lo)[:, 2]], -1)
                            for c in range(8)], 1)
        wc = _xfm64(g, corners)
        fin = np.isfinite(lo).all(1) & np.isfinite(hi).all(1)
        P.lo = np.where(fin[:, None], wc.min(1), np.inf)
        P.hi = np.where(fin[:, None], wc.max(1), -np.inf)
        P.slack = np.abs(P.slack) @ np.abs(g.xfm[:9].astype(np.float64).reshape(3, 3))
        inside = np.isfinite(P.lo).all(1) & (np.abs(P.lo) < float(FLT_LARGE)).all(1) & (np.abs(P.hi) < float(FLT_LARGE)).all(1)
        if g.kind in (FLAT_CUBIC, ROUND_CUBIC):
            P.maybe |= P.valid & _near_limit(P.lo, P.hi)
        P.valid &= inside
    gone = ~P.valid & ~P.maybe          # an invalid primitive has no extent
    P.lo[gone], P.hi[gone] = np.inf, -np.inf
    return P


def _near_limit(lo, hi):
    m = np.maximum(np.abs(lo), np.abs(hi)).max(1)
    return (m > float(FLT_LARGE) * (1 - 1e-5)) & (m < float(FLT_LARGE) * (1 + 1e-5))


def _cubic_prims(g, P):
    V = g.verts
    nv = len(V)
    vid = g.idx.reshape(-1).astype(np.int64)
    ncurve = len(vid)
    ok = vid + (1 if g.hermite else 3) < nv
    base = np.where(ok, vid, 0)
    if g.hermite:
        T = np.asarray(g.tangents, np.float32).reshape(-1, 4)
        p0, p1, t0, t1 = V[base], V[base + 1], T[base], T[base + 1]
        ok &= _inside(np.concatenate([p0, p1, t0, t1], 1))
        p0, p1, t0, t1 = (x.astype(np.float64) for x in (p0, p1, t0, t1))
        cp = np.stack([p0, p0 + t0 / 3, p1 - t1 / 3, p1], 1)          # Hermite -> Bezier (hermite_curve.h:19-20)
        basis = 0
    else:
        cp32 = np.stack([V[base + k] for k in range(4)], 1)
        ok &= _inside(cp32.reshape(ncurve, 16))
        cp = cp32.astype(np.float64)
        basis = g.basis
    mag = np.abs(cp[:, :, :3]).max((1, 2))                            # largest control-point coordinate of each curve
    per = 7 if g.kind == ROUND_CUBIC else g.tess
    lo = np.empty((ncurve, per, 3))
    hi = np.empty((ncurve, per, 3))
    if g.kind == FLAT_CUBIC:
        u = np.arange(per + 1) / per
        c, _ = _basis(basis, u)                                       # [N+1, 4]
        pts = np.einsum("jk,ckd->cjd", c, cp)                         # [C, N+1, 4]
        rmax = np.abs(pts[:, :, 3]).max(1)
        for s in range(per):
            a, b = pts[:, s, :3], pts[:, s + 1, :3]
            lo[:, s] = np.minimum(a, b) - rmax[:, None]
            hi[:, s] = np.maximum(a, b) + rmax[:, None]
        pad = CUBIC_MARGIN * (mag + rmax)
    else:
        pad = np.zeros(ncurve)
        for s in range(per):
            a, b = s / 7.0, (s + 1) / 7.0
            ca, da = _basis(basis, a)
            cb, db = _basis(basis, b)
            Pa, dPa = ca @ cp, da @ cp                                # [C, 4]
            Pb, dPb = cb @ cp, db @ cp
            hull = np.stack([Pa, Pa + dPa / 21.0, Pb - dPb / 21.0, Pb], 1)   # Bezier control points of the sub-segment (de Casteljau)
            r = np.abs(hull[:, :, 3]).max(1)
            lo[:, s] = hull[:, :, :3].min(1) - r[:, None]
            hi[:, s] = hull[:, :, :3].max(1) + r[:, None]
            # the swept spheres of the sub-segment lie inside the hull +- its largest radius (convex hull property)
            cu, _ = _basis(basis, np.linspace(a, b, 17))
            samp = np.einsum("jk,ckd->cjd", cu, cp)
            rs = np.abs(samp[:, :, 3])
            tol = 1e-12 * (mag + r)[:, None]
            assert ((samp[:, :, :3] - rs[..., None] >= lo[:, s][:, None] - tol[..., None]) |
                    ~ok[:, None, None]).all(), "checker: swept sphere outside its sub-segment hull"
            pad = np.maximum(pad, CUBIC_MARGIN * (mag + r))
    P.lo = lo.reshape(-1, 3)
    P.hi = hi.reshape(-1, 3)
    P.slack = np.repeat(pad, per)[:, None] * np.ones(3)
    okp = np.repeat(ok, per)
    fin = np.isfinite(P.lo).all(1) & np.isfinite(P.hi).all(1)
    inside = fin & (np.abs(P.lo) < float(FLT_LARGE)).all(1) & (np.abs(P.hi) < float(FLT_LARGE)).all(1)
    P.maybe = okp & fin & _near_limit(P.lo, P.hi)
    P.valid = okp & inside
    curve = np.repeat(np.arange(ncurve, dtype=np.uint32), per)
    seg = np.tile(np.arange(per, dtype=np.uint32), ncurve)
    P.rec[:, 3] = curve
    P.rec[:, 8] = seg
    P.rec[:, 10] = np.repeat(vid.astype(np.uint32), per)
    P.rec[:, 11] = g.mask


# ---------------------------------------------------------------------------------------------------------------------------
# node decoding
# ---------------------------------------------------------------------------------------------------------------------------
class Nodes:
    def __init__(self, words):
        w = np.ascontiguousarray(words, np.uint32).reshape(-1, 24)
        self.w = w
        self.n = len(w)
        self.p = w[:, 0:3].view(np.float32).astype(np.float64)               # [N, 3]
        self.e = np.stack([(w[:, 3] >> (8 * a)) & 0xFF for a in range(3)], 1).astype(np.int64)
        self.imask = (w[:, 3] >> 24).astype(np.int64)
        self.child_base = w[:, 4].astype(np.int64)
        self.tri_base = w[:, 5].astype(np.int64)
        b = w.view(np.uint8).reshape(-1, 96)
        mb = b[:, 24:48].reshape(-1, 8, 3).astype(np.int64)
        self.leaf = mb[:, :, 0] | (mb[:, :, 1] << 8) | (mb[:, :, 2] << 16)     # [N, 8]
        q = b[:, 48:96].reshape(-1, 6, 8).astype(np.int64)
        self.qlo = q[:, 0:3].transpose(0, 2, 1)                               # [N, 8, 3]
        self.qhi = q[:, 3:6].transpose(0, 2, 1)
        self.inner = ((self.imask[:, None] >> np.arange(8)) & 1).astype(bool)  # [N, 8]
        self.scale = np.ldexp(1.0, self.e - 127)                               # [N, 3], exact powers of two

    def plane(self, q):
        """exact decoded planes p + q * 2^(e-127) for q[N, 8, 3]: float64 values and a mask of the entries float64 cannot hold"""
        a = self.p[:, None, :]
        b = q * self.scale[:, None, :]
        s = a + b
        bb = s - a
        err = (a - (s - bb)) + (b - bb)          # TwoSum: exact rounding error of a + b
        return s, err != 0


def exact_plane(p, q, e):
    return Fraction(float(p)) + q * Fraction(2) ** (int(e) - 127)


def _round_f32(x, up):
    """fp32 rounding of the exact value x (Fraction) towards +inf (up) or -inf"""
    f = np.float32(float(x))
    inf = np.float32(np.inf) if up else np.float32(-np.inf)
    if not np.isfinite(f):
        return f
    while (Fraction(float(f)) < x) if up else (Fraction(float(f)) > x):
        f = np.nextafter(f, inf)
    other = np.nextafter(f, -inf)
    while np.isfinite(other) and ((Fraction(float(other)) >= x) if up else (Fraction(float(other)) <= x)):
        f, other = other, np.nextafter(other, -inf)
    return f


def _round_f32_vec(x, inexact, up, p, q, e):
    """directed fp32 rounding of the float64 values x (exact where ~inexact)"""
    with np.errstate(over="ignore", invalid="ignore"):     # planes beyond the fp32 range round to +-inf
        f = x.astype(np.float32)
        if up:
            f = np.where(f.astype(np.float64) < x, np.nextafter(f, np.float32(np.inf)), f)
        else:
            f = np.where(f.astype(np.float64) > x, np.nextafter(f, np.float32(-np.inf)), f)
    for idx in zip(*np.nonzero(inexact)):
        f[idx] = _round_f32(exact_plane(p[idx], q[idx], e[idx]), up)
    return f


# ---------------------------------------------------------------------------------------------------------------------------
# the checker
# ---------------------------------------------------------------------------------------------------------------------------
def _fail(msg):
    raise BVHCheckError(msg)


def check_bvh(arr, geoms, robust=False, tight=None, refit=False, scene_bounds=None):
    """Checks the scene `arr` (the dict of RTCLib.scene_arrays, or the same keys from the emulator) against the geometries
    `geoms` (list of Geom; an instanced geometry appears once per instance with its xfm and instID).

    tight: also check the tightness invariants (default: scenes of plain or quad triangles without instances).
    refit: the arrays come from a refit (a node with an empty slot is exempt from tightness, as refit_level documents).
    scene_bounds: six floats from rtcGetSceneBounds, compared with the union of the valid primitives.
    Returns a report dict."""
    N = Nodes(arr["nodes"])
    rec = np.ascontiguousarray(arr["records"], np.uint32).reshape(-1, 12)
    R = len(rec)
    general = bool(arr.get("general", 0))
    two_level = arr.get("builder", 0) == 3
    if tight is None:
        tight = all(g.kind == TRIANGLE and g.xfm is None for g in geoms)

    # ---- descriptors / geometry lookup
    prims = [primitives(g, robust) for g in geoms]
    if general:
        descs = arr["descs"]
        expect = [i for i, g in enumerate(geoms) if g.nprims() > 0]
        if len(descs) != len(expect):
            _fail(f"descriptors: {len(descs)} descriptors for {len(expect)} non-empty geometries")
        first = 0
        for d, gi in zip(descs, expect):
            g = geoms[gi]
            want = dict(geomID=g.geomID, instID=g.instID, kind=g.kind, first=first, count=g.nprims(), is_quad=int(g.quad))
            for k, v in want.items():
                if int(d[k]) != v:
                    _fail(f"descriptor of geometry {g.geomID} (instance {g.instID}): {k} = {int(d[k])}, expected {v}")
            if g.kind in (FLAT_CUBIC, ROUND_CUBIC) and (int(d["basis"]) != (0 if g.hermite else g.basis) or int(d["hermite"]) != int(g.hermite)):
                _fail(f"descriptor of geometry {g.geomID}: basis {int(d['basis'])} / hermite {int(d['hermite'])}")
            if g.kind == FLAT_CUBIC and int(d["tess"]) != g.tess:
                _fail(f"descriptor of geometry {g.geomID}: tess {int(d['tess'])}, expected {g.tess}")
            if g.xfm is not None and not np.array_equal(d["xfm"].view(np.uint32), g.xfm.view(np.uint32)):
                _fail(f"descriptor of geometry {g.geomID} (instance {g.instID}): transform differs")
            first += g.nprims()
        desc_geom = np.array(expect, np.int64)
    else:
        by_id = {g.geomID: i for i, g in enumerate(geoms)}
        if len(by_id) != len(geoms) or any(g.xfm is not None or g.quad or g.kind != TRIANGLE for g in geoms):
            _fail("scene without descriptors must hold plain triangle meshes with distinct geomIDs")

    # ---- structure: reach every node from the root exactly once
    if N.n == 0:
        _fail("structure: no nodes")
    reached = np.zeros(N.n, np.int64)
    depth = np.full(N.n, -1, np.int64)
    parent = np.full(N.n, -1, np.int64)
    pslot = np.full(N.n, -1, np.int64)
    reached[0] = 1
    depth[0] = 0
    frontier = np.array([0])
    levels = [frontier]
    rank = np.bitwise_count(np.arange(256)[:, None] & ((1 << np.arange(8)) - 1))   # rank[imask, s]: internal slots before slot s
    while len(frontier):
        if len(levels) > STACK:
            _fail(f"structure: deeper than the traversal stack ({STACK} levels)")
        nd, sl = np.nonzero(N.inner[frontier])
        src = frontier[nd]
        child = N.child_base[src] + rank[N.imask[src], sl]
        bad = child >= N.n
        if bad.any():
            k = np.argmax(bad)
            _fail(f"structure: node {src[k]} slot {sl[k]}: child {child[k]} beyond the {N.n} nodes")
        np.add.at(reached, child, 1)
        twice = reached > 1
        if twice.any():
            k = int(np.argmax(twice))
            _fail(f"structure: node {k} reached {reached[k]} times (child_base of its parents overlap)")
        depth[child] = len(levels)
        parent[child] = src
        pslot[child] = sl
        frontier = child
        if len(frontier):
            levels.append(frontier)
    nlevels = len(levels)
    if nlevels >= STACK:
        _fail(f"structure: {nlevels} levels, the traversal stack holds {STACK}")
    unreached = np.nonzero(reached == 0)[0]
    if two_level:
        subs = np.asarray(arr["subs"], np.int64).reshape(-1, 4)
        allowed = set(range(int(arr["top_nodes"]))) | set(int(s[0]) for s in subs if s[2] > 0)
        stray = [int(u) for u in unreached if int(u) not in allowed]
        if stray:
            _fail(f"structure: node {stray[0]} is not reached from the root ({len(stray)} such nodes)")
        for i, (noff, toff, nn, nt) in enumerate(subs):
            if nn == 0:
                continue
            top = np.nonzero((reached == 1) & (np.arange(N.n) < int(arr["top_nodes"])) &
                                            (N.w == N.w[noff]).all(1))[0]
            if len(top) == 0:
                _fail(f"two-level: no copy of mesh {i}'s root node {noff} in the top level")
            rng = slice(noff, noff + nn)
            inner_used = N.imask[rng] != 0
            cb = N.child_base[rng][inner_used]
            if ((cb < noff) | (cb >= noff + nn)).any():
                _fail(f"two-level: mesh {i}: child_base not relocated into its nodes [{noff}, {noff + nn})")
            leaf_used = N.leaf[rng].any(1)
            tb = N.tri_base[rng][leaf_used]
            if ((tb < toff) | (tb >= toff + nt)).any():
                _fail(f"two-level: mesh {i}: tri_base not relocated into its records [{toff}, {toff + nt})")
    elif len(unreached):
        _fail(f"structure: node {unreached[0]} is not reached from the root ({len(unreached)} such nodes)")
    md = int(arr.get("max_depth", 0))
    if not two_level and md and md != nlevels:
        _fail(f"structure: reported max_depth {md}, the tree has {nlevels} levels")

    # ---- leaf masks
    live = np.nonzero(reached > 0)[0]
    leaf = N.leaf[live]
    inner = N.inner[live]
    pop = np.bitwise_count(leaf)
    if (pop > MAX_LEAF).any():
        k, s = np.argwhere(pop > MAX_LEAF)[0]
        _fail(f"leaf mask: node {live[k]} slot {s} holds {pop[k, s]} records (at most {MAX_LEAF})")
    if (inner & (leaf != 0)).any():
        k, s = np.argwhere(inner & (leaf != 0))[0]
        _fail(f"leaf mask: node {live[k]} slot {s} is internal and has a leaf mask")
    union = np.bitwise_or.reduce(leaf, axis=1)
    if (np.bitwise_count(union) != pop.sum(1)).any():
        k = int(np.argmax(np.bitwise_count(union) != pop.sum(1)))
        _fail(f"leaf mask: node {live[k]}: the leaf masks of its slots overlap")
    empty = ~inner & (leaf == 0)
    qany = (N.qlo[live] != 0).any(2) | (N.qhi[live] != 0).any(2)
    if (empty & qany).any():
        k, s = np.argwhere(empty & qany)[0]
        _fail(f"node {live[k]} slot {s}: empty slot with non-zero planes")
    kk, ss, bb = np.nonzero(((leaf[:, :, None] >> np.arange(24)) & 1).astype(bool))
    rid = N.tri_base[live][kk] + bb
    if (rid >= R).any():
        j = int(np.argmax(rid >= R))
        _fail(f"leaf mask: node {live[kk[j]]} slot {ss[j]} refers to record {rid[j]} of {R}")
    cnt = np.bincount(rid, minlength=R)
    if (cnt != 1).any():
        j = int(np.argmax(cnt != 1))
        _fail(f"leaf mask: record {j} is referenced by {cnt[j]} leaf slots")
    rec_node, rec_slot = np.empty(R, np.int64), np.empty(R, np.int64)
    rec_node[rid], rec_slot[rid] = live[kk], ss

    # ---- coverage and record contents
    if general:
        d = rec[:, 7].astype(np.int64)
        if (d >= len(desc_geom)).any():
            j = int(np.argmax(d >= len(desc_geom)))
            _fail(f"record {j}: descriptor {d[j]} of {len(desc_geom)}")
        gi = desc_geom[d]
    else:
        ids = rec[:, 7].astype(np.int64)
        lut = {gid: i for gid, i in by_id.items()}
        gi = np.array([lut.get(int(x), -1) for x in ids], np.int64) if R else np.zeros(0, np.int64)
        if (gi < 0).any():
            j = int(np.argmax(gi < 0))
            _fail(f"record {j}: geomID {ids[j]} is not in the scene")
    req_lo = np.full((R, 3), np.inf)
    req_hi = np.full((R, 3), -np.inf)
    vmin = np.full((R, 3), np.inf)
    vmax = np.full((R, 3), -np.inf)
    valid_lo, valid_hi = np.full(3, np.inf), np.full(3, -np.inf)
    for i, g in enumerate(geoms):
        P = prims[i]
        sel = np.nonzero(gi == i)[0]
        r = rec[sel]
        if g.kind == TRIANGLE and g.quad:
            loc = 2 * (r[:, 3] & 0x7FFFFFFF).astype(np.int64) + (r[:, 3] >> 31)
        elif g.kind in (FLAT_CUBIC, ROUND_CUBIC):
            per = 7 if g.kind == ROUND_CUBIC else g.tess
            loc = r[:, 3].astype(np.int64) * per + r[:, 8].astype(np.int64)
            if (r[:, 8] >= per).any():
                _fail(f"record {sel[np.argmax(r[:, 8] >= per)]}: segment {r[:, 8].max()} of {per}")
        else:
            loc = r[:, 3].astype(np.int64)
        if (loc >= len(P.valid)).any():
            j = int(np.argmax(loc >= len(P.valid)))
            _fail(f"record {sel[j]}: primitive {loc[j]} of geometry {g.geomID} does not exist")
        c = np.bincount(loc, minlength=len(P.valid))
        if (c > 1).any():
            _fail(f"coverage: primitive {int(np.argmax(c > 1))} of geometry {g.geomID} (instance {g.instID}) is in {c.max()} leaf records")
        missing = P.valid & ~P.maybe & (c == 0)
        if missing.any():
            _fail(f"coverage: valid primitive {int(np.argmax(missing))} of geometry {g.geomID} (instance {g.instID}) is in no leaf "
                  f"({int(missing.sum())} missing)")
        extra = ~P.valid & ~P.maybe & (c > 0)
        if extra.any():
            _fail(f"coverage: invalid primitive {int(np.argmax(extra))} of geometry {g.geomID} (instance {g.instID}) is in a leaf")
        want = P.rec[loc].copy()
        want[:, 7] = d[sel] if general else g.geomID
        diff = (want != r).any(1)
        if diff.any():
            j = int(np.argmax(diff))
            w = int(np.argmax(want[j] != r[j]))
            _fail(f"record contents: record {sel[j]} (geometry {g.geomID}, primitive {loc[j]}) word {w} is {r[j][w]:#010x}, "
                  f"expected {want[j][w]:#010x}")
        req_lo[sel] = P.lo[loc] + P.slack[loc]
        req_hi[sel] = P.hi[loc] - P.slack[loc]
        vmin[sel] = P.lo[loc]
        vmax[sel] = P.hi[loc]
        ok = P.valid & ~P.maybe
        if ok.any():
            valid_lo = np.minimum(valid_lo, P.lo[ok].min(0))
            valid_hi = np.maximum(valid_hi, P.hi[ok].max(0))

    # ---- subtree boxes, bottom-up: slot_lo/hi = union of the required boxes of the records below each slot
    slot_lo = np.full((N.n, 8, 3), np.inf)
    slot_hi = np.full((N.n, 8, 3), -np.inf)
    np.minimum.at(slot_lo, (rec_node, rec_slot), req_lo)
    np.maximum.at(slot_hi, (rec_node, rec_slot), req_hi)
    tight_lo = np.full((N.n, 8, 3), np.inf)
    tight_hi = np.full((N.n, 8, 3), -np.inf)
    np.minimum.at(tight_lo, (rec_node, rec_slot), vmin)
    np.maximum.at(tight_hi, (rec_node, rec_slot), vmax)
    for lv in reversed(levels[1:]):
        pa, ps = parent[lv], pslot[lv]
        slot_lo[pa, ps] = slot_lo[lv].min(1)
        slot_hi[pa, ps] = slot_hi[lv].max(1)
        tight_lo[pa, ps] = tight_lo[lv].min(1)
        tight_hi[pa, ps] = tight_hi[lv].max(1)

    # ---- containment: every slot box contains the exact extent of everything beneath it
    L = live
    dlo, xlo = N.plane(N.qlo)
    dhi, xhi = N.plane(N.qhi)
    used = (N.inner | (N.leaf != 0))[:, :, None] & np.ones(3, bool)
    for side, dec, inexact, need, cmp in (("low", dlo, xlo, slot_lo, np.less_equal), ("high", dhi, xhi, slot_hi, np.greater_equal)):
        bad = used & ~cmp(dec, need) & np.isfinite(need)
        bad[~np.isin(np.arange(N.n), L)] = False
        for k, s, a in np.argwhere(bad & inexact):     # float64 could not hold the plane: decide with exact rationals
            q = (N.qlo if side == "low" else N.qhi)[k, s, a]
            ex = exact_plane(N.p[k, a], q, N.e[k, a])
            if (ex <= Fraction(need[k, s, a])) if side == "low" else (ex >= Fraction(need[k, s, a])):
                bad[k, s, a] = False
        if bad.any():
            k, s, a = np.argwhere(bad)[0]
            _fail(f"containment: node {k} slot {s} axis {'xyz'[a]}: {side} plane {dec[k, s, a]!r} does not contain the primitives' "
                  f"{side} bound {need[k, s, a]!r}")
    # the node's grid reaches the top of its content: p + 255 * 2^(e-127) >= every child's high bound
    top = N.p + 255.0 * N.scale
    nhi = slot_hi.max(1)
    badt = (top < nhi) & np.isin(np.arange(N.n), L)[:, None]
    if badt.any():
        k, a = np.argwhere(badt)[0]
        _fail(f"containment: node {k} axis {'xyz'[a]}: grid top {top[k, a]!r} below its content {nhi[k, a]!r} (exponent {N.e[k, a]})")

    # ---- tightness (triangle scenes): origin = fp32 minimum of the subtree, planes the tightest encode_node_boxes allows
    if tight:
        nonempty = np.isfinite(tight_lo).all(2) & (N.inner | (N.leaf != 0))      # [N, 8]
        exempt = np.zeros(N.n, bool)
        if refit:
            exempt = ((N.inner | (N.leaf != 0)) & ~np.isfinite(tight_lo).all(2)).any(1)
        chk = np.isin(np.arange(N.n), L) & ~exempt
        nlo = tight_lo.min(1)
        orig = chk[:, None] & np.isfinite(nlo) & (N.p != nlo)
        if orig.any():
            k, a = np.argwhere(orig)[0]
            _fail(f"tightness: node {k} axis {'xyz'[a]}: grid origin {N.p[k, a]!r}, subtree minimum {nlo[k, a]!r}")
        m = (chk[:, None] & nonempty)[:, :, None] & np.ones(3, bool)
        e3 = np.broadcast_to(N.e[:, None, :], N.qlo.shape)
        p3 = np.broadcast_to(N.p[:, None, :], N.qlo.shape)
        ru = _round_f32_vec(dlo, xlo & m, True, p3, N.qlo, e3).astype(np.float64)
        nxt_q = np.minimum(N.qlo + 1, 255)
        dn, xn = N.plane(nxt_q)
        ru_next = _round_f32_vec(dn, xn & m & (N.qlo < 255), True, p3, nxt_q, e3).astype(np.float64)
        bad = m & ((ru > tight_lo) | ((N.qlo < 255) & (ru_next <= tight_lo)))
        if bad.any():
            k, s, a = np.argwhere(bad)[0]
            _fail(f"tightness: node {k} slot {s} axis {'xyz'[a]}: low plane q = {N.qlo[k, s, a]} is not the largest q with "
                  f"round_up(p + q s) <= {tight_lo[k, s, a]!r}")
        rd = _round_f32_vec(dhi, xhi & m, False, p3, N.qhi, e3).astype(np.float64)
        prv_q = np.maximum(N.qhi - 1, 0)
        dp_, xp_ = N.plane(prv_q)
        rd_prev = _round_f32_vec(dp_, xp_ & m & (N.qhi > 0), False, p3, prv_q, e3).astype(np.float64)
        bad = m & ((rd < tight_hi) | ((N.qhi > 0) & (rd_prev >= tight_hi)))
        if bad.any():
            k, s, a = np.argwhere(bad)[0]
            _fail(f"tightness: node {k} slot {s} axis {'xyz'[a]}: high plane q = {N.qhi[k, s, a]} is not the smallest q with "
                  f"round_down(p + q s) >= {tight_hi[k, s, a]!r}")

    # ---- scene bounds
    if scene_bounds is not None and tight:
        b = np.asarray(scene_bounds, np.float64)
        if np.isfinite(valid_lo).all():
            want = np.concatenate([valid_lo, valid_hi])
            if not np.array_equal(b, want):
                _fail(f"scene bounds: {b.tolist()}, the valid primitives span {want.tolist()}")
    root_lo, root_hi = N.p[0], N.p[0] + 255.0 * N.scale[0]
    return dict(nodes=N.n, records=R, levels=nlevels, valid_lo=valid_lo, valid_hi=valid_hi, root_exponent=N.e[0].tolist(),
                root_lo=root_lo, root_hi=root_hi, root_extent=root_hi - root_lo)
