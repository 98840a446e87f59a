"""Curve primitives and rays at the corners of the curve intersectors' domain, for all ten curve kinds (the curve counterpart of
tests/parity.py point_edge_cases).

`curve_edge_cases(kind, seed)` returns the geometry in the formats OracleScene and the rtc.py helpers take and about 4 000 rays:
thin and fat strands, radii that vanish at one end or change faster than the centreline moves (the cone of a linear segment lies
inside its bigger end sphere), zero-length segments, straight, cusped and looping control polygons, radii larger than the radius of
curvature, Hermite curves with zero tangents, multi-segment strands with joints (library-derived and application neighbour flags),
strands 3 000 units from the origin and at a 1e-3 scale, tessellation rates 1, 4 and 16, invalid primitives and geometry masks.  Rays
start outside, on the centreline, inside the tube, on its surface (pointing in and out), graze the silhouette, run along the axis
through the end caps, pass through joints, and carry tnear / tfar windows that cut between the entry and the exit; |dir| spans
1e-3 to 1e3 and ray masks vary."""
import numpy as np

CURVE_KINDS = ["round_linear", "flat_linear"] + [f"{s}_{b}" for s in ("flat", "round") for b in ("bezier", "bspline", "catmull_rom", "hermite")]

# P(u) = [1, u, u^2, u^3] @ M @ control points (the power-basis form of each cubic basis; a Hermite curve is the Bezier curve
# p0, p0 + t0 / 3, p1 - t1 / 3, p1)
BASIS_MATRIX = {
    "bezier": np.array([[1, 0, 0, 0], [-3, 3, 0, 0], [3, -6, 3, 0], [-1, 3, -3, 1]], np.float64),
    "bspline": np.array([[1, 4, 1, 0], [-3, 0, 3, 0], [3, -6, 3, 0], [-1, 3, -3, 1]], np.float64) / 6.0,
    "catmull_rom": np.array([[0, 2, 0, 0], [-1, 0, 1, 0], [2, -5, 4, -1], [-1, 3, -3, 1]], np.float64) / 2.0,
}


def kind_parts(kind):
    """'round_bezier' -> (True, 'bezier'); 'flat_linear' -> (False, None)."""
    shape, basis = kind.split("_", 1)
    return shape == "round", (None if basis == "linear" else basis)


def control_points(cv, ci, basis, tang=None):
    """[n, 4, 4] float64 control points (xyz, radius) of the cubic curves ci of a vertex buffer (Hermite: the Bezier form)."""
    cv = cv.astype(np.float64)
    if basis == "hermite":
        tg = tang.astype(np.float64)
        p0, p1, t0, t1 = cv[ci], cv[ci + 1], tg[ci], tg[ci + 1]
        return np.stack([p0, p0 + t0 / 3.0, p1 - t1 / 3.0, p1], 1)
    return np.stack([cv[ci + j] for j in range(4)], 1)


def cubic_eval(cp, basis, u, der=0):
    """The der-th derivative in u of the cubic curves cp [n, 4, 4] at u [n] or [n, m] -> [n, (m,) 4], float64."""
    M = BASIS_MATRIX["bezier" if basis == "hermite" else basis]
    u = np.asarray(u, np.float64)
    pw = np.stack([np.ones_like(u), u, u * u, u * u * u], -1)
    if der >= 1:
        pw = np.stack([np.zeros_like(u), np.ones_like(u), 2 * u, 3 * u * u], -1)
    if der >= 2:
        pw = np.stack([np.zeros_like(u), np.zeros_like(u), 2 * np.ones_like(u), 6 * u], -1)
    W = pw @ M                                                                   # [..., 4] weights of the control points
    if W.ndim == 2:
        return np.einsum("nk,nkc->nc", W, cp)
    return np.einsum("nmk,nkc->nmc", W, cp)


def _walk(rng, m, step, r0, r1, bend):
    """A random-walk strand of m vertices [m, 4] (xyz, radius) from the origin along +x, the radius going linearly from r0 to r1."""
    p, d = np.zeros(3), np.array([1.0, 0, 0])
    out = []
    for k in range(m):
        out.append(np.concatenate([p, [r0 + (r1 - r0) * k / max(m - 1, 1)]]))
        d = d + rng.normal(scale=bend, size=3)
        d /= np.linalg.norm(d)
        p = p + d * step
    return np.array(out)


def _linear_shapes(rng):
    """Polylines [m, 4] (xyz, radius) in unit scale: each the vertices of one strand of m - 1 segments."""
    def walk(*a):
        return _walk(rng, *a)
    return [
        ("thin", walk(5, 0.25, 0.01, 0.008, 0.3)),
        ("fat", walk(4, 0.3, 0.1, 0.6, 0.5)),                                    # r / length 0.3 to 2
        ("fatter", walk(3, 0.25, 0.5, 0.3, 0.8)),
        ("taper0", np.array([[0, 0, 0, 0.3], [1.0, 0.1, 0, 0.0]])),              # r = 0 at one end
        ("tip0", np.array([[0, 0, 0, 0.0], [0.6, 0.2, 0.1, 0.25], [1.2, 0.1, 0.0, 0.0]])),
        ("vanish", np.array([[0, 0, 0, 0.8], [0.3, 0.05, 0, 0.1]])),             # |r1 - r0| > |p1 - p0|: no cone, one sphere
        ("vanish_mid", np.array([[0, 0, 0, 0.1], [0.4, 0, 0, 0.12], [0.55, 0.05, 0, 0.6], [1.1, 0.1, 0, 0.1]])),
        ("zero_len", np.array([[0, 0, 0, 0.2], [0, 0, 0, 0.2], [0.7, 0.3, 0, 0.15]])),   # p0 == p1: a sphere
        ("zero_len_fat", np.array([[0, 0, 0, 0.3], [0.6, 0, 0, 0.3], [0.6, 0, 0, 0.5]])),
        ("sharp", np.array([[0, 0, 0, 0.1], [0.6, 0, 0, 0.1], [0.65, 0.6, 0, 0.1], [0.05, 0.62, 0.1, 0.12]])),   # joints at ~90 / ~150 degrees
        ("hairpin", np.array([[0, 0, 0, 0.15], [0.8, 0, 0, 0.15], [0.0, 0.1, 0, 0.15]])),
        ("straight", np.array([[0, 0, 0, 0.1], [0.3, 0.3, 0.3, 0.1], [0.6, 0.6, 0.6, 0.1], [0.9, 0.9, 0.9, 0.1]])),   # collinear joints
        ("zero_r", np.array([[0, 0, 0, 0.0], [0.5, 0.2, 0, 0.0], [1.0, 0.0, 0.2, 0.0]])),
        ("long", walk(7, 0.18, 0.06, 0.01, 0.6)),
    ]


def _cubic_shapes(rng):
    """Control vertex sequences [m, 4] (xyz, radius) in unit scale; None tangents: taken from the neighbours (Hermite)."""
    def walk(*a):
        return _walk(rng, *a)
    arc = np.array([[np.cos(a) * 0.2, np.sin(a) * 0.2, 0.05 * a, 0.3] for a in np.linspace(0, 2.5, 7)])   # r > radius of curvature
    return [
        ("thin", walk(7, 0.15, 0.01, 0.008, 0.3), None),
        ("fat", walk(7, 0.15, 0.06, 0.3, 0.4), None),                            # r / length 0.3 to 2
        ("straight", np.array([[0.1 * k, 0.05 * k, 0.0, 0.08] for k in range(7)]), None),   # collinear control points
        ("cusp", np.array([[0, 0, 0, 0.05], [1, 1, 0, 0.05], [0, 1, 0, 0.05], [1, 0, 0, 0.05]]), None),
        ("loop", np.array([[0, 0, 0, 0.06], [1.6, 1.2, 0, 0.06], [-1.6, 1.2, 0.1, 0.06], [0.1, 0, 0.2, 0.06]]), None),
        ("taper0", np.array([[0, 0, 0, 0.25], [0.3, 0.1, 0, 0.15], [0.6, 0.1, 0, 0.07], [0.9, 0, 0, 0.0]]), None),
        ("vanish", np.array([[0, 0, 0, 0.8], [0.1, 0.02, 0, 0.6], [0.2, 0.03, 0, 0.3], [0.3, 0.0, 0, 0.05]]), None),
        ("tight_arc", arc, None),
        ("coincident", np.array([[0, 0, 0, 0.1], [0, 0, 0, 0.1], [0.8, 0.2, 0, 0.1], [0.8, 0.2, 0, 0.1]]), None),   # zero end derivatives
        ("zero_tangents", np.array([[0, 0, 0, 0.1], [0.5, 0.3, 0, 0.12], [1.0, 0.0, 0.1, 0.08], [1.4, 0.4, 0, 0.1]]), "zero"),
        ("zero_r", np.array([[0, 0, 0, 0.0], [0.3, 0.2, 0, 0.0], [0.6, 0.0, 0.1, 0.0], [0.9, 0.1, 0, 0.0]]), None),
        ("long", walk(10, 0.12, 0.05, 0.01, 0.6), None),
    ]


def _strand_buffers(verts, basis, tangent_mode, v_off):
    """Index buffer (first vertex of every curve) and tangents of one strand of control vertices under `basis`."""
    m = len(verts)
    if basis == "bezier":
        m = 1 + 3 * ((m - 1) // 3)
        verts = verts[:m]
        starts = np.arange(0, m - 3, 3)
    elif basis == "hermite":
        starts = np.arange(0, m - 1)
    else:
        starts = np.arange(0, m - 3)
    tg = None
    if basis == "hermite":
        nxt = np.concatenate([verts[1:], verts[-1:] * 2 - verts[-2:-1]])
        prv = np.concatenate([verts[:1] * 2 - verts[1:2], verts[:-1]])
        tg = (nxt - prv) * 0.5
        if tangent_mode == "zero":
            tg = np.zeros_like(tg)
    return verts, (starts + v_off).astype(np.uint32), tg


def _frame(t):
    t = t / max(np.linalg.norm(t), 1e-300)
    a = np.array([1.0, 0, 0]) if abs(t[0]) < 0.9 else np.array([0, 1.0, 0])
    n = np.cross(t, a)
    n /= np.linalg.norm(n)
    return t, n, np.cross(t, n)


def curve_edge_cases(kind, seed=91):
    """Curve sets of one kind and ~4 000 rays at the corners of its intersector's domain.

    Returns dict(curves=[(vertices4, indices, flags or None, geomID, mask, flat)] for the linear kinds,
    cubics=[(vertices4, indices, geomID, mask, basis, tess, tangents or None, round)] for the cubic ones, rays (RTCRayHit[]),
    targets: per ray (geomID, primID, u) of the primitive it was aimed at, mode: per ray the index into RAY_MODES, tscale: per ray
    the size of the problem in units of t -- the distance of the origin from the target plus its diameter, over |dir|; strand:
    {(geomID, primID): name of the strand shape}).
    Geometry 0: unit-scale strands (library neighbour flags, tessellation rate 4, every mask), geometry 1: the same shapes scaled by
    20 about centres 3 000 units from the origin (application neighbour flags, rate 16), geometry 2: a 1e-3 scale copy (mask 0x2,
    rate 1).  Each set ends with invalid primitives: a NaN, a +inf and a -inf vertex and, for linear curves, a negative radius."""
    from embree_b200.rtc import make_rayhits
    rnd, basis = kind_parts(kind)
    rng = np.random.RandomState(seed)
    linear = basis is None
    shapes = _linear_shapes(rng) if linear else _cubic_shapes(rng)
    sets = [(1.0, np.zeros(3), 8.0, 0xFFFFFFFF, 4), (20.0, np.array([3000.0, -3000.0, 3000.0]), 160.0, 0xFFFFFFFF, 16),
            (1e-3, np.array([-2.0, -2.0, 2.0]), 8e-3, 0x2, 1)]
    curves, cubics, prims = [], [], []          # prims: (geomID, strand name, its primIDs, scale) for the ray generator
    invalid = []                                # (geomID, first vertex, radius) of every strand with an invalid vertex
    for gid, (scale, centre, spacing, mask, tess) in enumerate(sets):
        vs, idx, tgs, flags = [], [], [], []
        nv = nprim = 0
        strand_prims = []
        for s, shp in enumerate(shapes):
            name, pts = shp[0], shp[1]
            pts = pts.copy()
            cell = np.array([s % 4, (s // 4) % 4, s // 16], np.float64) * spacing
            pts[:, :3] = (pts[:, :3] - pts[:, :3].mean(0)) * scale + centre + cell
            pts[:, 3] *= scale
            if linear:
                m = len(pts)
                first = np.arange(nv, nv + m - 1, dtype=np.uint32)
                f = np.zeros(m - 1, np.uint8)
                f[1:] |= 1
                f[:-1] |= 2
                if gid == 1 and m > 3:
                    f[1] &= ~np.uint8(2)                  # application flags: the strand is cut in two after its second segment
                    f[2] &= ~np.uint8(1)
                vs.append(pts); idx.append(first); flags.append(f)
                nv += m
            else:
                verts, first, tg = _strand_buffers(pts, basis, shp[2], nv)
                vs.append(verts); idx.append(first); tgs.append(tg if tg is not None else np.zeros_like(verts))
                nv += len(verts)
            strand_prims.append((name, list(range(nprim, nprim + len(first)))))
            nprim += len(first)
        # invalid primitives (dropped by the validity rules), far from every ray's target
        bad_at = centre + np.array([-2.0, -2.0, -2.0]) * spacing
        bad = []
        for val in (np.nan, np.inf, -np.inf) + ((-1.0,) if linear else ()):
            b = np.array([[0, 0, 0, 0.1], [0.3, 0, 0, 0.1], [0.6, 0.1, 0, 0.1], [0.9, 0, 0, 0.1]], np.float64)
            b[:, :3] = b[:, :3] * scale + bad_at
            b[:, 3] *= scale
            if val == -1.0:
                b[1, 3] = -0.05 * scale
            else:
                b[1, 0] = val
            bad_at = bad_at + np.array([0, 1.0, 0]) * spacing * 0.5
            bad.append(b)
            invalid.append((gid, b[0, :3].copy(), 0.1 * scale))
        for b in bad:
            if linear:
                m = len(b)
                vs.append(b); idx.append(np.arange(nv, nv + m - 1, dtype=np.uint32))
                f = np.zeros(m - 1, np.uint8); f[1:] |= 1; f[:-1] |= 2
                flags.append(f)
                nv += m
            else:
                verts, first, tg = _strand_buffers(b, basis, None, nv)
                vs.append(verts); idx.append(first); tgs.append(tg if tg is not None else np.zeros_like(verts))
                nv += len(verts)
        cv = np.concatenate(vs).astype(np.float32)
        ci = np.concatenate(idx).astype(np.uint32)
        if linear:
            cf = np.concatenate(flags).astype(np.uint8) if gid == 1 else None
            curves.append((cv, ci, cf, gid, mask, not rnd))
        else:
            tg = np.concatenate(tgs).astype(np.float32) if basis == "hermite" else None
            cubics.append((cv, ci, gid, mask, basis, tess, tg, rnd))
        for name, plist in strand_prims:
            prims.append((gid, name, plist, scale))

    # ---- rays
    def centreline(gid, p, u):
        """float64 centre, radius and tangent of primitive p of geometry gid at u."""
        if linear:
            cv, ci = curves[gid][0].astype(np.float64), curves[gid][1]
            a, b = cv[ci[p]], cv[ci[p] + 1]
            q = a + (b - a) * u
            return q[:3], q[3], (b - a)[:3]
        cv, ci, _g, _m, _b, _t, tg = cubics[gid][:7]
        cp = control_points(cv, ci[p:p + 1], basis, tg)
        P = cubic_eval(cp, basis, np.array([u]))[0]
        dP = cubic_eval(cp, basis, np.array([u]), der=1)[0]
        return P[:3], P[3], dP[:3]

    org, dirs, tn, tf, tgt, modes, tsc = [], [], [], [], [], [], []
    per = max(1, 4000 // len(prims))
    for (gid, name, plist, scale) in prims:
        for k in range(per):
            mode = k % len(STRAND_MODES)
            p = plist[rng.randint(len(plist))]
            u = rng.uniform(0.05, 0.95)
            if RAY_MODES[mode] == "joint" and len(plist) > 1:
                j = rng.randint(len(plist) - 1)
                p, u = plist[j], 1.0
            if RAY_MODES[mode] == "axis_cap":
                p, u = (plist[0], 0.0) if k % 2 else (plist[-1], 1.0)
            c, r, tv = centreline(gid, p, u)
            if not np.isfinite(tv).all() or np.linalg.norm(tv) < 1e-12 * scale:
                tv = rng.normal(size=3)
            T, N, B = _frame(tv)
            th = rng.uniform(0, 2 * np.pi)
            n = np.cos(th) * N + np.sin(th) * B                                    # a normal of the tube at c
            rr = max(abs(r), 0.02 * scale)
            tnear, tfar = 0.0, np.inf
            m = RAY_MODES[mode]
            if m in ("outside", "joint", "window_near", "window_far", "window_entry"):
                o = c + n * rr * rng.uniform(1.5, 6.0) + T * rr * rng.normal()
                d = c + (N * rng.normal() + B * rng.normal()) * rr * 0.5 - o
            elif m == "on_centreline":
                o, d = c.copy(), rng.normal(size=3)
            elif m == "inside":
                o = c + n * abs(r) * rng.uniform(0.9, 0.999)
                d = rng.normal(size=3)
            elif m == "surface_in":
                o = c + n * abs(r)
                d = -n + rng.normal(size=3) * 0.6
            elif m == "surface_out":
                o = c + n * abs(r)
                d = n + rng.normal(size=3) * 0.6
            elif m == "graze":
                w = np.cos(th) * B - np.sin(th) * N                                # perpendicular to n and to the axis
                w = w + T * rng.normal() * 0.3
                o = c + n * rr * rng.uniform(0.98, 1.02) - w * rr * 4.0
                d = w
            elif m == "axis_cap":
                out = -T if u == 0.0 else T
                o = c + out * rr * rng.uniform(1.5, 4.0) + (N * rng.normal() + B * rng.normal()) * rr * 0.3
                d = -out + (N * rng.normal() + B * rng.normal()) * 0.05
            else:                                                                   # "random": anywhere near the strand
                o = c + rng.normal(size=3) * rr * 4.0
                d = c + rng.normal(size=3) * rr - o
            d = d / max(np.linalg.norm(d), 1e-300)
            tc = float((c - o) @ d)                                                 # the centreline point, in units of |d| = 1
            if m == "window_near":
                tnear = tc * rng.uniform(0.98, 1.02)                                # between the entry and the exit
            elif m == "window_far":
                tfar = tc * rng.uniform(0.99, 1.05)                                 # just before the exit
            elif m == "window_entry":
                tfar = max(tc - abs(r) * rng.uniform(0.9, 1.1), 0.0)                # near the entry
            elif k % 3 == 0:
                tnear = abs(tc) * rng.uniform(0.0, 0.3)
            scale_d = 10.0 ** rng.uniform(-3, 3)
            org.append(o); dirs.append(d * scale_d)
            tn.append(tnear / scale_d); tf.append(tfar / scale_d)
            tgt.append((gid, p, u)); modes.append(mode)
            tsc.append((np.linalg.norm(c - o) + 2 * abs(r) + 1e-30) / scale_d)     # the size of the problem in units of t
    # rays through the first vertex of every strand with an invalid vertex, across the strand: the primitives there are dropped by the
    # validity rules (tests/bvh_check.py), and the strand's valid segments / curves lie past x + 0.5 scale, out of these rays' way
    n_strand = len(org)
    rng2 = np.random.RandomState(seed + 1)
    for (gid, v0, r) in invalid:
        for k in range(24):
            th = rng2.uniform(0, 2 * np.pi)
            n = np.array([0.0, np.cos(th), np.sin(th)])
            w = np.array([0.0, -np.sin(th), np.cos(th)])
            o = v0 + n * r * rng2.uniform(2.0, 6.0) + w * r * rng2.uniform(-0.5, 0.5)
            d = v0 + w * r * rng2.uniform(-0.5, 0.5) - o
            scale_d = 10.0 ** rng2.uniform(-3, 3)
            org.append(o); dirs.append(d / np.linalg.norm(d) * scale_d)
            tn.append(0.0); tf.append(np.inf)
            tgt.append((gid, -1, 0.0)); modes.append(len(STRAND_MODES))
            tsc.append((np.linalg.norm(v0 - o) + 2 * r) / scale_d)
    rays = make_rayhits(np.array(org, np.float32), np.array(dirs, np.float32))
    rays["tnear"] = np.array(tn, np.float32)
    rays["tfar"] = np.maximum(np.array(tf, np.float32), rays["tnear"])
    rays["mask"] = np.array([0xFFFFFFFF, 0x1, 0x2, 0xFFFFFFFF, 0x4], np.uint32)[np.arange(len(rays)) % 5]
    rays["mask"][n_strand:] = 0xFFFFFFFF
    strand = {(gid, p): name for (gid, name, plist, _s) in prims for p in plist}
    return dict(curves=curves, cubics=cubics, rays=rays, strand=strand, targets=np.array(tgt, np.float64), mode=np.array(modes, np.int32),
                tscale=np.array(tsc, np.float64))


STRAND_MODES = ["outside", "on_centreline", "inside", "surface_in", "surface_out", "graze", "axis_cap", "joint",
                "window_near", "window_far", "window_entry", "random"]
RAY_MODES = STRAND_MODES + ["invalid"]      # "invalid": across a strand whose primitives there are invalid -- every layer must miss


def oracle_scene(oracle, S, meshes=()):
    """The curve sets of curve_edge_cases() (+ triangle meshes) as an OracleScene."""
    return oracle.scene(list(meshes), curves=S["curves"], cubics=[c[:5] + (4 if c[5] is None else c[5],) + c[6:] for c in S["cubics"]])


def add_curve_sets(L, dev, sc, S):
    """The curve sets of curve_edge_cases() on a library behind the rtc.py binding; returns the arrays to keep alive."""
    keep = [L.add_round_linear_curves(dev, sc, cv, ci, cf, mask=mask, geom_id=gid, flat=flat)[1] for (cv, ci, cf, gid, mask, flat) in S["curves"]]
    keep += [L.add_flat_cubic_curves(dev, sc, cv, ci, basis, tess, tg, mask=mask, geom_id=gid, round=rnd)[1]
             for (cv, ci, gid, mask, basis, tess, tg, rnd) in S["cubics"]]
    return keep


def _prim_cp(S, gid, prim):
    """float64 control points [1, 4, 4] of cubic curve `prim` of geometry `gid`, or the two vertices [2, 4] of a linear segment."""
    for c in S["curves"]:
        if c[3] == gid:
            return c[0][c[1][prim]:c[1][prim] + 2].astype(np.float64)
    for c in S["cubics"]:
        if c[2] == gid:
            return control_points(c[0], c[1][prim:prim + 1], c[4], c[6])


def curve_edge_disagreements(kind, S, rays, a, b, margin=1e-3, t_tol=1e-4, tie_ulps=None):
    """Rays on which two implementations of one curve kind disagree, and which boundary rule explains each.  A ray differs on hit vs
    miss, on a different primitive at a different distance (beyond TIE_ULPS), or on the same primitive at distances more than t_tol
    apart relative to the size of the problem in units of t (a front hit on one side, a back hit on the other).  tie_ulps (default
    tests/parity.py TIE_ULPS): how far apart two primitives' distances may be and still be a tie (0: only a bit-identical t).  Rules:
      window -- a reported hit distance lies within `margin` (relative to that size) of tnear or tfar;
      graze  -- round linear: tests/parity.py curve_grazing for a primitive either side reports; flat linear: the float64 ribbon
                (tests/curve_exact.py) puts the ray within `margin` of the ribbon's edge or of the self-intersection cut t = 2 r / |d|;
                flat cubics: the nearer hit lies on the edge of its ribbon (|v| >= 0.999, tests/parity.py
                unexplained_ribbon_disagreements) or at the self-intersection cut; round cubics: the nearer hit's normal is
                perpendicular to the ray (|cos| < 0.1, tests/parity.py sweep_disagreements).
      zero_radius -- a primitive either side reports has radius 0 everywhere (a line, met only by rounding);
      stationary  -- cubics: a reported hit lies within 0.05 in u of a point where its curve's centreline stops (a cusp, coincident
                     control points, zero Hermite tangents: |C'(u)| < 1e-2 of its mean) or where the radius reaches the radius of
                     curvature: the sweep's Newton step divides by |C'(u)|, and where the tube folds over itself the ray meets
                     several roots, of which each implementation's subdivision order picks one;
      beyond_the_solid -- round linear: the nearer hit lies outside its segment's float64 solid (tests/curve_exact.py).  The cone's
                     band test y > -ulp takes an absolute ulp, so at a 1e-3 scale it accepts points past the end sphere, outside the
                     segment's box; whether a traversal offers that segment depends on its leaf boxes.
    Returns dict(differ, differ_rows, one count per rule, unexplained, rows=the unexplained rows)."""
    from tests.parity import TIE_ULPS, curve_grazing
    tie_ulps = TIE_ULPS if tie_ulps is None else tie_ulps
    rnd, basis = kind_parts(kind)
    ah, bh = a["geomID"] != 0xFFFFFFFF, b["geomID"] != 0xFFFFFFFF
    ulps = np.abs(a["tfar"].view(np.int32).astype(np.int64) - b["tfar"].view(np.int32).astype(np.int64))
    same = ah & bh & (a["primID"] == b["primID"]) & (a["geomID"] == b["geomID"])
    tscale = S["tscale"]
    with np.errstate(invalid="ignore"):
        far_apart = np.abs(a["tfar"].astype(np.float64) - b["tfar"]) > t_tol * np.maximum(np.abs(a["tfar"].astype(np.float64)), tscale)
    differ = (ah != bh) | (ah & bh & ~same & (ulps > tie_ulps)) | (same & far_apart)
    out = dict(differ=int(differ.sum()), differ_rows=np.nonzero(differ)[0], window=0, graze=0, zero_radius=0, stationary=0, beyond_the_solid=0, unexplained=0, rows=[])
    for i in np.nonzero(differ)[0]:
        tn, tf = float(rays["tnear"][i]), float(rays["tfar"][i])
        hits = [x for x, h in ((a, ah[i]), (b, bh[i])) if h]
        if any(min(abs(float(x["tfar"][i]) - tn), abs(float(x["tfar"][i]) - tf) if np.isfinite(tf) else np.inf) <= margin * tscale[i] for x in hits):
            out["window"] += 1
            continue
        near = min(hits, key=lambda x: float(x["tfar"][i]))
        d = np.array([rays["dir_x"][i], rays["dir_y"][i], rays["dir_z"][i]], np.float64)
        cps = [(x, _prim_cp(S, int(x["geomID"][i]), int(x["primID"][i]))) for x in hits]
        if any(np.abs(cp[..., 3]).max() == 0 for _x, cp in cps):
            out["zero_radius"] += 1        # a tube of radius 0 is a line: whether a ray from on it meets it is decided by rounding alone
            continue
        if basis is not None:
            us = np.linspace(0, 1, 257)
            near_stop = False
            for x, cp in cps:
                cpn = np.repeat(cp, len(us), 0)
                d1, d2 = cubic_eval(cpn, basis, us, der=1)[:, :3], cubic_eval(cpn, basis, us, der=2)[:, :3]
                v = np.linalg.norm(d1, axis=1)
                with np.errstate(invalid="ignore", divide="ignore"):
                    folds = np.abs(cubic_eval(cpn, basis, us)[:, 3]) * np.linalg.norm(np.cross(d1, d2), axis=1) >= v ** 3   # r >= 1 / curvature
                stops = us[(v <= 1e-2 * v.mean()) | folds]
                near_stop |= bool(stops.size) and np.abs(stops - float(x["u"][i])).min() <= 0.05
            if near_stop:
                out["stationary"] += 1     # a cusp or a vanishing end derivative: the sweep's Newton step divides by |C'(u)|
                continue
        elif rnd:
            from tests.curve_exact import round_segment_interval
            cp = _prim_cp(S, int(near["geomID"][i]), int(near["primID"][i]))
            o = np.array([[rays["org_x"][i], rays["org_y"][i], rays["org_z"][i]]], np.float64)
            t_in, t_out = round_segment_interval(o, d[None], cp[:1], cp[1:])
            t = float(near["tfar"][i])
            if not (t_in[0] - margin * tscale[i] <= t <= t_out[0] + margin * tscale[i]):
                out["beyond_the_solid"] += 1   # the cone's band test y > -ulp has an absolute ulp: at a 1e-3 scale it accepts points
                continue                       # past the end sphere, which a traversal offers or not depending on its leaf boxes
        graze = False
        if basis is None and rnd:
            graze = any(curve_grazing(S["curves"][int(x["geomID"][i])][0], S["curves"][int(x["geomID"][i])][1], int(x["primID"][i]), rays[i]) for x in hits)
        elif basis is None:
            from tests.curve_exact import flat_linear_f64
            for x in hits:
                cv, ci = S["curves"][int(x["geomID"][i])][:2]
                t, _u, rim, cut = flat_linear_f64(rays[i:i + 1], cv, ci[int(x["primID"][i]):int(x["primID"][i]) + 1])
                graze |= bool(abs(rim[0, 0]) < margin or abs(t[0, 0] - cut[0, 0]) <= margin * tscale[i])
        elif not rnd:
            cp = _prim_cp(S, int(near["geomID"][i]), int(near["primID"][i]))
            r = cubic_eval(cp, basis, np.array([float(near["u"][i])]))[0, 3]
            graze = abs(float(near["v"][i])) >= 0.999 or abs(float(near["tfar"][i]) - 2 * abs(r) / np.linalg.norm(d)) <= margin * tscale[i]
        else:
            ng = np.array([near["Ng_x"][i], near["Ng_y"][i], near["Ng_z"][i]], np.float64)
            graze = abs(ng @ d) < 0.1 * max(np.linalg.norm(ng) * np.linalg.norm(d), 1e-300)
        if graze:
            out["graze"] += 1
        else:
            out["unexplained"] += 1
            out["rows"].append(int(i))
    return out
