"""Float64 statements of what the curve kinds are, derived from their geometry rather than from any implementation, for
checking the hit records of the fp32 intersectors and deciding whether a difference between two of them sits on a boundary of the
exact test (tests/curve_cases.py).

* Round linear: a segment's solid is the convex hull of its two end spheres, the union of the spheres c(s) = p0 + s (p1 - p0),
  r(s) = r0 + s (r1 - r0), s in [0, 1].  f(P, s) = |P - c(s)| - r(s) is convex in (P, s), so along a ray the solid is one interval
  and its ends are roots of the two sphere quadratics or of the cone quadratic (the lateral surface, where d f / d s = 0, i.e.
  s = ((P - p0) . dP + r0 dr) / g with g = |dP|^2 - dr^2, inside 0 <= s <= 1).  With g <= 0 one end sphere contains the other and
  the solid is that sphere.
  A strand is the union of its segments' solids, so for a ray that starts outside every solid the first hit is the smallest entry
  (where the reference's cone / sphere pieces leave that union, at sharp joints, it departs from this statement).
* Flat linear: the ray-facing ribbon -- the point of the segment whose projection along the ray is closest to the ray, hit when that
  projected distance is at most the interpolated radius, at the distance of that point along the ray.
* Round cubics: the surface of disks of radius r(u) perpendicular to the centreline C(u): a hit P has Q = P - C(u) with |Q| = r(u)
  and Q . C'(u) = 0."""
import numpy as np


def _roots(a, b, c):
    """Real roots of a t^2 + b t + c (float64, [n]) as (lo, hi), NaN where there are none; a ~ 0: the linear root twice."""
    with np.errstate(invalid="ignore", divide="ignore"):
        disc = b * b - 4 * a * c
        q = -0.5 * (b + np.copysign(np.sqrt(np.maximum(disc, 0.0)), b))
        r1, r2 = q / a, c / q
        lin = np.abs(a) <= 1e-300
        r1 = np.where(lin, -c / b, r1)
        r2 = np.where(lin, -c / b, r2)
        ok = (disc >= 0) | lin
        lo, hi = np.where(ok, np.minimum(r1, r2), np.nan), np.where(ok, np.maximum(r1, r2), np.nan)
    return lo, hi


def round_segment_interval(o, d, v0, v1):
    """Entry and exit distance of rays o + t d ([n, 3]) through the solids of round linear segments (v0, v1: [n, 4] xyz + radius);
    (inf, -inf) where a ray misses."""
    p0, r0, p1, r1 = v0[:, :3], v0[:, 3], v1[:, :3], v1[:, 3]
    cands = []
    for c, r in ((p0, r0), (p1, r1)):
        w = o - c
        cands += list(_roots((d * d).sum(1), 2 * (w * d).sum(1), (w * w).sum(1) - r * r))
    dP, dr = p1 - p0, r1 - r0
    g = (dP * dP).sum(1) - dr * dr
    with np.errstate(invalid="ignore", divide="ignore"):
        gg = np.where(g > 0, g, np.nan)
        Q0 = o - p0
        s0, s1 = ((Q0 * dP).sum(1) + r0 * dr) / gg, (d * dP).sum(1) / gg            # s(t) = s0 + t s1 on the cone
        v, w = Q0 - s0[:, None] * dP, d - s1[:, None] * dP
        rs, rt = r0 + dr * s0, dr * s1
        lo, hi = _roots((w * w).sum(1) - rt * rt, 2 * ((v * w).sum(1) - rs * rt), (v * v).sum(1) - rs * rs)
        for t in (lo, hi):
            s = s0 + t * s1
            cands.append(np.where((s >= 0) & (s <= 1) & (rs + rt * t >= 0), t, np.nan))   # (the mirror nappe has negative radius)
    C = np.stack(cands, 1)
    with np.errstate(invalid="ignore"):
        return np.nanmin(np.where(np.isnan(C), np.inf, C), 1), np.nanmax(np.where(np.isnan(C), -np.inf, C), 1)


def flat_linear_f64(rays, cv, ci):
    """The ray-facing ribbon of every segment ci, for every ray: [rays, segments] arrays (t, u, rim) in float64, where rim =
    projected distance / interpolated radius - 1 (a hit needs rim <= 0, tnear <= t <= tfar and t > 2 r(u) / |d|)."""
    o = np.stack([rays["org_x"], rays["org_y"], rays["org_z"]], 1).astype(np.float64)[:, None, :]
    d = np.stack([rays["dir_x"], rays["dir_y"], rays["dir_z"]], 1).astype(np.float64)[:, None, :]
    cv = cv.astype(np.float64)
    p0, p1 = cv[ci][None, :, :3], cv[ci + 1][None, :, :3]
    r0, r1 = cv[ci][None, :, 3], cv[ci + 1][None, :, 3]
    dd = (d * d).sum(-1)
    N = d / np.sqrt(dd)[..., None]
    a, b = p0 - o, p1 - o
    ap = a - (a * N).sum(-1)[..., None] * N
    bp = b - (b * N).sum(-1)[..., None] * N
    e = bp - ap
    with np.errstate(invalid="ignore", divide="ignore"):
        u = np.clip(-(ap * e).sum(-1) / (e * e).sum(-1), 0.0, 1.0)
        u = np.where(np.isfinite(u), u, 0.0)
        q = ap + u[..., None] * e
        rr = r0 + u * (r1 - r0)
        rim = np.sqrt((q * q).sum(-1)) / rr - 1.0
        t = ((a * d).sum(-1) + u * ((b - a) * d).sum(-1)) / dd
    return t, u, rim, 2 * rr / np.sqrt(dd)


def _od(rays):
    o = np.stack([rays["org_x"], rays["org_y"], rays["org_z"]], 1).astype(np.float64)
    d = np.stack([rays["dir_x"], rays["dir_y"], rays["dir_z"]], 1).astype(np.float64)
    return o, d


def round_linear_first_entry(rays, curve_sets):
    """Per ray: the float64 distance of the first entry into the union of the solids of every valid round linear segment the ray's
    mask admits at or after tnear (inf: none), and whether the ray starts outside all of them at tnear (only then is that entry the
    first hit).  curve_sets: [(vertices4, indices, geomID, mask)]."""
    o, d = _od(rays)
    tn = rays["tnear"].astype(np.float64)
    first = np.full(len(rays), np.inf)
    outside = np.ones(len(rays), bool)
    for (cv, ci, _gid, mask) in curve_sets:
        cv = cv.astype(np.float64)
        ok = np.isfinite(cv[ci]).all(1) & np.isfinite(cv[ci + 1]).all(1) & (np.minimum(cv[ci, 3], cv[ci + 1, 3]) >= 0)
        admit = (rays["mask"] & np.uint32(mask)) != 0
        for i in np.nonzero(ok)[0]:
            t_in, t_out = round_segment_interval(o, d, np.broadcast_to(cv[ci[i]], (len(o), 4)), np.broadcast_to(cv[ci[i] + 1], (len(o), 4)))
            outside &= ~(admit & (t_in <= tn) & (tn <= t_out))
            first = np.where(admit & (t_in >= tn), np.minimum(first, t_in), first)
    return first, outside


def flat_linear_closest(rays, curve_sets, tscale, margin=1e-3):
    """Per ray: the float64 distance of the nearest ribbon hit over every valid flat linear segment the ray's mask admits (inf: none),
    and whether no segment sits within `margin` of a decision boundary (the ribbon's edge, tnear, tfar, the self-intersection cut
    t = 2 r / |d|; distances relative to tscale)."""
    tn, tf = rays["tnear"].astype(np.float64)[:, None], rays["tfar"].astype(np.float64)[:, None]
    first = np.full(len(rays), np.inf)
    clear = np.ones(len(rays), bool)
    ts = tscale[:, None]
    for (cv, ci, _gid, mask) in curve_sets:
        v = cv.astype(np.float64)
        ok = np.isfinite(v[ci]).all(1) & np.isfinite(v[ci + 1]).all(1) & (np.minimum(v[ci, 3], v[ci + 1, 3]) >= 0)
        ok &= (v[ci, :3] != v[ci + 1, :3]).any(1)                                   # a segment of zero length has no ribbon
        t, _u, rim, cut = flat_linear_f64(rays, cv, ci[ok])
        admit = ((rays["mask"] & np.uint32(mask)) != 0)[:, None]
        with np.errstate(invalid="ignore"):
            hit = admit & (rim <= 0) & (tn <= t) & (t <= tf) & (t > cut)
            edge = admit & ((np.abs(rim) <= margin) | (np.abs(t - tn) <= margin * ts) | (np.abs(t - tf) <= margin * ts) |
                            (np.abs(t - cut) <= margin * ts))
        first = np.minimum(first, np.where(hit, t, np.inf).min(1, initial=np.inf))
        clear &= ~edge.any(1)
    return first, clear


def sweep_residuals(rays, rec, cp, basis):
    """For round cubic hit records `rec` on curves with control points cp ([n, 4, 4], one per record): |Q| / r(u) - 1 and the cosine
    between Q and C'(u), Q = o + t d - C(u), in float64."""
    from tests.curve_cases import cubic_eval
    o, d = _od(rays)
    u = rec["u"].astype(np.float64)
    C = cubic_eval(cp, basis, u)
    dC = cubic_eval(cp, basis, u, der=1)[:, :3]
    Q = o + rec["tfar"].astype(np.float64)[:, None] * d - C[:, :3]
    nq = np.linalg.norm(Q, axis=1)
    with np.errstate(invalid="ignore", divide="ignore"):
        return nq / C[:, 3] - 1.0, (Q * dC).sum(1) / (nq * np.linalg.norm(dC, axis=1))


def f64_departures(kind, S, rays, rec, sweep_tol=1e-2):
    """The records `rec` of one curve kind's edge-case rays (tests/curve_cases.py) against the float64 statements above.  Returns
    (checked, departs): boolean per ray -- which rays the statement decides, and on which of them the record departs from it.
      round linear: rays that start outside every solid, with no entry within 1e-3 of tnear / tfar: hit iff the first entry into the
                    union lies in [tnear, tfar], at that distance (1e-3 of the size of the problem);
      flat linear:  rays with no ribbon within 1e-3 of a decision boundary: the nearest float64 ribbon hit, at that distance (ditto);
      round cubics: every hit on a curve of nonzero radius: |Q| / r(u) - 1 and the cosine of Q and C'(u) within sweep_tol;
      flat cubics:  none (the ribbon of a tessellated curve is defined by its fp32 tessellation)."""
    from tests.curve_cases import _prim_cp, kind_parts
    rnd, basis = kind_parts(kind)
    ts, tn, tf = S["tscale"], rays["tnear"].astype(np.float64), rays["tfar"].astype(np.float64)
    h = rec["geomID"] != 0xFFFFFFFF
    t = rec["tfar"].astype(np.float64)
    sets = [(c[0], c[1], c[3], c[4]) for c in S["curves"]]
    with np.errstate(invalid="ignore"):
        if basis is None:
            if rnd:
                first, checked = round_linear_first_entry(rays, sets)
                checked &= ~(np.abs(first - tn) <= 1e-3 * ts) & ~(np.abs(first - tf) <= 1e-3 * ts)
            else:
                first, checked = flat_linear_closest(rays, sets, ts)
            want_hit = np.isfinite(first) & (first <= tf)
            departs = checked & ((h != want_hit) | (h & (np.abs(t - first) > 1e-3 * np.maximum(np.abs(first), ts))))
            return checked, departs
        checked = np.zeros(len(rays), bool)
        departs = np.zeros(len(rays), bool)
        if not rnd:
            return checked, departs
        k = np.nonzero(h)[0]
        cp = np.concatenate([_prim_cp(S, int(rec["geomID"][i]), int(rec["primID"][i])) for i in k]) if len(k) else np.zeros((0, 4, 4))
        rr, cc = sweep_residuals(rays[k], rec[k], cp, basis)
        nz = np.abs(cp[:, :, 3]).max(1) > 0
        checked[k[nz]] = True
        departs[k[nz]] = ~((np.abs(rr[nz]) <= sweep_tol) & (np.abs(cc[nz]) <= sweep_tol))
    return checked, departs
