"""Scene edits across commits, checked against a scene built from scratch.

A plain Python model follows every geometry of a scene (kind, vertices, indices, mask, enabled flag, build quality, instance transform
and child scene) and the scene's flags and quality.  A seeded generator edits the scene through the public API and commits; after
every commit the library's closest hits, occlusion and bounds must equal those of the oracle scene built from the model, a commit
with no change must launch nothing and leave the records as they were, and at a few commits the derived caches (the batched
interpolation tables, the device traversable) must agree with the host paths.  Three profiles drive the commit paths: `two_level`
(a DYNAMIC scene of small meshes beside one large static mesh: the per-mesh BVHs kept across commits), `refit` (REFIT meshes in one
BVH) and `mixed` (quads, points, curves and instances).  One seed per profile is also replayed on the unmodified reference (its
answers for every 40th ray are stored under tests/golden/reference/).

Regression tests: a kept per-mesh BVH is not reused under another geomID; a REFIT mesh whose index buffer changed is rebuilt; a
triangle made valid again by a vertex update is hit after the next commit where the reference hits it (a scene that is not DYNAMIC, or
not of LOW quality: the reference rebuilds those) and missed where the reference refits and misses it (DYNAMIC at LOW quality).  The
reference's
EnableDisableGeometryTest / DisableAndDetachGeometryTest (tutorials/verify/verify.cpp:1645-1790) are ported over triangle, quad, curve
and point geometries."""
import ctypes as C

import numpy as np
import pytest

from embree_b200 import scenes
from embree_b200.rtc import (RTCBounds, RTC_BUFFER_TYPE_INDEX, RTC_BUFFER_TYPE_VERTEX, RTC_BUILD_QUALITY_LOW, RTC_BUILD_QUALITY_MEDIUM,
                             RTC_BUILD_QUALITY_REFIT, RTC_FORMAT_FLOAT3, RTC_FORMAT_FLOAT3X4_COLUMN_MAJOR, RTC_FORMAT_FLOAT4, RTC_FORMAT_UINT,
                             RTC_FORMAT_UINT3, RTC_FORMAT_UINT4, RTC_SCENE_FLAG_DYNAMIC, RTC_SCENE_FLAG_NONE, RTC_SCENE_FLAG_ROBUST, _ptr,
                             make_rayhits, rays_of)
from tests.parity import (api_trace_mt, compare_hits, explain_hit_miss, load_oracle, point_disagreements, reference_outputs,
                          unexplained_curve_disagreements)
from tests.test_device_traversal import compare_queries, devtrace  # noqa: F401  (devtrace: the fixture of the device-side queries)

pytestmark = pytest.mark.gpu
TOL = 1e-4
INVALID = 0xFFFFFFFF
TRI, QUAD, POINTS, CURVE, INST = "tri", "quad", "points", "curve", "inst"
GEOM_TYPE = {TRI: 0, QUAD: 1, CURVE: 16, POINTS: 50, INST: 121}
CHILD_ID = 100            # geomID of the instanced child scene's mesh: apart from every top-level ID
N_RAYS = 20000
N_COMMITS = 30
REF_STRIDE = 40           # every REF_STRIDE-th ray of each commit is pinned to the reference's answer
MASKS = [0xFFFFFFFF, 0x1, 0x2, 0x3, 0xFFFFFFFE]


# ---- the model ----------------------------------------------------------------------------------------------------------
class Geo:
    """One geometry object of the model: its handle (one reference held by the model) and the host arrays its shared buffers
    point at.  Every array ever handed to the library stays alive with the object."""

    def __init__(self, L, dev, kind, v=None, idx=None, quality=RTC_BUILD_QUALITY_MEDIUM, mask=0xFFFFFFFF, child=None, xfm=None):
        self.L, self.kind, self.quality, self.mask, self.enabled, self.child = L, kind, quality, mask, True, child
        self.keep, self.broken = [], None     # broken: (rows, original index rows) of the triangles given out-of-range indices
        self.h = L.rtcNewGeometry(dev, GEOM_TYPE[kind])
        if kind == INST:
            L.rtcSetGeometryInstancedScene(self.h, child.sc)
            self.set_xfm(xfm)
        else:
            self.set_vertices(v)
            if kind != POINTS:
                self.set_indices(idx)
                self.full = self.idx.copy()     # the index rows a halved buffer is restored from
        L.rtcSetGeometryMask(self.h, mask)
        if kind in (TRI, QUAD):
            L.rtcSetGeometryBuildQuality(self.h, quality)
        L.rtcCommitGeometry(self.h)

    def set_vertices(self, v):
        w = 3 if self.kind in (TRI, QUAD) else 4
        v = np.ascontiguousarray(v, np.float32).reshape(-1, w)
        buf = np.zeros(v.size + 4, np.float32)          # 16 B of padding after the last vertex (README.md:4830)
        buf[:v.size] = v.ravel()
        self.keep.append(buf)
        self.v = buf[:v.size].reshape(-1, w)            # a view: edits in place reach the shared buffer
        self.L.rtcSetSharedGeometryBuffer(self.h, RTC_BUFFER_TYPE_VERTEX, 0, RTC_FORMAT_FLOAT3 if w == 3 else RTC_FORMAT_FLOAT4,
                                          _ptr(buf), 0, 4 * w, len(v))

    def set_indices(self, idx):
        fmt, w = {TRI: (RTC_FORMAT_UINT3, 3), QUAD: (RTC_FORMAT_UINT4, 4), CURVE: (RTC_FORMAT_UINT, 1)}[self.kind]
        self.idx = np.ascontiguousarray(idx, np.uint32).reshape(-1, w) if w > 1 else np.ascontiguousarray(idx, np.uint32).reshape(-1)
        self.keep.append(self.idx)
        self.L.rtcSetSharedGeometryBuffer(self.h, RTC_BUFFER_TYPE_INDEX, 0, fmt, _ptr(self.idx), 0, 4 * w, len(self.idx))

    def set_xfm(self, xfm):
        self.xfm = np.ascontiguousarray(xfm, np.float32).reshape(12)
        self.keep.append(self.xfm)
        self.L.rtcSetGeometryTransform(self.h, 0, RTC_FORMAT_FLOAT3X4_COLUMN_MAJOR, _ptr(self.xfm))

    def update(self, buffer_type):
        self.L.rtcUpdateGeometryBuffer(self.h, buffer_type, 0)

    def commit(self):
        self.L.rtcCommitGeometry(self.h)


class Child:
    """The scene the instances of the mixed profile instantiate: one triangle mesh (geomID CHILD_ID)."""

    def __init__(self, L, dev, rng):
        self.L = L
        self.sc = L.rtcNewScene(dev)
        v, t = scenes.triangle_sphere(int(rng.randint(8, 16)))
        self.geo = Geo(L, dev, TRI, (v * np.float32(0.6)).astype(np.float32), t)
        L.rtcAttachGeometryByID(self.sc, self.geo.h, CHILD_ID)
        L.rtcCommitScene(self.sc)

    def release(self):
        self.L.rtcReleaseGeometry(self.geo.h)
        self.L.rtcReleaseScene(self.sc)


class Model:
    def __init__(self, L, dev, flags, quality):
        self.L, self.dev, self.flags, self.quality = L, dev, flags, quality
        self.sc = L.rtcNewScene(dev)
        L.rtcSetSceneFlags(self.sc, flags)
        L.rtcSetSceneBuildQuality(self.sc, quality)
        self.geos, self.children, self.retired = {}, [], []

    def lowest_free(self):
        i = 0
        while i in self.geos:
            i += 1
        return i

    def attach(self, geo, gid=None):
        if gid is None:
            want = self.lowest_free()
            gid = self.L.rtcAttachGeometry(self.sc, geo.h)
            assert gid == want, (gid, want)             # the lowest free ID, as the reference's IDPool
        else:
            self.L.rtcAttachGeometryByID(self.sc, geo.h, gid)
        self.geos[gid] = geo
        return gid

    def detach(self, gid):
        self.L.rtcDetachGeometry(self.sc, gid)
        return self.geos.pop(gid)

    def set_flags(self, flags):
        self.flags = flags
        self.L.rtcSetSceneFlags(self.sc, flags)

    def set_quality(self, q):
        self.quality = q
        self.L.rtcSetSceneBuildQuality(self.sc, q)

    def commit(self):
        self.L.rtcCommitScene(self.sc)
        self.L.check(self.dev)

    def release(self):
        for g in set(self.geos.values()) | set(self.retired):
            self.L.rtcReleaseGeometry(g.h)
        self.L.rtcReleaseScene(self.sc)
        for c in self.children:
            c.release()

    def snapshot(self):
        """What the oracle needs of the committed scene: copies of every enabled geometry's arrays."""
        out = []
        for gid, g in sorted(self.geos.items()):
            if not g.enabled:
                continue
            if g.kind == INST:
                out.append((gid, INST, g.child.geo.v.copy(), g.child.geo.idx.copy(), g.mask, g.xfm.copy()))
            else:
                out.append((gid, g.kind, g.v.copy(), None if g.kind == POINTS else g.idx.copy(), g.mask, None))
        # the REFIT quad meshes the reference refits (a DYNAMIC scene of LOW quality), see test_refit_quad_mesh_follows_its_vertices
        refit_quads = [gid for gid, g in self.geos.items() if g.enabled and g.kind == QUAD and g.quality == RTC_BUILD_QUALITY_REFIT] \
            if (self.flags & RTC_SCENE_FLAG_DYNAMIC) and self.quality == RTC_BUILD_QUALITY_LOW else []
        return dict(geoms=out, robust=bool(self.flags & RTC_SCENE_FLAG_ROBUST), refit_quads=refit_quads)


def oracle_scene(O, snap, only=None):
    """The oracle scene of a snapshot; only=(geomID, primID, instID): the one primitive a hit reports, alone."""
    meshes, points, curves, instances = [], [], [], []
    for (gid, kind, v, idx, mask, xfm) in snap["geoms"]:
        if only is not None and gid != (only[0] if only[2] == INVALID else only[2]):
            continue
        if kind == INST:
            ci = idx if only is None else idx[only[1]:only[1] + 1]
            instances.append((O.scene([(v, ci, CHILD_ID, 0xFFFFFFFF)]), xfm, gid, mask))
            continue
        if only is not None:
            p = only[1]
            if kind == POINTS:
                v = v[p:p + 1]
            else:
                idx = idx[p:p + 1]
        if kind in (TRI, QUAD):
            meshes.append((v, idx, gid, mask))
        elif kind == POINTS:
            points.append((v, "sphere", None, gid, mask))
        else:
            curves.append((v, idx, None, gid, mask, False))
    return O.scene(meshes, robust=snap["robust"], instances=instances, curves=curves, points=points)


def check_hits(O, snap, rays, want, got, stage):
    """`got` (this library) against `want` (the oracle or the reference) for the same scene.  No hit may name a geomID the scene
    does not hold enabled.  Rays on which either side hits a point or a curve go through the graze explainers of tests/parity.py
    (points with t_tol: the same point at another distance is a difference too), and where both sides hit the same curve segment t
    must agree within TOL; on every other ray ids must be equal (or a tie on a shared vertex), t / u / v within TOL, and every
    hit / miss difference must be a hit the reference's own arithmetic accepts for that primitive alone (explain_hit_miss)."""
    curve_sets = {gid: (v, idx) for (gid, kind, v, idx, _m, _x) in snap["geoms"] if kind == CURVE}
    point_sets = {gid: (v, "sphere", None) for (gid, kind, v, _i, _m, _x) in snap["geoms"] if kind == POINTS}
    enabled = {gid for (gid, *_rest) in snap["geoms"]}
    stray = np.setdiff1d(got["geomID"][(got["geomID"] != INVALID) & (got["instID"] == INVALID)], list(enabled))
    assert len(stray) == 0, (stage, "hits on geomIDs that are not enabled in the scene", stray)
    for (gid, kind, v, idx, _m, _x) in snap["geoms"]:
        if kind in (TRI, QUAD):
            on = (got["geomID"] == gid) & (got["instID"] == INVALID)
            assert (got["primID"][on] < len(idx)).all(), (stage, "primIDs beyond the mesh", gid, got["primID"][on].max())
    top = [r["instID"] == INVALID for r in (want, got)]
    on_point = [np.isin(r["geomID"], list(point_sets)) & t for r, t in zip((want, got), top)]
    on_curve = [np.isin(r["geomID"], list(curve_sets)) & t for r, t in zip((want, got), top)]
    inv = on_point[0] | on_point[1] | on_curve[0] | on_curve[1]
    for i in np.nonzero(inv)[0]:
        s = slice(i, i + 1)
        c = unexplained_curve_disagreements(rays[s], want[s], got[s], curve_sets)[1]
        p = point_disagreements(rays[s], want[s], got[s], point_sets, t_tol=1e-4)[1]
        points, curves = on_point[0][i] or on_point[1][i], on_curve[0][i] or on_curve[1][i]
        ok = (p == 0 or (curves and c == 0)) if points else c == 0
        assert ok, (stage, "point / curve disagreement", i, want[s], got[s])
    same_curve = on_curve[0] & on_curve[1]
    rep = compare_hits(want[same_curve], got[same_curve], TOL)
    assert rep["max_rel_t"] <= TOL, (stage, "curve distances", rep)
    rest = np.nonzero(~inv)[0]
    tie_meshes = [(v, idx, gid, 0) for (gid, kind, v, idx, _m, _x) in snap["geoms"] if kind in (TRI, QUAD)]
    tie_meshes += [(v, idx, CHILD_ID, 0) for (gid, kind, v, idx, _m, _x) in snap["geoms"] if kind == INST][:1]
    rep = compare_hits(want[rest], got[rest], TOL, meshes=tie_meshes)
    assert rep["id_mismatch"] == 0 and rep["tie"] <= 20, (stage, rep)
    assert rep["max_rel_t"] <= TOL and rep["max_abs_uv"] <= TOL and rep["miss_untouched"], (stage, rep)
    lost, bad = explain_hit_miss(O, rays[rest], want[rest], got[rest], lambda g, p, i: oracle_scene(O, snap, (g, p, i)))
    assert lost == 0 and bad == 0, (stage, "hit / miss", lost, bad, rep)
    return rep


def scene_bounds(L, sc):
    b = RTCBounds()
    L.rtcGetSceneBounds(sc, C.byref(b))
    return np.array([b.lower_x, b.lower_y, b.lower_z, b.upper_x, b.upper_y, b.upper_z], np.float32)


# ---- geometry generators ------------------------------------------------------------------------------------------------
def small_sphere(rng, box=3.0):
    v, t = scenes.triangle_sphere(int(rng.randint(6, 20)))
    c = rng.uniform(-box, box, 3).astype(np.float32)
    return (v * np.float32(rng.uniform(0.2, 0.9)) + c).astype(np.float32), t.copy()


def quad_sphere(n, center=(0.0, 0.0, 0.0), radius=1.0):
    """A latitude-longitude sphere of quads (the poles are quads with two equal vertices)."""
    th = np.linspace(0, np.pi, n + 1)
    ph = np.linspace(0, 2 * np.pi, 2 * n, endpoint=False)
    T, P = np.meshgrid(th, ph, indexing="ij")
    v = np.stack([np.sin(T) * np.cos(P), np.cos(T), np.sin(T) * np.sin(P)], -1).reshape(-1, 3) * radius + np.asarray(center)
    q = []
    m = 2 * n
    for i in range(n):
        for j in range(m):
            a, b = i * m + j, i * m + (j + 1) % m
            q.append((a, a + m, b + m, b))
    return v.astype(np.float32), np.array(q, np.uint32)


def point_set(rng, n=300, box=3.0):
    c = rng.uniform(-box, box, (n, 3))
    return np.concatenate([c, rng.uniform(0.05, 0.2, (n, 1))], 1).astype(np.float32)


def curve_set(rng, strands=60, segs=4, box=3.0):
    """Round linear curves: `strands` polylines of `segs` segments; index = first vertex of each segment."""
    v, idx = [], []
    for s in range(strands):
        p = rng.uniform(-box, box, 3)
        d = rng.normal(size=3) * 0.25
        for k in range(segs + 1):
            v.append([*(p + k * d + rng.normal(scale=0.05, size=3)), rng.uniform(0.02, 0.08)])
        idx += [s * (segs + 1) + k for k in range(segs)]
    return np.array(v, np.float32), np.array(idx, np.uint32)


def random_xfm(rng):
    q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
    m = q * rng.uniform(0.7, 1.3, 3)[None, :]
    return np.concatenate([m[:, 0], m[:, 1], m[:, 2], rng.uniform(-2.5, 2.5, 3)]).astype(np.float32)


def profile_rays(seed, box):
    rng = np.random.RandomState(seed)
    r = make_rayhits(rng.uniform(-box, box, (N_RAYS, 3)), rng.normal(size=(N_RAYS, 3)))
    r["mask"][1::7] = 0x1
    r["mask"][2::7] = 0x2
    r["tfar"][3::11] = rng.uniform(0.5, 3.0, len(r["tfar"][3::11])).astype(np.float32)
    return r


# ---- the edit sequence --------------------------------------------------------------------------------------------------
class Editor:
    """Seeded edits on a Model.  Every edit returns a label, or None when it does not apply to the scene as it is."""

    def __init__(self, model, rng, profile):
        self.m, self.rng, self.profile = model, rng, profile
        self.L, self.dev = model.L, model.dev

    def pick(self, kinds=(TRI,), cond=lambda g: True, n=1):
        ids = [gid for gid, g in sorted(self.m.geos.items()) if g.kind in kinds and cond(g) and getattr(g, "small", True)]
        if len(ids) < n:
            return None
        return [int(x) for x in self.rng.choice(ids, n, replace=False)]

    def new_geo(self, kind, like=None):
        rng = self.rng
        if kind == TRI:
            v, t = small_sphere(rng) if like is None else ((like.v + np.float32(rng.uniform(-0.5, 0.5))).astype(np.float32), like.full)
            return Geo(self.L, self.dev, TRI, v, t, quality=like.quality if like is not None else RTC_BUILD_QUALITY_MEDIUM)
        if kind == QUAD:
            v, q = quad_sphere(int(rng.randint(6, 14)), rng.uniform(-3, 3, 3), rng.uniform(0.3, 0.9)) if like is None else \
                ((like.v + np.float32(rng.uniform(-0.5, 0.5))).astype(np.float32), like.full)
            return Geo(self.L, self.dev, QUAD, v, q, quality=like.quality if like is not None else RTC_BUILD_QUALITY_MEDIUM)
        if kind == POINTS:
            return Geo(self.L, self.dev, POINTS, point_set(rng) if like is None else like.v + np.float32([0.3, 0, 0, 0]))
        if kind == CURVE:
            cv, ci = curve_set(rng) if like is None else (like.v + np.float32([0, 0.3, 0, 0]), like.full)
            return Geo(self.L, self.dev, CURVE, cv, ci)
        child = self.m.children[0] if like is None else like.child
        return Geo(self.L, self.dev, INST, child=child, xfm=random_xfm(rng))

    def kinds(self):
        return {"two_level": (TRI,), "refit": (TRI, QUAD), "mixed": (TRI, QUAD, POINTS, CURVE, INST)}[self.profile]

    # -- geometry edits
    def move_vertices(self, n=1):
        ids = self.pick(tuple(k for k in self.kinds() if k != INST), n=n)
        if ids is None:
            return None
        for gid in ids:
            g = self.m.geos[gid]
            g.v[:, :3] += self.rng.normal(scale=0.3, size=3).astype(np.float32)
            g.update(RTC_BUFFER_TYPE_VERTEX)
            g.commit()
        return f"move vertices of {ids}"

    def deform_refit(self, every=False):
        ids = self.pick((TRI, QUAD), lambda g: g.quality == RTC_BUILD_QUALITY_REFIT)
        if every:
            ids = [gid for gid, g in sorted(self.m.geos.items()) if g.kind in (TRI, QUAD) and g.quality == RTC_BUILD_QUALITY_REFIT]
        if not ids:
            return None
        for gid in ids:
            g = self.m.geos[gid]
            c = g.v.mean(0)
            g.v[:] = (c + (g.v - c) * self.rng.uniform(0.8, 1.2, 3) + self.rng.normal(scale=0.05, size=3)).astype(np.float32)
            g.update(RTC_BUFFER_TYPE_VERTEX)
            g.commit()
        return f"deform REFIT {ids}"

    def rewrite_indices(self, new_buffer):
        """Same triangle count: rows permuted and rotated, or a few triangles given an out-of-range index, or those fixed again."""
        ids = self.pick((TRI, QUAD), lambda g: len(g.idx) == len(g.full))
        if ids is None:
            return None
        g = self.m.geos[ids[0]]
        idx = g.idx.copy()
        if g.broken is not None:
            rows, orig = g.broken
            idx[rows] = orig
            g.broken, what = None, "fixed"
        elif self.rng.rand() < 0.5:
            rows = self.rng.choice(len(idx), 3, replace=False)
            g.broken = (rows, idx[rows].copy())
            idx[rows, 0] = len(g.v) + 7
            what = "broken"
        else:
            perm = self.rng.permutation(len(idx))
            idx = np.roll(idx[perm], 1, axis=1)
            g.full = idx.copy()
            what = "permuted"
        if new_buffer:
            g.set_indices(idx)
        else:
            g.idx[:] = idx
            g.update(RTC_BUFFER_TYPE_INDEX)
        g.commit()
        return f"indices of {ids[0]} {what} ({'new buffer' if new_buffer else 'update'})"

    def change_count(self):
        ids = self.pick((TRI, QUAD), lambda g: g.broken is None)
        if ids is None:
            return None
        g = self.m.geos[ids[0]]
        g.set_indices(g.full if len(g.idx) < len(g.full) else g.full[: len(g.full) // 2].copy())
        g.commit()
        return f"{ids[0]}: {len(g.idx)} primitives"

    def mask(self):
        ids = self.pick(self.kinds())
        if ids is None:
            return None
        g = self.m.geos[ids[0]]
        g.mask = int(self.rng.choice(MASKS))
        self.L.rtcSetGeometryMask(g.h, g.mask)
        g.commit()
        return f"mask of {ids[0]} = {g.mask:#x}"

    def toggle_enabled(self):
        ids = self.pick(self.kinds())
        if ids is None:
            return None
        g = self.m.geos[ids[0]]
        g.enabled = not g.enabled
        (self.L.rtcEnableGeometry if g.enabled else self.L.rtcDisableGeometry)(g.h)
        return f"{ids[0]} {'enabled' if g.enabled else 'disabled'}"

    def detach(self):
        if len(self.m.geos) < 5:
            return None
        ids = self.pick(self.kinds())
        if ids is None:
            return None
        self.m.retired.append(self.m.detach(ids[0]))
        return f"{ids[0]} detached"

    def attach_lowest(self):
        kinds = self.kinds()
        g = self.new_geo(kinds[int(self.rng.randint(len(kinds)))])
        return f"attached at {self.m.attach(g)}"

    def move_id(self):
        ids = self.pick(self.kinds())
        if ids is None:
            return None
        free = [i for i in range(40) if i not in self.m.geos]
        to = int(self.rng.choice(free))
        self.m.attach(self.m.detach(ids[0]), to)
        return f"{ids[0]} moved to ID {to}"

    def swap_ids(self):
        ids = self.pick(self.kinds(), n=2)
        if ids is None:
            return None
        a, b = ids
        ga, gb = self.m.detach(a), self.m.detach(b)
        self.m.attach(ga, b)
        self.m.attach(gb, a)
        return f"{a} and {b} swapped IDs"

    def replace(self):
        ids = self.pick(self.kinds(), lambda g: g.broken is None)
        if ids is None:
            return None
        old = self.m.detach(ids[0])
        self.m.retired.append(old)
        new = self.new_geo(old.kind, like=old)
        if old.mask != 0xFFFFFFFF:
            new.mask = old.mask
            self.L.rtcSetGeometryMask(new.h, old.mask)
            new.commit()
        self.m.attach(new, ids[0])
        return f"{ids[0]} replaced by a new object of the same size"

    def switch_refit(self):
        ids = self.pick((TRI, QUAD))
        if ids is None:
            return None
        g = self.m.geos[ids[0]]
        g.quality = RTC_BUILD_QUALITY_MEDIUM if g.quality == RTC_BUILD_QUALITY_REFIT else RTC_BUILD_QUALITY_REFIT
        self.L.rtcSetGeometryBuildQuality(g.h, g.quality)
        g.commit()
        return f"{ids[0]} quality {g.quality}"

    def scene_quality(self):
        self.m.set_quality(RTC_BUILD_QUALITY_LOW if self.m.quality == RTC_BUILD_QUALITY_MEDIUM else RTC_BUILD_QUALITY_MEDIUM)
        return f"scene quality {self.m.quality}"

    def toggle_robust(self):
        self.m.set_flags(self.m.flags ^ RTC_SCENE_FLAG_ROBUST)
        return f"flags {self.m.flags}"

    def toggle_dynamic(self):
        self.m.set_flags(self.m.flags ^ RTC_SCENE_FLAG_DYNAMIC)
        return f"flags {self.m.flags}"

    def add_remove_other_kind(self):
        """A quad mesh or a point set in a scene of triangle meshes: the scene leaves the two-level regime while it is there."""
        extra = [gid for gid, g in self.m.geos.items() if g.kind in (QUAD, POINTS) and getattr(g, "extra", False)]
        if extra:
            self.m.retired.append(self.m.detach(extra[0]))
            return f"{extra[0]} ({'quad' if self.m.retired[-1].kind == QUAD else 'points'}) removed"
        g = self.new_geo(QUAD if self.rng.rand() < 0.5 else POINTS)
        g.extra = True
        return f"{g.kind} attached at {self.m.attach(g)}"

    def child_edit(self):
        if not self.m.children:
            return None
        c = self.m.children[0]
        c.geo.v[:] += self.rng.normal(scale=0.1, size=3).astype(np.float32)
        c.geo.update(RTC_BUFFER_TYPE_VERTEX)
        c.geo.commit()
        self.L.rtcCommitScene(c.sc)
        return "child scene edited and re-committed"

    def transform(self):
        ids = self.pick((INST,))
        if ids is None:
            return None
        g = self.m.geos[ids[0]]
        g.set_xfm(random_xfm(self.rng))
        g.commit()
        return f"instance {ids[0]} transform"

    def no_change(self):
        return "no change"

    WEIGHTS = {
        "two_level": dict(move_vertices=6, move_many=2, deform_refit=2, rewrite_update=2, rewrite_new=2, change_count=1, mask=1, toggle_enabled=2,
                          detach=1, attach_lowest=1, move_id=3, swap_ids=2, replace=1, switch_refit=1, scene_quality=1, toggle_robust=1,
                          toggle_dynamic=0.3, add_remove_other_kind=1, no_change=1),
        "refit": dict(deform_all=8, rewrite_update=3, rewrite_new=2, change_count=1, mask=1, toggle_enabled=1, move_id=1, swap_ids=1, replace=1,
                      switch_refit=1, scene_quality=1, toggle_robust=1, toggle_dynamic=1, add_remove_quad=1, no_change=1),
        "mixed": dict(move_vertices=4, rewrite_update=1, rewrite_new=1, change_count=1, mask=2, toggle_enabled=2, detach=1, attach_lowest=2,
                      move_id=2, swap_ids=2, replace=1, scene_quality=1, toggle_robust=1, child_edit=2, transform=2, no_change=1),
    }

    def run(self, name):
        return {"move_many": lambda: self.move_vertices(n=4), "deform_all": lambda: self.deform_refit(every=True),
                "rewrite_update": lambda: self.rewrite_indices(False), "rewrite_new": lambda: self.rewrite_indices(True),
                "add_remove_quad": self.add_remove_quad}.get(name, getattr(self, name, None))()

    def add_remove_quad(self):
        quads = [gid for gid, g in self.m.geos.items() if g.kind == QUAD]
        if quads:
            self.m.retired.append(self.m.detach(quads[0]))
            return f"quad mesh {quads[0]} removed"
        g = self.new_geo(QUAD)
        g.quality = RTC_BUILD_QUALITY_REFIT
        self.L.rtcSetGeometryBuildQuality(g.h, g.quality)
        g.commit()
        return f"quad mesh attached at {self.m.attach(g)}"

    def random_edit(self):
        w = self.WEIGHTS[self.profile]
        names = sorted(w)
        p = np.array([w[n] for n in names], np.float64)
        while True:
            label = self.run(names[self.rng.choice(len(names), p=p / p.sum())])
            if label is not None:
                return label


def build_profile(L, dev, profile, seed):
    """The scene a profile starts from, committed once, and the edits of its fixed prologue (one commit each: every path the
    profile is for is reached whatever the seed) before the random ones."""
    rng = np.random.RandomState(seed)
    if profile == "two_level":
        m = Model(L, dev, RTC_SCENE_FLAG_DYNAMIC, RTC_BUILD_QUALITY_MEDIUM)
        for i in range(24):
            v, t = small_sphere(rng)
            m.attach(Geo(L, dev, TRI, v, t, quality=RTC_BUILD_QUALITY_REFIT if i in (5, 9) else RTC_BUILD_QUALITY_MEDIUM), i)
        v, t = scenes.triangle_sphere(250)     # ~250 k triangles: a commit that changes one or two small meshes takes the two-level path
        big = Geo(L, dev, TRI, (v * np.float32([6.0, 0.4, 6.0]) + np.float32([0.0, -4.0, 0.0])).astype(np.float32), t)
        big.small = False
        m.attach(big, 24)
        prologue = ["move_vertices", "scene_quality+move_many"]
    elif profile == "refit":
        m = Model(L, dev, RTC_SCENE_FLAG_DYNAMIC, RTC_BUILD_QUALITY_MEDIUM)
        for i in range(5):
            v, t = scenes.triangle_sphere(int(rng.randint(12, 30)), rng.uniform(-2.5, 2.5, 3), rng.uniform(0.4, 1.2))
            m.attach(Geo(L, dev, TRI, v, t, quality=RTC_BUILD_QUALITY_REFIT), i)
        v, q = quad_sphere(12, rng.uniform(-2.5, 2.5, 3), 0.8)
        m.attach(Geo(L, dev, QUAD, v, q, quality=RTC_BUILD_QUALITY_REFIT), 5)
        prologue = ["deform_all", "scene_quality"]
    else:
        m = Model(L, dev, RTC_SCENE_FLAG_NONE, RTC_BUILD_QUALITY_MEDIUM)
        m.children.append(Child(L, dev, rng))
        ed = Editor(m, rng, profile)
        for kind in (TRI, TRI, QUAD, POINTS, CURVE, INST, INST):
            m.attach(ed.new_geo(kind))
        prologue = ["scene_quality"]
    return m, rng, prologue


PATHS = {"two_level": {0, 1, 3}, "refit": {0, 1, 2}, "mixed": {0, 1}}   # rtcb200GetSceneStats builder: 0 LBVH, 1 SAH, 2 refit, 3 two-level
RAY_BOX = {"two_level": 5.0, "refit": 4.0, "mixed": 4.0}


def run_sequence(L, dev, profile, seed, on_commit):
    """Build the profile's scene and apply its prologue and random edits, N_COMMITS commits in all; on_commit(k, label, model)
    after each commit (k = 0 is the first)."""
    m, rng, prologue = build_profile(L, dev, profile, seed)
    ed = Editor(m, rng, profile)
    try:
        m.commit()
        on_commit(0, "first commit", m)
        for k in range(1, N_COMMITS + 1):
            if k <= len(prologue):
                label = "; ".join(ed.run(e) for e in prologue[k - 1].split("+"))
            else:
                label = ed.random_edit()
            if label != "no change":
                m.commit()
            on_commit(k, label, m)
    finally:
        m.release()


def reference_answers(profile, seed):
    """The unmodified reference's hits at every commit of one sequence (live where oracle/_ref is built, stored otherwise)."""
    rays = profile_rays(seed, RAY_BOX[profile])

    def run(R):
        rd = R.new_device(None)
        out = {}

        def on_commit(k, label, m):
            out[f"c{k}"] = api_trace_mt(R, m.sc, rays.copy(), 8)
        run_sequence(R, rd, profile, seed, on_commit)
        R.rtcReleaseDevice(rd)
        return out
    return reference_outputs(f"scene_edits_{profile}", run, {f"c{k}": rays for k in range(N_COMMITS + 1)}, stride=REF_STRIDE)


PINNED_SEED = {"two_level": 11, "refit": 21, "mixed": 31}
SEEDS = {"two_level": [11, 12], "refit": [21, 22], "mixed": [31, 32]}


# ---- 1, 3, 4: edit sequences against a from-scratch oracle scene, the reference and the derived caches ---------------------
@pytest.mark.parametrize("profile,seed", [(p, s) for p in ("two_level", "refit", "mixed") for s in SEEDS[p]])
def test_edit_sequence_matches_a_scene_built_from_scratch(b200, devtrace, profile, seed):
    from tests.test_interpolate import host_interpolate
    lib, dev = b200
    O = load_oracle()
    rays = profile_rays(seed, RAY_BOX[profile])
    ref, rows = reference_answers(profile, seed) if seed == PINNED_SEED[profile] else (None, None)
    builders, last = [], {}

    def on_commit(k, label, m):
        stage = f"{profile} seed {seed} commit {k}: {label}"
        st = lib.scene_stats(m.sc)
        if label == "no change":       # nothing to do: no launch, the same arrays and records
            l0 = lib.rtcb200GetLaunchCount()
            m.commit()
            assert lib.rtcb200GetLaunchCount() == l0, stage
            arr = lib.scene_arrays(m.sc)
            for f in ("nodes", "records", "descs"):
                assert arr[f].tobytes() == last["arrays"][f].tobytes(), (stage, f)
            got = lib.intersect(m.sc, rays.copy(), "1M")
            assert got.tobytes() == last["hits"].tobytes(), stage
        builders.append(st.builder)
        snap = m.snapshot()
        osc = oracle_scene(O, snap)
        want = osc.trace(rays.copy(), nthreads=8)
        ob = osc.bounds()
        osc.free()
        got = lib.intersect(m.sc, rays.copy(), "1M")
        lib.check(dev)
        rep = check_hits(O, snap, rays, want, got, stage)
        assert rep["hits"] > N_RAYS // 50, (stage, rep)
        occ = lib.occluded(m.sc, rays_of(rays), "1M")
        assert ((occ["tfar"] == -np.inf) == (got["geomID"] != INVALID)).all(), stage
        b = scene_bounds(lib, m.sc)
        if all(g[1] in (TRI, QUAD) for g in snap["geoms"]):
            assert np.array_equal(b, ob), (stage, b, ob)
        else:   # curve, point and instance boxes: as the golden tests of those kinds compare them
            assert np.allclose(b, ob, rtol=1e-6, atol=1e-6) and (b[:3] <= ob[:3]).all() and (b[3:] >= ob[3:]).all(), (stage, b, ob)
        if ref is not None:
            r, g = ref[f"c{k}"], got[rows]
            keep = np.ones(len(r), bool)
            # the reference's refit of a quad mesh does not follow its vertices (test_refit_quad_mesh_follows_its_vertices): rays that
            # meet a quad mesh it refitted are left out
            keep = ~np.isin(r["geomID"], snap["refit_quads"]) & ~np.isin(g["geomID"], snap["refit_quads"])
            check_hits(O, snap, rays[rows][keep], r[keep], g[keep], stage + " (reference)")
        if k % 8 == 4:   # derived caches: the batched interpolation table and the device traversable of this commit
            P = lib.interpolate_hits(m.sc, got.copy(), RTC_BUFFER_TYPE_VERTEX, 0, 3, want=("P",))["P"]
            lib.check(dev)
            child = m.children[0].sc if m.children else None
            hp, refused = host_interpolate(lib, dev, m.sc, child, got, RTC_BUFFER_TYPE_VERTEX, 0, 3)
            ok = (got["geomID"] != INVALID) & ~refused
            assert ok.sum() > 100 and (P[:, ok].view(np.uint32) == hp["P"][:, ok].view(np.uint32)).all(), stage
            compare_queries(lib, dev, devtrace, m.sc, rays, expect_hits=False)
        last.update(arrays=lib.scene_arrays(m.sc), hits=got)

    run_sequence(lib, dev, profile, seed, on_commit)
    missing = PATHS[profile] - set(builders)
    assert not missing, (profile, seed, "builder paths never reached", missing, builders)
    print(f"[scene_edits] {profile} seed {seed}: builders per commit {builders}")


# ---- 2: regressions -----------------------------------------------------------------------------------------------------
def two_level_scene(lib, dev, extra=()):
    """The two_level profile's start, committed once and then once more with one mesh moved (the per-mesh BVHs are built)."""
    m, _rng, _p = build_profile(lib, dev, "two_level", 5)
    for g in extra:
        m.attach(g)
    m.commit()
    move(m, 2)
    m.commit()
    assert lib.scene_stats(m.sc).builder == 3
    return m


def move(m, gid, d=0.2):
    g = m.geos[gid]
    g.v[:] += np.float32(d)
    g.update(RTC_BUFFER_TYPE_VERTEX)
    g.commit()


def check_against_oracle(lib, m, stage, rays=None):
    O = load_oracle()
    rays = profile_rays(3, 5.0) if rays is None else rays
    snap = m.snapshot()
    osc = oracle_scene(O, snap)
    want = osc.trace(rays.copy(), nthreads=8)
    osc.free()
    got = lib.intersect(m.sc, rays.copy(), "1M")
    lib.check(m.dev)
    check_hits(O, snap, rays, want, got, stage)
    return got


def test_mesh_moved_to_a_new_id_in_a_two_level_scene(b200):
    lib, dev = b200
    m = two_level_scene(lib, dev)
    try:
        m.attach(m.detach(3), 30)
        m.commit()
        assert lib.scene_stats(m.sc).builder == 3
        got = check_against_oracle(lib, m, "mesh 3 moved to ID 30")
        assert (got["geomID"] == 30).sum() > 20 and not (got["geomID"] == 3).any()
    finally:
        m.release()


def test_two_meshes_swap_ids_in_a_two_level_scene(b200):
    lib, dev = b200
    m = two_level_scene(lib, dev)
    try:
        a, b = m.detach(4), m.detach(6)
        m.attach(a, 6)
        m.attach(b, 4)
        m.commit()
        assert lib.scene_stats(m.sc).builder == 3
        check_against_oracle(lib, m, "meshes 4 and 6 swapped IDs")
    finally:
        m.release()


def test_mesh_moved_in_the_single_bvh_regime_then_two_level_again(b200):
    """The per-mesh BVHs are kept through single-BVH commits while the scene may return to the two-level path: one of them must
    not come back under its old ID."""
    lib, dev = b200
    m = two_level_scene(lib, dev)
    try:
        for gid in range(24):
            if gid != 3:
                move(m, gid, 0.05)
        m.attach(m.detach(3), 31)
        m.commit()
        assert lib.scene_stats(m.sc).builder != 3
        check_against_oracle(lib, m, "single BVH: everything moved, mesh 3 moved to ID 31")
        move(m, 7)
        m.commit()
        assert lib.scene_stats(m.sc).builder == 3
        got = check_against_oracle(lib, m, "two-level again")
        assert (got["geomID"] == 31).sum() > 20
    finally:
        m.release()


def test_one_geometry_under_two_ids(b200):
    """The reference's Scene::bind accepts one geometry under two IDs of one scene (scene.cpp:717-741).  Both copies are hit at the
    oracle's distance with an ID of the pair, and 20 two-level commits leave device memory flat."""
    import torch
    lib, dev = b200
    m = two_level_scene(lib, dev)
    try:
        big = m.geos[24]
        m.attach(big, 30)
        m.commit()
        rays = profile_rays(4, 5.0)
        O = load_oracle()

        def check(stage):
            osc = oracle_scene(O, m.snapshot())
            want = osc.trace(rays.copy(), nthreads=8)
            osc.free()
            pair = np.isin(want["geomID"], [24, 30])
            got = lib.intersect(m.sc, rays.copy(), "1M")
            lib.check(dev)
            assert np.isin(got["geomID"][pair], [24, 30]).all(), stage
            assert (np.abs(got["tfar"][pair] - want["tfar"][pair]) <= TOL * np.abs(want["tfar"][pair])).all(), stage
            rest = ~pair
            rep = compare_hits(want[rest], got[rest], TOL)
            assert rep["id_mismatch"] == 0 and rep["hit_miss_disagree"] == 0, (stage, rep)
            assert pair.sum() > 1000, stage
        check("attached under 24 and 30")
        move(m, 2)
        m.commit()
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        free0 = torch.cuda.mem_get_info()[0]
        for i in range(20):
            move(m, 2 + i % 3, 0.01)
            m.commit()
            assert lib.scene_stats(m.sc).builder == 3
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        free1 = torch.cuda.mem_get_info()[0]
        assert free0 - free1 < 32 << 20, (free0, free1)
        check("after 20 commits")
    finally:
        m.release()


def aimed_rays(v, t, rows, n=8):
    """Rays from outside a sphere-like mesh towards the centroid of each of `rows`' triangles."""
    c = v[t[rows]].mean(1).astype(np.float64)
    org = np.repeat(c * 3.0, n, 0) + np.random.RandomState(1).normal(scale=1e-3, size=(len(rows) * n, 3))
    return make_rayhits(org, np.repeat(c, n, 0) - org)


REFIT_V, REFIT_T = scenes.triangle_sphere(40)
BROKEN_ROWS = np.array([100, 1700, 2900])


def refit_case(L, dev, case, trace):
    """The REFIT cases on one library: one REFIT mesh committed with invalid triangles, fixed, committed again.  'index*': a
    DYNAMIC scene, three triangles holding an out-of-range index, fixed by an index-buffer update; 'nan*': one vertex NaN, fixed by
    a vertex update only, in a scene that is not DYNAMIC ('nan_static') or is ('nan_dynamic*').  '_low': scene quality LOW, else
    MEDIUM.  Returns trace(scene) after the fix, and the builder of the last commit (None on the reference)."""
    t = REFIT_T.copy()
    v = REFIT_V.copy()
    if case.startswith("index"):
        t[BROKEN_ROWS, 1] = len(v) + 3
    else:
        v[REFIT_T[BROKEN_ROWS[0], 0]] = np.nan
    sc = L.rtcNewScene(dev)
    L.rtcSetSceneFlags(sc, RTC_SCENE_FLAG_NONE if case == "nan_static" else RTC_SCENE_FLAG_DYNAMIC)
    L.rtcSetSceneBuildQuality(sc, RTC_BUILD_QUALITY_LOW if case.endswith("_low") else RTC_BUILD_QUALITY_MEDIUM)
    g = Geo(L, dev, TRI, v, t, quality=RTC_BUILD_QUALITY_REFIT)
    L.rtcAttachGeometryByID(sc, g.h, 0)
    L.rtcCommitScene(sc)
    L.check(dev)
    if case.startswith("index"):
        g.idx[:] = REFIT_T
        g.update(RTC_BUFFER_TYPE_INDEX)
    else:
        g.v[:] = REFIT_V
        g.update(RTC_BUFFER_TYPE_VERTEX)
    g.commit()
    L.rtcCommitScene(sc)
    L.check(dev)
    out = trace(sc)
    builder = L.scene_stats(sc).builder if L.is_b200 else None
    L.rtcReleaseGeometry(g.h)
    L.rtcReleaseScene(sc)
    return out, builder


def refit_rows(case):
    """The triangles the REFIT case makes invalid at the first commit."""
    return BROKEN_ROWS if case.startswith("index") else np.nonzero((REFIT_T == REFIT_T[BROKEN_ROWS[0], 0]).any(1))[0]


def refit_against_the_reference(lib, dev, case):
    """This library's and the reference's hits for rays aimed at the fixed triangles of a REFIT case (the reference live where
    oracle/_ref is built, else its stored answers); the ids must be equal and t within TOL.  Returns (hits, reference hits, builder)."""
    rays = aimed_rays(REFIT_V, REFIT_T, refit_rows(case))

    def run(R):
        rd = R.new_device(None)
        out, _ = refit_case(R, rd, case, lambda sc: api_trace_mt(R, sc, rays.copy(), 1))
        R.rtcReleaseDevice(rd)
        return {"hits": out}
    ref = reference_outputs(f"scene_edits_refit_{case}", run, {"hits": rays})[0]["hits"]
    got, builder = refit_case(lib, dev, case, lambda sc: lib.intersect(sc, rays.copy(), "1M"))
    assert (got["geomID"] == ref["geomID"]).all() and (got["primID"] == ref["primID"]).all(), \
        (case, builder, got[["geomID", "primID"]], ref[["geomID", "primID"]])
    hit = ref["geomID"] != INVALID
    assert (np.abs(got["tfar"][hit] - ref["tfar"][hit]) <= TOL * ref["tfar"][hit]).all(), case
    return got, ref, builder


def on_fixed(hits, case):
    return np.isin(hits["primID"], refit_rows(case)) & (hits["geomID"] == 0)


@pytest.mark.parametrize("case", ["index", "index_low"])
def test_refit_mesh_hit_after_its_indices_are_fixed(b200, case):
    """Single BVH: a REFIT commit keeps only the primitives valid at the last build, so new indices must rebuild, as the reference
    does (bvh_refit.cpp:184-192), at MEDIUM and at LOW quality."""
    lib, dev = b200
    got, ref, builder = refit_against_the_reference(lib, dev, case)
    assert on_fixed(ref, case).all() and builder != 2, builder


def test_two_level_refit_mesh_hit_after_its_indices_are_fixed(b200):
    lib, dev = b200
    m, _rng, _p = build_profile(lib, dev, "two_level", 5)
    try:
        g = m.geos[5]                                   # a REFIT mesh
        rows = np.array([len(g.idx) // 4, len(g.idx) // 2, 3 * len(g.idx) // 4])
        orig = g.idx[rows].copy()
        g.idx[rows, 2] = len(g.v) + 1
        g.update(RTC_BUFFER_TYPE_INDEX)
        g.commit()
        m.commit()
        move(m, 2)
        m.commit()
        assert lib.scene_stats(m.sc).builder == 3
        g.idx[rows] = orig
        g.update(RTC_BUFFER_TYPE_INDEX)
        g.commit()
        m.commit()
        assert lib.scene_stats(m.sc).builder == 3
        c = g.v[g.idx[rows]].mean(1)
        n = (c - g.v.mean(0)) / np.linalg.norm(c - g.v.mean(0), axis=1, keepdims=True)
        rays = make_rayhits(c + n * np.float32(0.05), -n, tfar=0.1)     # from just outside, towards the triangle's centroid
        check_against_oracle(lib, m, "two-level REFIT mesh with fixed indices")
        got = check_against_oracle(lib, m, "two-level REFIT mesh with fixed indices, rays at its fixed triangles", rays)
        assert (got["geomID"] == 5).all() and (got["primID"] == rows).all(), got[["geomID", "primID"]]
    finally:
        m.release()


@pytest.mark.parametrize("case", ["nan_static", "nan_dynamic", "nan_dynamic_low"])
def test_refit_mesh_with_a_fixed_nan_vertex_as_the_reference(b200, case):
    """A triangle with a NaN vertex at the first build, the vertex fixed by a vertex update only.  The reference refits only a
    DYNAMIC scene of LOW quality (scene.cpp:158-194) and its refit keeps the primitives of the last build, which dropped the NaN
    triangle (scene_triangle_mesh.h:195-207): there the fixed triangle stays unhittable (the rays pass through the hole to the far
    side).  Any other scene it rebuilds and hits the triangle.  This library refits in the first case and rebuilds in the others."""
    lib, dev = b200
    got, ref, builder = refit_against_the_reference(lib, dev, case)
    if case == "nan_dynamic_low":
        assert builder == 2 and not on_fixed(ref, case).any() and (ref["geomID"] == 0).all(), builder
    else:
        assert builder == 1 and on_fixed(ref, case).all(), builder


def test_refit_quad_mesh_follows_its_vertices(b200):
    """A REFIT quad mesh in a DYNAMIC scene of LOW quality, scaled three times: each refit gives the hits of a build from scratch.
    The reference's refit there does not follow the quads' new vertices (its answers, pinned here, differ from a scene built from
    scratch), so the reference comparison of the edit sequences leaves out rays that meet such a mesh."""
    lib, dev = b200
    O = load_oracle()
    rays = profile_rays(5, 2.0)
    scales = (np.float32(1.3), np.float32([1.2, 0.8, 1.1]), np.float32(0.7))

    def run(L, dev, on_step):
        m = Model(L, dev, RTC_SCENE_FLAG_DYNAMIC, RTC_BUILD_QUALITY_LOW)
        v, q = quad_sphere(12)
        g = Geo(L, dev, QUAD, v, q, quality=RTC_BUILD_QUALITY_REFIT)
        m.attach(g, 0)
        try:
            m.commit()
            for k, sc in enumerate(scales):
                g.v[:] = (g.v * sc).astype(np.float32)
                g.update(RTC_BUFFER_TYPE_VERTEX)
                g.commit()
                m.commit()
                on_step(k, m)
        finally:
            m.release()

    def reference(R):
        rd = R.new_device(None)
        out = {}
        run(R, rd, lambda k, m: out.__setitem__(f"s{k}", api_trace_mt(R, m.sc, rays.copy(), 8)))
        R.rtcReleaseDevice(rd)
        return out
    ref, rows = reference_outputs("scene_edits_refit_quads_low", reference, {f"s{k}": rays for k in range(len(scales))}, stride=10)

    def ours(k, m):
        assert lib.scene_stats(m.sc).builder == 2, k
        check_against_oracle(lib, m, f"quad mesh scaled, step {k}", rays)
        osc = oracle_scene(O, m.snapshot())
        want = osc.trace(rays.copy(), nthreads=8)[rows]
        osc.free()
        r = ref[f"s{k}"]
        assert ((r["geomID"] != want["geomID"]) | (r["primID"] != want["primID"])).sum() > 10, k
    run(lib, dev, ours)


# ---- 3: the reference's enable / disable / detach tests ------------------------------------------------------------------
def four_kinds(L, dev, sc):
    """verify.cpp:1659-1662 with a point set where the reference uses a subdivision sphere: a triangle sphere at (-1, 0, -1), a quad
    sphere at (-1, 0, +1), a sphere point at (+1, 0, -1) and a round linear curve across (+1, 0, +1)."""
    v, t = scenes.triangle_sphere(50, center=(-1.0, 0.0, -1.0))
    vq, q = quad_sphere(25, (-1.0, 0.0, 1.0))
    geos = [Geo(L, dev, TRI, v, t), Geo(L, dev, QUAD, vq, q), Geo(L, dev, POINTS, np.float32([[1, 0, -1, 0.5]])),
            Geo(L, dev, CURVE, np.float32([[0.5, 0, 1, 0.1], [1.5, 0, 1, 0.1]]), np.uint32([0]))]
    ids = [L.rtcAttachGeometry(sc, g.h) for g in geos]
    assert ids == [0, 1, 2, 3]
    return geos


def four_rays():
    return make_rayhits([[-1, 10, -1], [-1, 10, 1], [1, 10, -1], [1, 10, 1]], np.tile([[0, -1, 0]], (4, 1)))


SCENE_FLAGS = {"none": RTC_SCENE_FLAG_NONE, "dynamic": RTC_SCENE_FLAG_DYNAMIC, "robust": RTC_SCENE_FLAG_ROBUST}


@pytest.mark.parametrize("flags", list(SCENE_FLAGS))
def test_enable_disable_geometry(b200, flags):
    """EnableDisableGeometryTest (verify.cpp:1645-1690): 17 commits through every combination of enabled geometries."""
    lib, dev = b200
    sc = lib.rtcNewScene(dev)
    lib.rtcSetSceneFlags(sc, SCENE_FLAGS[flags])
    geos = four_kinds(lib, dev, sc)
    for i in range(17):
        on = [bool(i & (1 << k)) for k in range(4)]
        for g, e in zip(geos, on):
            (lib.rtcEnableGeometry if e else lib.rtcDisableGeometry)(g.h)
        lib.rtcCommitScene(sc)
        lib.check(dev)
        for mode in ("1", "1M"):
            got = lib.intersect(sc, four_rays(), mode)
            assert list(got["geomID"]) == [k if on[k] else INVALID for k in range(4)], (i, mode, got["geomID"])
    for g in geos:
        lib.rtcReleaseGeometry(g.h)
    lib.rtcReleaseScene(sc)


@pytest.mark.parametrize("flags", list(SCENE_FLAGS))
def test_disable_and_detach_geometry(b200, flags):
    """DisableAndDetachGeometryTest (verify.cpp:1694-1760): one geometry after the other is disabled, detached and the scene
    committed; the others are still hit."""
    lib, dev = b200
    sc = lib.rtcNewScene(dev)
    lib.rtcSetSceneFlags(sc, SCENE_FLAGS[flags])
    geos = four_kinds(lib, dev, sc)
    for g in geos:
        lib.rtcEnableGeometry(g.h)
    lib.rtcCommitScene(sc)
    for i in range(5):
        for mode in ("1", "1M"):
            got = lib.intersect(sc, four_rays(), mode)
            assert list(got["geomID"]) == [k if i <= k else INVALID for k in range(4)], (i, mode, got["geomID"])
        if i < 4:
            lib.rtcDisableGeometry(geos[i].h)
            lib.rtcDetachGeometry(sc, i)
            lib.rtcCommitScene(sc)
            lib.check(dev)
    for g in geos:
        lib.rtcReleaseGeometry(g.h)
    lib.rtcReleaseScene(sc)
