"""Filter-callback scenarios shared by tests/golden/make_golden.py (run on the unmodified reference, outputs committed as
tests/golden/filters.npz) and tests/test_filter.py (run on the CUDA library through the same C-ABI and compared).

The callbacks are Python functions behind ctypes (rtc.FILTER_FUNCTION) that handle any N, as the reference's own test
callback does (tutorials/verify/verify.cpp:2771-2786): the reference calls them with N = 1 or the packet width, the CUDA
library always with N = 1.  The accept / reject rule is a pure function of the candidate's ids, so the final hit of a ray
does not depend on the order in which a traversal meets the candidates."""
import numpy as np

from embree_b200 import rtc
from embree_b200.rtc import FILTER_FUNCTION, RayQueryContext, filter_lane


def rejects(geomID, primID, instID=0xFFFFFFFF):
    h = (primID * 2654435761 + geomID * 40503 + (0 if instID == 0xFFFFFFFF else (instID + 1) * 97)) & 0xFFFFFFFF
    return ((h >> 7) & 3) == 0          # one candidate in four


class Recorder:
    """A filter callback + what it saw: (ray id, geomID, primID, instID, context instID, tfar, userPtr) per active lane."""

    def __init__(self, rule=rejects):
        self.calls = []
        self.rule = rule
        self.errors = []
        self.fn = FILTER_FUNCTION(self._call)

    def _call(self, args):
        try:
            a = args.contents
            for lane in range(a.N):
                if a.valid[lane] != -1:
                    continue
                f = filter_lane(args, lane)
                ctx_inst = a.context.contents.instID if a.context else None
                self.calls.append((f["id"], f["geomID"], f["primID"], f["instID"], ctx_inst, f["tfar"], a.geometryUserPtr))
                if self.rule(f["geomID"], f["primID"], f["instID"]):
                    a.valid[lane] = 0
        except Exception as e:   # an exception must not unwind through the C caller
            self.errors.append(repr(e))


def number_rays(rayhits):
    rayhits["id"] = np.arange(len(rayhits), dtype=np.uint32)
    return rayhits


def build(lib, dev, meshes, setup):
    """Scene of `meshes` [(v, t, geomID, mask)]; setup(lib, geomID, geometry handle) installs the callbacks."""
    sc = lib.rtcNewScene(dev)
    keep = []
    for (v, t, gid, mask) in meshes:
        _, k = lib.add_triangle_mesh(dev, sc, v, t, mask=mask, geom_id=gid)
        keep.append(k)
        setup(lib, gid, lib.rtcGetGeometry(sc, gid))
    lib.rtcCommitScene(sc)
    lib.check(dev)
    return sc, keep


CONFIGS = ["geometry", "argument_all", "argument_enabled"]


def run_config(lib, dev, meshes, rayhits, config, mode="1"):
    """One configuration on one library: returns (intersect_out, occluded_out, intersect Recorder, occluded Recorder).
      geometry         : geometry 0 carries an intersect and an occluded filter (rtcSetGeometry*FilterFunction), user data 123
      argument_all     : the arguments' filter with RTC_RAY_QUERY_FLAG_INVOKE_ARGUMENT_FILTER -> every geometry
      argument_enabled : the arguments' filter, enabled on the LAST geometry only (rtcSetGeometryEnableFilterFunctionFromArguments)"""
    ri, ro = Recorder(), Recorder()
    last = max(g for (_v, _t, g, _m) in meshes)

    def setup(L, gid, g):
        if config == "geometry" and gid == 0:
            L.rtcSetGeometryUserData(g, 123)
            L.rtcSetGeometryIntersectFilterFunction(g, ri.fn)
            L.rtcSetGeometryOccludedFilterFunction(g, ro.fn)
        if config == "argument_enabled" and gid == last:
            L.rtcSetGeometryEnableFilterFunctionFromArguments(g, True)
    sc, keep = build(lib, dev, meshes, setup)
    ctx = RayQueryContext(0xFFFFFFFF, 0xFFFFFFFF)
    if config == "geometry":
        ai = ao = lib.args(context=ctx)
    else:
        inv = config == "argument_all"
        ai = lib.args(filter=ri.fn, invoke_argument_filter=inv, context=ctx)
        ao = lib.args(filter=ro.fn, invoke_argument_filter=inv, context=ctx)
    out_i = lib.intersect(sc, number_rays(rayhits.copy()), mode, args=ai)
    out_o = lib.occluded(sc, rtc.rays_of(number_rays(rayhits.copy())), mode, args=ao)
    lib.check(dev)
    lib.rtcReleaseScene(sc)
    assert not ri.errors and not ro.errors, (ri.errors, ro.errors)
    return out_i, out_o, ri, ro


# ---- tutorials/hair_geometry: shadow rays through hair with a STATEFUL argument filter -------------------------------------
import ctypes as C  # noqa: E402


class HairShadowContext(C.Structure):
    """RayQueryContext of tutorials/common/tutorial/tutorial_device.h: the RTCRayQueryContext first, then the tutorial's
    own fields -- here the transparency the occlusion filter accumulates (hair_geometry_device.cpp:208-238)."""
    _fields_ = [("context", RayQueryContext), ("T", C.c_float * 3)]


HAIR_KT = (0.8 * 0.8, 0.8 * 0.57, 0.8 * 0.32)     # TutorialData: hair_Kt = 0.8 * hair_K


def hair_shadow_filter():
    """occlusionFilter of hair_geometry_device.cpp:208-238: every hair multiplies the ray's transparency by Kt and is rejected
    (the ray goes on) until the transparency drops below 2 %."""
    def cb(args):
        a = args.contents
        if a.valid[0] == 0:
            return
        ctx = C.cast(a.context, C.POINTER(HairShadowContext)).contents
        for k in range(3):
            ctx.T[k] = C.c_float(HAIR_KT[k] * ctx.T[k]).value
        if max(ctx.T[0], ctx.T[1], ctx.T[2]) > 0.02:
            a.valid[0] = 0
    return FILTER_FUNCTION(cb)


def hair_scene():
    """A small fur ball of flat Bezier curves around an (unfiltered) triangle sphere + shadow rays from its surroundings."""
    from embree_b200 import scenes
    cv, ci, _tg = scenes.cubic_hair(600, "bezier", seed=41, radius=0.8, step=0.06, width=0.012)
    v, t = scenes.triangle_sphere(12)
    v = (v * np.float32(0.8)).astype(np.float32)
    rng = np.random.RandomState(43)
    org = rng.normal(size=(1536, 3)).astype(np.float32)
    org = org / np.linalg.norm(org, axis=1, keepdims=True) * rng.uniform(1.05, 1.6, (1536, 1)).astype(np.float32)
    d = (-org + rng.normal(scale=0.55, size=org.shape)).astype(np.float32)      # towards the ball, many graze only its fur
    return (v, t), (cv, ci), rtc.rays_of(rtc.make_rayhits(org, d, tnear=1e-4))


def run_hair_shadows(lib, dev, single=True):
    """occluded() of hair_geometry_device.cpp:240-262 for every ray: returns (transparency[n,3], occluded[n])."""
    (v, t), (cv, ci), rays = hair_scene()
    sc = lib.rtcNewScene(dev)
    keep = [lib.add_triangle_mesh(dev, sc, v, t, geom_id=0)[1], lib.add_flat_cubic_curves(dev, sc, cv, ci, "bezier", geom_id=1)[1]]
    lib.rtcSetGeometryEnableFilterFunctionFromArguments(lib.rtcGetGeometry(sc, 1), True)   # convertHairSet: hair only
    lib.rtcCommitScene(sc)
    lib.check(dev)
    fn = hair_shadow_filter()
    T = np.ones((len(rays), 3), np.float32)
    occ = np.zeros(len(rays), bool)
    base, st = rays.ctypes.data, rays.dtype.itemsize
    for i in range(len(rays)):
        ctx = HairShadowContext()
        ctx.context.instID = ctx.context.instPrimID = 0xFFFFFFFF
        ctx.T[0] = ctx.T[1] = ctx.T[2] = 1.0
        a = lib.args(filter=fn, context=ctx)
        lib.rtcOccluded1(sc, C.c_void_p(base + i * st), C.byref(a))
        occ[i] = rays["tfar"][i] < 0
        T[i] = (0.0, 0.0, 0.0) if occ[i] else (ctx.T[0], ctx.T[1], ctx.T[2])
    lib.check(dev)
    lib.rtcReleaseScene(sc)
    return T, occ
