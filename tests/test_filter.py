"""Filter callbacks (SURVEY 8 a6 / a15 / a16): geometry filters, the arguments' filter, RTC_RAY_QUERY_FLAG_INVOKE_ARGUMENT_FILTER,
rtcSetGeometryEnableFilterFunctionFromArguments -- through every host-pointer entry point of the CUDA library, against
golden outputs of the unmodified reference (tests/golden/filters.npz, generator tests/golden/make_golden.py filters) and,
when oracle/_ref is built, the reference run side by side with the same Python callbacks.
Reference: kernels/geometry/filter.h:15-84, intersector_epilog.h:264-280,347-361; test model tutorials/verify/verify.cpp:2762-2838."""
import ctypes as C
import os

import numpy as np
import pytest

from embree_b200 import rtc, scenes
from embree_b200.rtc import FILTER_FUNCTION, RayQueryContext, make_rayhits, rays_of
from tests import filter_cases as fc
from tests.conftest import ROOT, load_golden, load_golden_instances
from tests.parity import compare_hits, load_reference, reference_outputs

pytestmark = pytest.mark.gpu
MODES = ["1", "4", "8", "16", "1M", "4M", "8M", "16M"]


def _golden(cfg):
    from embree_b200.rtc import RAYHIT_DTYPE, RAY_DTYPE, aligned_empty
    z = np.load(os.path.join(ROOT, "tests", "golden", "filters.npz"))

    def rec(a, dt):
        out = aligned_empty(a.shape[0], dt)
        out.view(np.uint8).reshape(a.shape)[:] = a
        return out
    return rec(z[cfg + "_intersect"], RAYHIT_DTYPE), rec(z[cfg + "_occluded"], RAY_DTYPE)


@pytest.mark.parametrize("cfg", fc.CONFIGS)
def test_filters_match_the_reference(b200, cfg):
    lib, dev = b200
    meshes, rin, _wi, _wo, _b = load_golden("cube_ground")
    want_i, want_o = _golden(cfg)
    for mode in MODES:
        got_i, got_o, ri, ro = fc.run_config(lib, dev, meshes, rin, cfg, mode)
        rep = compare_hits(want_i, got_i, 1e-4, meshes=meshes)
        assert rep["id_mismatch"] == 0 and rep["hit_miss_disagree"] == 0 and rep["tie"] <= 2, (cfg, mode, rep)
        assert rep["max_rel_t"] <= 1e-4 and rep["max_abs_uv"] <= 1e-4 and rep["miss_untouched"], (cfg, mode, rep)
        assert (got_o["tfar"].view(np.uint32) == want_o["tfar"].view(np.uint32)).all(), (cfg, mode)
        for rec in (ri, ro):
            # every candidate is offered at most once per ray, and only candidates the configuration covers
            seen = [(c[0], c[1], c[2]) for c in rec.calls]
            assert len(seen) == len(set(seen)), (cfg, mode)
            if cfg == "geometry":
                assert all(c[1] == 0 and c[6] == 123 for c in rec.calls)
            if cfg == "argument_enabled":
                assert all(c[1] == max(m[2] for m in meshes) for c in rec.calls)
            assert all(c[4] == 0xFFFFFFFF for c in rec.calls)            # not instanced: context instID stays invalid
        # the accepted hit is what the callback saw last for that ray (tfar = candidate distance)
        last = {}
        for c in ri.calls:
            last[c[0]] = c
        for i in np.nonzero(got_i["geomID"] != 0xFFFFFFFF)[0]:
            if int(i) in last and not fc.rejects(last[int(i)][1], last[int(i)][2]):
                assert last[int(i)][2] == got_i["primID"][i] and np.float32(last[int(i)][5]) == got_i["tfar"][i]
    ref = load_reference()
    if ref is not None:   # side by side with the live reference, same callbacks, single-ray mode
        rdev = ref.new_device(None)
        ref_i, ref_o, _a, _b2 = fc.run_config(ref, rdev, meshes, rin, cfg, "1")
        ref.rtcReleaseDevice(rdev)
        assert (ref_i["primID"] == want_i["primID"]).all() and (ref_o["tfar"].view(np.uint32) == want_o["tfar"].view(np.uint32)).all()


def test_intersection_filter_test_of_verify(b200):
    """IntersectionFilterTest (verify.cpp:2762-2838): a 4x4 plane, the geometry filter rejects primID & 2."""
    lib, dev = b200
    v, t = scenes.triangle_plane((-0.75, -0.25, -10.0), (4, 0, 0), (0, 4, 0), 4, 4)

    def cb(args):
        a = args.contents
        if a.geometryUserPtr != 123:
            return
        for lane in range(a.N):
            if a.valid[lane] == -1 and (rtc.filter_lane(args, lane)["primID"] & 2):
                a.valid[lane] = 0
    fn = FILTER_FUNCTION(cb)
    sc = lib.rtcNewScene(dev)
    gid, keep = lib.add_triangle_mesh(dev, sc, v, t)
    g = lib.rtcGetGeometry(sc, gid)
    lib.rtcSetGeometryUserData(g, 123)
    lib.rtcSetGeometryIntersectFilterFunction(g, fn)
    lib.rtcSetGeometryOccludedFilterFunction(g, fn)
    lib.rtcCommitScene(sc)
    lib.check(dev)
    org = np.array([[ix, iy, 0.0] for iy in range(4) for ix in range(4)], np.float32)
    rays = make_rayhits(org, np.tile([[0, 0, -1]], (16, 1)))
    for mode in MODES:
        out = lib.intersect(sc, rays.copy(), mode)
        occ = lib.occluded(sc, rays_of(rays), mode)
        for i in range(16):
            prim = 2 * i
            if prim & 2:
                assert out["geomID"][i] == 0xFFFFFFFF and occ["tfar"][i] != -np.inf, (mode, i)
            else:
                assert out["geomID"][i] == 0 and occ["tfar"][i] == -np.inf, (mode, i)
    # removing the callbacks restores the plain traversal without a re-commit (geometry.cpp:142-156 keeps no commit state)
    lib.rtcSetGeometryIntersectFilterFunction(g, None)
    lib.rtcSetGeometryOccludedFilterFunction(g, None)
    out = lib.intersect(sc, rays.copy(), "1M")
    assert (out["geomID"] == 0).all()
    lib.check(dev)
    lib.rtcReleaseScene(sc)


def test_filter_on_instanced_geometry(b200):
    """The CHILD geometry's filter runs for hits through an instance; the callback sees the instance id in the hit and in
    the context (instance_intersector.cpp:15-38 pushes it), and the result equals the reference's."""
    lib, dev = b200
    g = load_golden_instances()

    def run(L, d):
        rec = fc.Recorder()
        child = L.rtcNewScene(d)
        keep = []
        for (v, t, gid, mask) in g["child"]:
            _, k = L.add_triangle_mesh(d, child, v, t, mask=mask, geom_id=gid)
            keep.append(k)
            if gid == 0:
                L.rtcSetGeometryIntersectFilterFunction(L.rtcGetGeometry(child, gid), rec.fn)
        L.rtcCommitScene(child)
        top = L.rtcNewScene(d)
        for (v, t, gid, mask) in g["top"]:
            _, k = L.add_triangle_mesh(d, top, v, t, mask=mask, geom_id=gid)
            keep.append(k)
        for i, xf in enumerate(g["xfms"]):
            L.add_instance(d, top, child, xf, mask=int(g["inst_masks"][i]), geom_id=g["first_inst"] + i)
        L.rtcCommitScene(top)
        L.check(d)
        ctx = RayQueryContext(0xFFFFFFFF, 0xFFFFFFFF)
        out = L.intersect(top, fc.number_rays(g["rays_in"].copy()), "1", args=L.args(context=ctx))
        L.check(d)
        L.rtcReleaseScene(top)
        L.rtcReleaseScene(child)
        assert not rec.errors, rec.errors
        return out, rec
    got, rec = run(lib, dev)
    assert len(rec.calls) > 100
    assert all(c[1] == 0 and c[3] != 0xFFFFFFFF and c[4] == c[3] for c in rec.calls)   # child geomID 0, instID in hit == context

    def run_reference(R):
        rdev = R.new_device(None)
        want, rrec = run(R, rdev)
        R.rtcReleaseDevice(rdev)
        assert all(c[4] == c[3] for c in rrec.calls)
        return {"hits": want}
    want = reference_outputs("filter_instanced", run_reference, {"hits": fc.number_rays(g["rays_in"].copy())})[0]["hits"]
    rep = compare_hits(want, got, 1e-4)
    assert rep["id_mismatch"] == 0 and rep["hit_miss_disagree"] == 0 and rep["tie"] <= 4, rep


def test_device_entry_points_refuse_filters(b200):
    """A host callback cannot run inside a device-pointer launch: RTC_ERROR_INVALID_OPERATION, nothing traced."""
    import torch
    lib, dev = b200
    v, t = scenes.triangle_sphere(11)
    sc = lib.rtcNewScene(dev)
    _, keep = lib.add_triangle_mesh(dev, sc, v, t)
    lib.rtcCommitScene(sc)
    rec = fc.Recorder()
    rays = scenes.as_numpy_rayhits(scenes.incoherent_rays_reference(64))
    d = torch.from_numpy(rays.view(np.uint8).reshape(-1, 96).copy()).cuda()
    a = lib.args(filter=rec.fn, invoke_argument_filter=True)
    lib.rtcb200Intersect1MDevice(sc, C.c_void_p(d.data_ptr()), 64, C.byref(a), None)
    torch.cuda.synchronize()
    assert lib.rtcGetDeviceError(dev) == rtc.RTC_ERROR_INVALID_OPERATION
    assert (d.cpu().numpy().view(rtc.RAYHIT_DTYPE)["geomID"] == 0xFFFFFFFF).all() and not rec.calls
    # the host-pointer form of the same call runs the callback
    out = lib.intersect(sc, fc.number_rays(rays.copy()), "1M", args=a)
    assert len(rec.calls) > 0 and lib.rtcGetDeviceError(dev) == rtc.RTC_ERROR_NONE
    want = [not fc.rejects(0, int(p)) for p in out["primID"][out["geomID"] != 0xFFFFFFFF]]
    assert all(want)
    lib.rtcReleaseScene(sc)


def test_hair_shadow_rays_with_transparency_filter(b200):
    """The shadow rays of tutorials/hair_geometry (hair_geometry_device.cpp:208-262): a stateful occlusion filter passed in the
    arguments and enabled on the hair geometry accumulates the transparency of every hair along the ray and lets the ray
    through until less than 2 % is left.  Transparency and occlusion per ray equal the reference's (golden; the product is
    taken in a different order, hence the 1e-5)."""
    lib, dev = b200
    z = np.load(os.path.join(ROOT, "tests", "golden", "filters.npz"))
    T, occ = fc.run_hair_shadows(lib, dev)
    assert (occ == z["hair_occluded"]).all()
    assert np.allclose(T, z["hair_T"], rtol=1e-5, atol=1e-7)
    assert occ.mean() > 0.05 and ((T < 1).any(1) & ~occ).mean() > 0.1
