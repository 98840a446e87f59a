"""Commits that fail after some kept BVHs were rebuilt.  The BVHs the failed commit rebuilt stay with the scene, so the next commit
neither loses their memory nor builds them again, and it traces them as they are now, not the copies the scene's arrays held before.
Both commit paths that keep BVHs across commits are covered: two-level scenes (one BVH per mesh) and instance traversal (one BVH per
instanced scene)."""
import re

import numpy as np
import pytest

from embree_b200 import scenes
from embree_b200.rtc import (RTC_BUFFER_TYPE_INDEX, RTC_BUFFER_TYPE_VERTEX, RTC_ERROR_INVALID_OPERATION, RTC_FORMAT_UINT3,
                             RTC_GEOMETRY_TYPE_TRIANGLE, _ptr, make_rayhits)
from tests.test_gpu_parity import build_scene
from tests.test_instance_traversal import same_but_ties
from tests.test_scene_edits import check_against_oracle, move, two_level_scene
from tests.test_trace_schedules import tuning

pytestmark = pytest.mark.gpu
TWO_LEVEL_LOG = re.compile(r"commit \(two-level\): (\d+) meshes, (\d+) rebuilt or refitted")


def no_vertex_buffer(lib, dev, idx):
    """A committed triangle geometry with an index buffer and no vertex buffer: a scene commit that uploads it fails."""
    g = lib.rtcNewGeometry(dev, RTC_GEOMETRY_TYPE_TRIANGLE)
    lib.rtcSetSharedGeometryBuffer(g, RTC_BUFFER_TYPE_INDEX, 0, RTC_FORMAT_UINT3, _ptr(idx), 0, 12, len(idx))
    lib.rtcCommitGeometry(g)
    return g


def test_two_level_commit_failing_after_a_rebuild(b200, capfd):
    """Mesh 3 moves and is rebuilt, then the geometry at the highest ID fails the upload.  The commit after that geometry is
    detached rebuilds nothing, traces mesh 3 at its new position, and ten such failed commits leave device memory flat."""
    import torch
    lib, _ = b200
    dev = lib.new_device("verbose=2")
    m = two_level_scene(lib, dev)    # 24 small meshes and one of ~250 k triangles: a commit that changes two small meshes is two-level
    idx = np.arange(12, dtype=np.uint32).reshape(4, 3)
    bad = no_vertex_buffer(lib, dev, idx)
    bad_id = max(m.geos) + 1

    def failed_commit(d):
        move(m, 3, d)
        lib.rtcAttachGeometryByID(m.sc, bad, bad_id)
        lib.rtcCommitScene(m.sc)
        assert lib.rtcGetDeviceError(dev) == RTC_ERROR_INVALID_OPERATION
        lib.rtcDetachGeometry(m.sc, bad_id)

    try:
        failed_commit(0.3)
        capfd.readouterr()
        m.commit()
        log = capfd.readouterr().err
        assert lib.scene_stats(m.sc).builder == 3, log
        found = TWO_LEVEL_LOG.findall(log)
        assert len(found) == 1 and int(found[0][1]) <= 1, log
        got = check_against_oracle(lib, m, "after a failed two-level commit")
        assert (got["geomID"] == 3).sum() > 20

        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        free0 = torch.cuda.mem_get_info()[0]
        for i in range(10):
            failed_commit(0.01)
        m.commit()
        assert lib.scene_stats(m.sc).builder == 3
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        free1 = torch.cuda.mem_get_info()[0]
        assert free0 - free1 < 32 << 20, (free0, free1)
        check_against_oracle(lib, m, "after ten failed two-level commits")
    finally:
        lib.rtcReleaseGeometry(bad)
        m.release()
        lib.rtcReleaseDevice(dev)


def test_instance_traversal_commit_failing_after_a_rebuild(b200, capfd):
    """Instanced scene 1 is re-committed, so the next commit rebuilds its BVH; an instance of a scene that holds an instance, at a
    higher geomID, then fails that commit.  Once it is removed, the commit rebuilds nothing and traces what flattening traces."""
    lib, _ = b200
    dev = lib.new_device("verbose=2")
    v, t = scenes.triangle_sphere(12)
    child, keep = build_scene(lib, dev, [(v, t, 0, 0xFFFFFFFF)])
    xfms = [np.array([1, 0, 0, 0, 1, 0, 0, 0, 1, 3.0 * k, 0.5 * (k % 3), 10], np.float32) for k in range(8)]
    tops = []
    for _ in range(2):                              # the scene under test, then the same instances flattened
        top = lib.rtcNewScene(dev)
        for k, x in enumerate(xfms):
            lib.add_instance(dev, top, child, x, geom_id=k)
        tops.append(top)
    inst, flat = tops
    nested = lib.rtcNewScene(dev)
    lib.add_instance(dev, nested, child, xfms[0])
    lib.rtcCommitScene(nested)
    lib.check(dev)
    try:
        with tuning(lib, instance_flatten_max=0):
            lib.rtcCommitScene(inst)
            lib.check(dev)
            keep[0][0][:v.size] *= np.float32(1.5)  # instanced scene 1 changes and is re-committed
            g = lib.rtcGetGeometry(child, 0)
            lib.rtcUpdateGeometryBuffer(g, RTC_BUFFER_TYPE_VERTEX, 0)
            lib.rtcCommitGeometry(g)
            lib.rtcCommitScene(child)
            lib.check(dev)
            lib.add_instance(dev, inst, nested, xfms[1], geom_id=len(xfms))
            lib.rtcCommitScene(inst)
            assert lib.rtcGetDeviceError(dev) == RTC_ERROR_INVALID_OPERATION
            lib.rtcDetachGeometry(inst, len(xfms))
            capfd.readouterr()
            lib.rtcCommitScene(inst)
            lib.check(dev)
            log = capfd.readouterr().err
            assert re.search(r"commit \(instance traversal\): 8 instances of 1 scenes, 0 rebuilt", log), log
        lib.rtcCommitScene(flat)
        lib.check(dev)
        ys, xs = np.meshgrid(np.linspace(-2.0, 3.0, 60), np.linspace(-2.5, 24.0, 240), indexing="ij")
        org = np.stack([xs.ravel(), ys.ravel(), np.zeros(xs.size)], 1)
        rays = make_rayhits(org, np.tile([0.0, 0.0, 1.0], (len(org), 1)))
        want = lib.intersect(flat, rays.copy(), "1M")
        assert (want["geomID"] != 0xFFFFFFFF).sum() > len(rays) // 4
        same_but_ties(lib.intersect(inst, rays.copy(), "1M"), want, "1M after a failed commit", len(rays) // 1000)
    finally:
        for sc in (inst, flat, nested, child):
            lib.rtcReleaseScene(sc)
        lib.rtcReleaseDevice(dev)
