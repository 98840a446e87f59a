"""Hit-gather entry point (rtcb200Intersect1MGatherDevice) on one GPU: the compact record stream in both delivery modes.
Named to sort after the other GPU test files: it is the newest entry point and must not shadow them under `-x`."""
import ctypes as C

import pytest

from embree_b200 import scenes
from tests.test_gpu_parity import build_scene

pytestmark = pytest.mark.gpu


def test_gather_records(b200):
    """rtcb200Intersect1MGatherDevice: the compact 32-byte record per ray {tfar, Ng, u, v, primID, geomID} equals the
    RTCRayHit result in both delivery modes ("gather_mode" 1: blocks staged in shared memory and stored as 1 KB, the
    default; 0: one 32-byte store per record), with work enqueued on the caller's stream after the call seeing the complete
    buffer; a ray count that is not a multiple of 32 exercises the partial tail block."""
    import torch
    from embree_b200 import sharding
    lib, dev = b200
    v, t = scenes.triangle_sphere(60)
    sc, keep = build_scene(lib, dev, [(v, t, 0, 0xFFFFFFFF)])
    rays = scenes.incoherent_rays_reference((3 << 20) + 13, device=torch.device("cuda", 0))
    rays[::5, 8] = 0.5                                     # some misses (tfar inside the sphere)
    a = lib.args()
    st = torch.cuda.current_stream().cuda_stream
    outs = []
    try:
        for mode in (1, 0, 1):
            assert lib.rtcb200SetTuning(b"gather_mode", mode) == 0
            B = rays.clone()
            out = torch.full((B.shape[0], 8), 7.0, device=B.device)
            lib.rtcb200Intersect1MGatherDevice(sc, C.c_void_p(B.data_ptr()), B.shape[0], C.byref(a), C.c_void_p(st), C.c_void_p(out.data_ptr()))
            got = out.clone()                              # stream-ordered after the call: must already see every record
            torch.cuda.synchronize()
            lib.check(dev)
            want = sharding.compact_hits(B)
            miss = B.view(torch.int32)[:, 18] == -1
            want[miss, 1:6] = 0.0
            want.view(torch.int32)[miss, 6] = -1
            want.view(torch.int32)[miss, 7] = -1
            assert miss.any() and (~miss).any()
            assert torch.equal(got.view(torch.int32), want.view(torch.int32)), mode
            outs.append(got)
        assert all(torch.equal(outs[0].view(torch.int32), o.view(torch.int32)) for o in outs[1:])   # and deterministic
    finally:
        lib.rtcb200SetTuning(b"gather_mode", 1)
    lib.rtcReleaseScene(sc)


def test_gather_empty_scene_writes_miss_records(b200):
    """A rank whose scene is empty (or holds only invalid triangles) must still deliver its slice of the gather buffer:
    one miss record {ray.tfar, 0, 0, 0, 0, 0, -1, -1} per ray, as the header promises."""
    import torch
    lib, dev = b200
    sc = lib.rtcNewScene(dev)
    lib.rtcCommitScene(sc)
    lib.check(dev)
    rays = scenes.incoherent_rays_reference(100000, device=torch.device("cuda", 0))
    rays[::3, 8] = 2.5
    out = torch.full((rays.shape[0], 8), 7.0, device=rays.device)
    a = lib.args()
    st = torch.cuda.current_stream().cuda_stream
    lib.rtcb200Intersect1MGatherDevice(sc, C.c_void_p(rays.data_ptr()), rays.shape[0], C.byref(a), C.c_void_p(st), C.c_void_p(out.data_ptr()))
    torch.cuda.synchronize()
    lib.check(dev)
    assert torch.equal(out[:, 0], rays[:, 8]) and (out[:, 1:6] == 0).all() and (out.view(torch.int32)[:, 6:8] == -1).all()
    lib.rtcReleaseScene(sc)

