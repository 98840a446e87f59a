"""The wavefront path-tracer driver kernels (embree_b200/csrc/pathstream.cu, BASELINE configs[4]) against their torch
restatement in embree_b200/scenes.py (path_primary / path_bounce, which follows tutorials/pathtracer/pathtracer_device.cpp
:1489-1603 and random_sampler.h:15-80), and the sharding rule of the path stream."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from embree_b200 import scenes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
W, H, SPP = 96, 54, 4
EYE, LOOK = (0.15, -0.1, 0.05), (0.3, 0.2, 1.0)
LIGHT = (0.2, 0.3, -0.1, 1.0, 0.8)


def test_path_stream_shards_are_the_single_stream():
    """Rank r owns paths [r*n, (r+1)*n): the union over ranks is the one-GPU stream (pixel = path // spp)."""
    cam = scenes.camera_basis(W, H, EYE, LOOK)
    n = W * H * SPP // 2
    full = scenes.path_primary(0, 2 * n, cam, W, H, SPP)
    parts = [scenes.path_primary(r * n, n, cam, W, H, SPP) for r in range(2)]
    assert torch.equal(torch.cat([p[0][:, :9] for p in parts]), full[0][:, :9])
    assert torch.equal(torch.cat([p[1] for p in parts]), full[1])


def test_pathstream_library_exports():
    """The driver library loads and exports its three entry points (no compute without a GPU)."""
    from embree_b200 import pathstream
    lib = C.CDLL(pathstream.LIB_PATH)
    for name in ("pts200_primary", "pts200_bounce", "pts200_shade"):
        assert hasattr(lib, name)
    out = subprocess.run(["cuobjdump", "-lelf", pathstream.LIB_PATH], stdout=subprocess.PIPE, text=True).stdout
    assert "sm_90a" in out and all("sm_90a" in l for l in out.splitlines() if "sm_" in l), out


@pytest.mark.gpu
def test_kernels_match_the_restatement(b200):
    from embree_b200 import pathstream
    from tests.test_gpu_parity import build_scene
    lib, dev = b200
    pts = pathstream.load()
    devt = torch.device("cuda", 0)
    st = torch.cuda.current_stream().cuda_stream
    cam = scenes.camera_basis(W, H, EYE, LOOK)
    n = W * H * SPP
    P = lambda x: C.c_void_p(x.data_ptr())   # noqa: E731
    R = torch.empty((n, 24), dtype=torch.float32, device=devt)
    S = torch.empty((n, 12), dtype=torch.float32, device=devt)
    rng = torch.empty(n, dtype=torch.int32, device=devt)
    Lw, pend, L = (torch.zeros(n, dtype=torch.float32, device=devt) for _ in range(3))
    first = 1000
    assert pts.pts200_primary(P(R), P(rng), P(Lw), first, n, (C.c_float * 12)(*cam.tolist()), W, H, SPP, C.c_void_p(st)) == 0
    want_r, want_s, want_lw = scenes.path_primary(first, n, cam, W, H, SPP, device=devt)
    torch.cuda.synchronize()
    assert torch.equal(rng.to(torch.int64) & 0xFFFFFFFF, want_s)                      # sampler state: exact
    assert (R[:, 0:9] - want_r[:, 0:9]).nan_to_num(posinf=0).abs().max() < 2e-6 and torch.equal(R.view(torch.int32)[:, 17:21], want_r.view(torch.int32)[:, 17:21])
    v, t = scenes.triangle_sphere(60)
    sc, keep = build_scene(lib, dev, [(v, t, 0, 0xFFFFFFFF)])
    a, ao = lib.args(), lib.args()
    light_c = (C.c_float * 5)(*LIGHT)
    R2, rng2, Lw2 = R.clone(), want_s.clone(), want_lw.clone()
    for b in range(3):
        lib.rtcb200Intersect1MDevice(sc, P(R), n, C.byref(a), C.c_void_p(st))
        torch.cuda.synchronize()
        R2.copy_(R)                                                                    # same traced records into both
        assert pts.pts200_bounce(P(R), P(S), P(rng), P(Lw), P(pend), n, light_c, C.c_void_p(st)) == 0
        shadow2, rng2, Lw2, pend2 = scenes.path_bounce(R2, rng2, Lw2, LIGHT)
        torch.cuda.synchronize()
        assert torch.equal(rng.to(torch.int64) & 0xFFFFFFFF, rng2), b
        for got, want, cols in ((R, R2, slice(0, 9)), (S, shadow2, slice(0, 9))):
            d = (got[:, cols] - want[:, cols]).nan_to_num(nan=0.0, posinf=0.0, neginf=0.0).abs().max()
            assert d < 2e-5, (b, float(d))
        assert (pend - pend2).abs().max() < 1e-5 and torch.allclose(Lw, Lw2)
        assert torch.equal(R.view(torch.int32)[:, 17:20], R2.view(torch.int32)[:, 17:20])   # geomID / primID reset to INVALID
        lib.rtcb200Occluded1MDevice(sc, P(S), n, C.byref(ao), C.c_void_p(st))
        assert pts.pts200_shade(P(S), P(pend), P(L), n, C.c_void_p(st)) == 0
        torch.cuda.synchronize()
        lib.check(dev)
    assert (R[:, 8] >= 0).all()                       # closed mesh: every path is still alive
    assert float(L.mean()) > 0 and torch.isfinite(L).all()
    lib.rtcReleaseScene(sc)


@pytest.mark.gpu
def test_dead_paths_stay_dead(b200):
    """A path that leaves the scene becomes an inactive record (tnear = +inf, tfar = -inf) that both query kinds skip."""
    from embree_b200 import pathstream
    from tests.test_gpu_parity import build_scene
    lib, dev = b200
    pts = pathstream.load()
    devt = torch.device("cuda", 0)
    st = torch.cuda.current_stream().cuda_stream
    tv, tt = scenes.terrain(64, seed=7)                   # open surface: bounce rays escape
    sc, keep = build_scene(lib, dev, [(tv, tt, 0, 0xFFFFFFFF)])
    cam = scenes.camera_basis(W, H, (0.0, 0.9, -0.2), (0.0, -1.0, 0.25))
    n = W * H * SPP
    P = lambda x: C.c_void_p(x.data_ptr())   # noqa: E731
    R = torch.empty((n, 24), dtype=torch.float32, device=devt)
    S = torch.empty((n, 12), dtype=torch.float32, device=devt)
    rng = torch.empty(n, dtype=torch.int32, device=devt)
    Lw, pend, L = (torch.zeros(n, dtype=torch.float32, device=devt) for _ in range(3))
    assert pts.pts200_primary(P(R), P(rng), P(Lw), 0, n, (C.c_float * 12)(*cam.tolist()), W, H, SPP, C.c_void_p(st)) == 0
    a, ao = lib.args(), lib.args()
    alive = []
    for b in range(4):
        lib.rtcb200Intersect1MDevice(sc, P(R), n, C.byref(a), C.c_void_p(st))
        assert pts.pts200_bounce(P(R), P(S), P(rng), P(Lw), P(pend), n, (C.c_float * 5)(0.0, 2.0, 0.0, 1.0, 0.8), C.c_void_p(st)) == 0
        lib.rtcb200Occluded1MDevice(sc, P(S), n, C.byref(ao), C.c_void_p(st))
        assert pts.pts200_shade(P(S), P(pend), P(L), n, C.c_void_p(st)) == 0
        torch.cuda.synchronize()
        alive.append(int((R[:, 8] >= 0).sum()))
        dead = R[:, 8] < 0
        assert (pend[dead] == 0).all() and (S[dead, 8] == float("-inf")).all()
    lib.check(dev)
    assert 0 < alive[-1] < alive[0] <= n and all(x >= y for x, y in zip(alive, alive[1:])), alive
    lib.rtcReleaseScene(sc)
