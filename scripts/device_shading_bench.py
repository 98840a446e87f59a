"""Shading in the caller's kernel (include/embree4_b200_device.cuh) against the batched path, with the launchers of
tests/device_shading/devshade.cu:

  megakernel    one thread per ray: rtcb200TraversableIntersect1, rtcb200Interpolate1 of the normal from a VERTEX_ATTRIBUTE slot,
                rtcb200GetGeometryTransformFromTraversable through the hit's instID[0], the world-space normal written out
  batched       rtcb200Intersect1MDevice, then rtcb200InterpolateHitsDevice of the same slot, then a kernel that transforms the
                interpolated normals with the same code

on two workloads:

  headline      bench.py's scene (10 M-triangle sphere, its normals as attribute slot 0) and its 64 Mi diffuse-bounce rays
  instanced     the scene of every kind with six instances (tests/test_interpolate.py mixed_scene; slot 0 is a FLOAT3 attribute
                at a 20-byte stride) and 4 Mi rays from a sphere around it

The two paths run alternately (one warm-up each, then --reps repetitions), timed with CUDA events from the first launch to the
last; the report gives median [min, max] ms and Mrays/s, the card's name, power limit and max SM clock read in the same call, and
whether the normals are bit-equal (NaN normals -- points and geometries without the slot -- must be NaN in both).  Prints one JSON
line; writes nothing.

    python scripts/device_shading_bench.py [--rays N] [--reps R] [--instanced-rays M]
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
import embree_b200  # noqa: E402
from embree_b200 import scenes  # noqa: E402
from embree_b200.rtc import RTC_BUFFER_TYPE_VERTEX_ATTRIBUTE, RTC_FORMAT_FLOAT3, _ptr  # noqa: E402
from scripts.device_traversal_bench import gpu_info  # noqa: E402

DEVSHADE = os.path.join(ROOT, "tests", "device_shading", "_build", "libdevshade.so")


def stat(x, n):
    m = float(np.median(x))
    return {"ms_median": m, "ms_range": [float(min(x)), float(max(x))], "Mrays_per_s": n / m * 1e-3}


def load_tool():
    L = C.CDLL(DEVSHADE)
    P = C.c_void_p
    L.devshade_shade.argtypes = [P, P, P, C.c_size_t, P, P]
    L.devshade_transform_normals.argtypes = [P, P, P, C.c_size_t, P, P]
    return L


def compare(lib, dev, L, sc, rays, reps):
    """rays: [n, 24] float32 RTCRayHit records on the GPU."""
    n = rays.shape[0]
    stream = torch.cuda.current_stream()
    s = C.c_void_p(stream.cuda_stream)
    t = lib.scene_device_traversable(sc)
    ip = lib.scene_device_interpolator(sc, RTC_BUFFER_TYPE_VERTEX_ATTRIBUTE, 0)
    lib.check(dev)
    a = lib.args()
    out_m = torch.empty((n, 3), dtype=torch.float32, device=rays.device)
    out_b = torch.empty_like(out_m)
    buf = torch.empty_like(rays)
    P = torch.empty((3, n), dtype=torch.float32, device=rays.device)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]

    def mega():
        assert L.devshade_shade(C.byref(t), C.byref(ip), C.c_void_p(rays.data_ptr()), n, C.c_void_p(out_m.data_ptr()), s) == 0

    def batched():
        lib.rtcb200Intersect1MDevice(sc, C.c_void_p(buf.data_ptr()), n, C.byref(a), s)
        lib.interpolate_hits(sc, buf, RTC_BUFFER_TYPE_VERTEX_ATTRIBUTE, 0, 3, want=("P",), stream=stream, out={"P": P})
        assert L.devshade_transform_normals(C.byref(t), C.c_void_p(buf.data_ptr()), C.c_void_p(P.data_ptr()), n, C.c_void_p(out_b.data_ptr()), s) == 0

    times = {"megakernel": [], "batched": []}
    for rep in range(reps + 1):
        for name, fn in (("megakernel", mega), ("batched", batched)):
            buf.copy_(rays)
            torch.cuda.synchronize()
            ev[0].record(stream)
            fn()
            ev[1].record(stream)
            ev[1].synchronize()
            if rep:
                times[name].append(ev[0].elapsed_time(ev[1]))
    lib.check(dev)
    hit = buf.view(torch.int32)[:, 18] != -1
    nan_m, nan_b = torch.isnan(out_m), torch.isnan(out_b)
    same = torch.equal(nan_m, nan_b) and torch.equal(out_m.view(torch.int32)[~nan_m], out_b.view(torch.int32)[~nan_b])
    out = {"rays": n, "hits": int(hit.sum().item()), "nan_normals": int(nan_m.any(1).sum().item())}
    for k in times:
        out[k] = stat(times[k], n)
    out["megakernel_over_batched_time"] = out["megakernel"]["ms_median"] / out["batched"]["ms_median"]
    out["normals_bit_equal"] = bool(same)
    out["normals_bit_equal_including_nan_payloads"] = bool(torch.equal(out_m.view(torch.int32), out_b.view(torch.int32)))
    return out


def headline(lib, dev, L, args):
    devt = torch.device("cuda:0")
    v, t = bench.make_scene(args.phi)
    sc = lib.rtcNewScene(dev)
    _gid, keep = lib.add_triangle_mesh(dev, sc, v, t, mask=0xFFFFFFFF)
    vv = np.asarray(v, np.float32).reshape(-1, 3)
    c = vv - vv.mean(0)
    nrm = np.ascontiguousarray(c / np.linalg.norm(c, axis=1, keepdims=True), np.float32)
    g = lib.rtcGetGeometry(sc, 0)
    lib.dll.rtcSetGeometryVertexAttributeCount(C.c_void_p(g), 1)
    lib.rtcSetSharedGeometryBuffer(g, RTC_BUFFER_TYPE_VERTEX_ATTRIBUTE, 0, RTC_FORMAT_FLOAT3, _ptr(nrm), 0, 12, len(nrm))
    lib.rtcCommitGeometry(g)
    lib.rtcCommitScene(sc)
    lib.check(dev)
    stream = torch.cuda.current_stream()
    prim = scenes.primary_rays(bench.PRIMARY_W, bench.PRIMARY_H, eye=bench.EYE, look=bench.LOOK, device=devt)
    lib.rtcb200Intersect1MDevice(sc, C.c_void_p(prim.data_ptr()), prim.shape[0], C.byref(lib.args()), C.c_void_p(stream.cuda_stream))
    torch.cuda.synchronize()
    n = args.rays
    rays = torch.empty((n, 24), dtype=torch.float32, device=devt)
    for c0 in range(0, n, 1 << 22):
        ids = torch.arange(c0, min(c0 + (1 << 22), n), device=devt, dtype=torch.int64)
        rays[c0:c0 + len(ids)] = bench.bounce_rays(prim, ids)
    del prim
    out = compare(lib, dev, L, sc, rays, args.reps)
    del rays
    lib.rtcReleaseScene(sc)
    del keep, nrm
    torch.cuda.empty_cache()
    return out


def instanced(lib, dev, L, args):
    from tests.test_interpolate import mixed_scene, rays
    top, child, keep = mixed_scene(lib, dev)
    r = torch.from_numpy(rays(args.instanced_rays).view(np.float32).reshape(-1, 24).copy()).cuda()
    out = compare(lib, dev, L, top, r, args.reps)
    lib.rtcReleaseScene(top)
    lib.rtcReleaseScene(child)
    del keep
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rays", type=int, default=64 << 20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--phi", type=int, default=1581)
    ap.add_argument("--instanced-rays", type=int, default=4 << 20)
    args = ap.parse_args()
    lib = embree_b200.load()
    L = load_tool()
    dev = lib.new_device(None)
    out = {"metric": "shading in the caller's kernel vs batched trace + interpolate + transform", "gpu": gpu_info(), "reps": args.reps}
    out["headline"] = headline(lib, dev, L, args)
    out["instanced_mixed"] = instanced(lib, dev, L, args)
    out["gpu_after"] = gpu_info()
    print(json.dumps(out))
    lib.rtcReleaseDevice(dev)


if __name__ == "__main__":
    main()
