"""What tracing from the caller's own kernel costs: the one-thread-per-ray launcher of tests/device_api/devtrace.cu (it calls
rtcb200TraversableIntersect1 / rtcb200TraversableOccluded1 of include/embree4_b200_device.cuh) against the batched
rtcb200Intersect1MDevice / rtcb200Occluded1MDevice on the same rays.

  headline      bench.py's scene (10 M-triangle sphere, numPhi 1581) and its 64 Mi diffuse-bounce rays, closest hit and any hit
  fur ball      bench.py's hair scene (120 000 flat cubic Bezier strands around a triangle sphere), 1920x1080 camera rays

Each pair runs alternately (one warm-up each, then --reps repetitions), timed with CUDA events around the launch alone; the
report gives median [min, max] ms and Mrays/s, and whether the two paths wrote byte-identical records.  Needs the test tool
(tests/device_api/build.sh, which __graft_entry__.build() runs).  Prints one JSON line; writes nothing.

    python scripts/device_traversal_bench.py [--rays N] [--reps R]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
import embree_b200  # noqa: E402
from embree_b200 import scenes  # noqa: E402

DEVTRACE = os.path.join(ROOT, "tests", "device_api", "_build", "libdevtrace.so")


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], stdout=subprocess.PIPE,
                           stderr=subprocess.DEVNULL, text=True, timeout=10).stdout.strip()
        return dict(zip(("name", "power_limit", "sm_max_clock"), [x.strip() for x in q.split(",")]))
    except Exception:   # noqa: BLE001
        return {"name": torch.cuda.get_device_name(0)}


def compare(lib, dev, dt, sc, rays, reps, occluded):
    """rays: [n, 24] (RTCRayHit) or [n, 12] (RTCRay) float32 on the GPU.  Alternating batched / per-thread runs."""
    n = rays.shape[0]
    stream = torch.cuda.current_stream()
    s = C.c_void_p(stream.cuda_stream)
    t = lib.scene_device_traversable(sc)
    a = lib.args()
    A, B = torch.empty_like(rays), torch.empty_like(rays)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]

    def timed(buf, fn):
        buf.copy_(rays)
        torch.cuda.synchronize()
        ev[0].record(stream)
        fn(C.c_void_p(buf.data_ptr()))
        ev[1].record(stream)
        ev[1].synchronize()
        return ev[0].elapsed_time(ev[1])
    if occluded:
        batched = lambda p: lib.rtcb200Occluded1MDevice(sc, p, n, C.byref(a), s)   # noqa: E731
        device = lambda p: dt.devtrace_occluded(C.byref(t), p, n, None, s)        # noqa: E731
    else:
        batched = lambda p: lib.rtcb200Intersect1MDevice(sc, p, n, C.byref(a), s)  # noqa: E731
        device = lambda p: dt.devtrace_intersect(C.byref(t), p, n, None, s)       # noqa: E731
    timed(A, batched)
    timed(B, device)
    tb, td = [], []
    for _ in range(reps):
        tb.append(timed(A, batched))
        td.append(timed(B, device))
    lib.check(dev)
    same = bool(torch.equal(A.view(torch.int32), B.view(torch.int32)))
    hits = int((A.view(torch.int32)[:, 18] != -1).sum().item()) if not occluded else int(torch.isinf(A[:, 8]).logical_and(A[:, 8] < 0).sum().item())

    def stat(x):
        m = float(np.median(x))
        return {"ms_median": m, "ms_range": [float(min(x)), float(max(x))], "Mrays_per_s": n / m * 1e-3}
    b, d = stat(tb), stat(td)
    return {"rays": n, "hits": hits, "batched": b, "per_thread": d, "per_thread_over_batched_time": d["ms_median"] / b["ms_median"],
            "byte_identical": same}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rays", type=int, default=64 << 20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--phi", type=int, default=1581)
    args = ap.parse_args()
    lib = embree_b200.load()
    dt = C.CDLL(DEVTRACE)
    P = C.c_void_p
    dt.devtrace_intersect.argtypes = [P, P, C.c_size_t, P, P]
    dt.devtrace_occluded.argtypes = [P, P, C.c_size_t, P, P]
    dev = lib.new_device(None)
    devt = torch.device("cuda:0")
    out = {"metric": "device-side queries (one thread per ray) vs the batched entry points", "gpu": gpu_info(), "reps": args.reps}

    # headline: 10 M triangles, 64 Mi diffuse-bounce rays (bench.py configs[2])
    v, t = bench.make_scene(args.phi)
    sc = lib.rtcNewScene(dev)
    _gid, keep = lib.add_triangle_mesh(dev, sc, v, t, mask=0xFFFFFFFF)
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
    out["headline_closest"] = compare(lib, dev, dt, sc, rays, args.reps, occluded=False)
    occ = rays[:, :12].contiguous()
    del rays
    out["headline_any_hit"] = compare(lib, dev, dt, sc, occ, args.reps, occluded=True)
    del occ
    lib.rtcReleaseScene(sc)
    del keep
    torch.cuda.empty_cache()

    # fur ball (bench.py hair_leg): camera rays
    strands = 120000
    cv, ci, _tg = scenes.cubic_hair(strands, "bezier", knots=10, seed=5, radius=1.0, step=0.05, width=0.0025)
    v, t = scenes.triangle_sphere(201)
    sc = lib.rtcNewScene(dev)
    keep = [lib.add_triangle_mesh(dev, sc, v, t, mask=0xFFFFFFFF, geom_id=0)[1],
            lib.add_flat_cubic_curves(dev, sc, cv, ci, "bezier", None, None, mask=0xFFFFFFFF, geom_id=1)[1]]
    lib.rtcCommitScene(sc)
    lib.check(dev)
    cam = scenes.primary_rays(bench.PRIMARY_W, bench.PRIMARY_H, eye=(0.0, 0.4, -2.6), look=(0.0, -0.15, 1.0), fov=60.0, device=devt)
    out["fur_ball_camera_closest"] = compare(lib, dev, dt, sc, cam, args.reps, occluded=False)
    out["fur_ball_camera_any_hit"] = compare(lib, dev, dt, sc, cam[:, :12].contiguous(), args.reps, occluded=True)
    lib.rtcReleaseScene(sc)
    del keep
    out["gpu_after"] = gpu_info()
    print(json.dumps(out))
    lib.rtcReleaseDevice(dev)


if __name__ == "__main__":
    main()
