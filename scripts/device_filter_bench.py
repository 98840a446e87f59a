"""What an argument filter costs in device-side queries (include/embree4_b200_device.cuh), with the launcher of
tests/device_filter/devfilter.cu (one thread per ray, arguments and context in the thread's memory).

  headline      bench.py's scene (10 M-triangle sphere) and its 64 Mi diffuse-bounce rays, closest hit and any hit: no filter,
                an accept-everything filter under RTC_RAY_QUERY_FLAG_INVOKE_ARGUMENT_FILTER, and the reject-one-in-four rule
  fur ball      bench.py's hair scene (120 000 flat cubic Bezier strands around a triangle sphere): shadow rays from the camera
                rays' hits, through the hair tutorial's transparency filter with its state indexed by ray.id (only the hair
                enables the filter); the device filter against rtcb200Occluded1M with the same filter as a host C callback,
                the host path on the first --host-rays rays only

Variants run alternately (one warm-up each, then --reps repetitions), timed with CUDA events (the host path: wall clock around
the call, which synchronises); the report gives median [min, max] ms and Mrays/s, the card's name, power limit and max SM clock,
and whether the outputs are byte-identical where they must be.  Prints one JSON line; writes nothing.

    python scripts/device_filter_bench.py [--rays N] [--reps R] [--host-rays M]
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
import embree_b200  # noqa: E402
from embree_b200 import rtc, scenes  # noqa: E402
from scripts.device_traversal_bench import gpu_info  # noqa: E402

DEVFILTER = os.path.join(ROOT, "tests", "device_filter", "_build", "libdevfilter.so")
F_NONE, F_ACCEPT, F_RULE, F_HAIR_ID = 0, 1, 2, 6   # devfilter.cu enum Filter
INVOKE = rtc.RTC_RAY_QUERY_FLAG_INVOKE_ARGUMENT_FILTER


def stat(x, n):
    m = float(np.median(x))
    return {"ms_median": m, "ms_range": [float(min(x)), float(max(x))], "Mrays_per_s": n / m * 1e-3}


def load_tool():
    L = C.CDLL(DEVFILTER)
    P = C.c_void_p
    L.devfilter_query.argtypes = [P, C.c_int, P, C.c_size_t, C.c_int, C.c_uint, C.c_uint, C.c_int, C.c_uint, C.c_uint, P, P, C.c_uint, P, P, P, P]
    L.devfilter_set_host_T_by_id.argtypes = [P]
    return L


def launch(L, t, occluded, buf, n, which, flags, T_by_id=None):
    s = torch.cuda.current_stream()
    e = L.devfilter_query(C.byref(t), int(occluded), C.c_void_p(buf.data_ptr()), n, which, flags, rtc.RTC_FEATURE_FLAG_ALL, 1, 0xFFFFFFFF,
                          0xFFFFFFFF, None, None, 0, None, C.c_void_p(T_by_id.data_ptr()) if T_by_id is not None else None, None,
                          C.c_void_p(s.cuda_stream))
    assert e == 0, e


def headline(lib, dev, L, sc, rays, reps, occluded):
    n = rays.shape[0]
    t = lib.scene_device_traversable(sc)
    lib.check(dev)
    variants = {"no_filter": (F_NONE, 0), "accept_all_invoke": (F_ACCEPT, INVOKE), "reject_one_in_four": (F_RULE, INVOKE)}
    bufs = {k: torch.empty_like(rays) for k in variants}
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    times = {k: [] for k in variants}
    for rep in range(reps + 1):
        for k, (which, flags) in variants.items():
            bufs[k].copy_(rays)
            torch.cuda.synchronize()
            ev[0].record()
            launch(L, t, occluded, bufs[k], n, which, flags)
            ev[1].record()
            ev[1].synchronize()
            if rep:
                times[k].append(ev[0].elapsed_time(ev[1]))
    lib.check(dev)
    out = {"rays": n}
    for k in variants:
        out[k] = stat(times[k], n)
    out["accept_all_over_no_filter_time"] = out["accept_all_invoke"]["ms_median"] / out["no_filter"]["ms_median"]
    out["accept_all_byte_identical_to_no_filter"] = bool(torch.equal(bufs["no_filter"].view(torch.int32), bufs["accept_all_invoke"].view(torch.int32)))
    col = 8 if occluded else 18
    A = bufs["reject_one_in_four"]
    out["reject_rule_hits"] = int(torch.isinf(A[:, 8]).logical_and(A[:, 8] < 0).sum().item()) if occluded else int((A.view(torch.int32)[:, col] != -1).sum().item())
    return out


def fur_shadows(lib, dev, L, reps, host_rays):
    devt = torch.device("cuda:0")
    cv, ci, _tg = scenes.cubic_hair(120000, "bezier", knots=10, seed=5, radius=1.0, step=0.05, width=0.0025)
    v, t = scenes.triangle_sphere(201)
    sc = lib.rtcNewScene(dev)
    keep = [lib.add_triangle_mesh(dev, sc, v, t, mask=0xFFFFFFFF, geom_id=0)[1],
            lib.add_flat_cubic_curves(dev, sc, cv, ci, "bezier", None, None, mask=0xFFFFFFFF, geom_id=1)[1]]
    lib.rtcSetGeometryEnableFilterFunctionFromArguments(lib.rtcGetGeometry(sc, 1), True)
    lib.rtcCommitScene(sc)
    lib.check(dev)
    cam = scenes.primary_rays(bench.PRIMARY_W, bench.PRIMARY_H, eye=(0.0, 0.4, -2.6), look=(0.0, -0.15, 1.0), fov=60.0, device=devt)
    s = torch.cuda.current_stream()
    lib.rtcb200Intersect1MDevice(sc, C.c_void_p(cam.data_ptr()), cam.shape[0], C.byref(lib.args()), C.c_void_p(s.cuda_stream))
    torch.cuda.synchronize()
    hit = cam.view(torch.int32)[:, 18] != -1
    h = cam[hit]
    n = h.shape[0]
    sh = torch.zeros((n, 12), dtype=torch.float32, device=devt)   # shadow rays from the hit points towards a directional light
    sh[:, 0:3] = h[:, 0:3] + h[:, 8:9] * h[:, 4:7]
    sh[:, 3] = 1e-3
    sh[:, 4:7] = torch.tensor([0.35, 1.0, -0.45], device=devt)
    sh[:, 8] = float("inf")
    sh.view(torch.int32)[:, 9] = -1
    sh.view(torch.int32)[:, 10] = torch.arange(n, dtype=torch.int32, device=devt)
    tr = lib.scene_device_traversable(sc)
    lib.check(dev)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    buf, T = torch.empty_like(sh), torch.ones((n, 3), dtype=torch.float32, device=devt)
    m = min(host_rays, n)
    host_rays_np = sh[:m].cpu().numpy().view(rtc.RAY_DTYPE).reshape(-1).copy()
    fn = rtc.FILTER_FUNCTION(C.cast(L.devfilter_host_hair_id, C.c_void_p).value)
    args = lib.args(filter=fn)
    td, tds, th = [], [], []
    for rep in range(reps + 1):
        for count, store in ((n, td), (m, tds)):
            buf[:count].copy_(sh[:count])
            T.fill_(1.0)
            torch.cuda.synchronize()
            ev[0].record()
            launch(L, tr, True, buf, count, F_HAIR_ID, 0, T)
            ev[1].record()
            ev[1].synchronize()
            if rep:
                store.append(ev[0].elapsed_time(ev[1]))
        hr = host_rays_np.copy()
        hT = np.ones((m, 3), np.float32)
        L.devfilter_set_host_T_by_id(hT.ctypes.data)
        t0 = time.perf_counter()
        lib.rtcb200Occluded1M(sc, C.c_void_p(hr.ctypes.data), m, C.byref(args))
        t1 = time.perf_counter()
        L.devfilter_set_host_T_by_id(None)
        if rep:
            th.append((t1 - t0) * 1e3)
    lib.check(dev)
    dev_rays = buf[:m].cpu().numpy().view(rtc.RAY_DTYPE).reshape(-1)
    dev_T = T[:m].cpu().numpy()
    occ = hr["tfar"] < 0
    out = {"shadow_rays": n, "device_filter": stat(td, n), "device_filter_on_host_subsample": stat(tds, m),
           "host_pointer_path_subsample": stat(th, m), "host_subsample_rays": m,
           "occluded_fraction": float(occ.mean()),
           "rays_byte_identical_on_subsample": dev_rays.tobytes() == hr.tobytes(),
           "transparency_byte_identical_on_unoccluded": dev_T[~occ].tobytes() == hT[~occ].tobytes()}
    lib.rtcReleaseScene(sc)
    del keep
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rays", type=int, default=64 << 20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--phi", type=int, default=1581)
    ap.add_argument("--host-rays", type=int, default=1 << 18)
    args = ap.parse_args()
    lib = embree_b200.load()
    L = load_tool()
    dev = lib.new_device(None)
    devt = torch.device("cuda:0")
    out = {"metric": "argument filters in device-side queries", "gpu": gpu_info(), "reps": args.reps}

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
    out["headline_closest"] = headline(lib, dev, L, sc, rays, args.reps, occluded=False)
    occ = rays[:, :12].contiguous()
    del rays
    torch.cuda.empty_cache()
    out["headline_any_hit"] = headline(lib, dev, L, sc, occ, args.reps, occluded=True)
    del occ
    lib.rtcReleaseScene(sc)
    del keep
    torch.cuda.empty_cache()
    out["fur_ball_shadows"] = fur_shadows(lib, dev, L, args.reps, args.host_rays)
    out["gpu_after"] = gpu_info()
    print(json.dumps(out))
    lib.rtcReleaseDevice(dev)


if __name__ == "__main__":
    main()
