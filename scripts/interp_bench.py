"""Batched interpolation of traced hits (rtcb200InterpolateHitsDevice) on the headline scene of bench.py: the 10 M-triangle sphere
(numPhi 1581) and 64 Mi diffuse-bounce rays traced device-resident, then three interpolations of the hits on the same stream:

  vertex      RTC_BUFFER_TYPE_VERTEX, valueCount 3, P + dPdu + dPdv
  texcoord    a FLOAT2 attribute (8-byte stride), P
  normal      a FLOAT3 attribute (12-byte stride), P

Reports per run the CUDA-event kernel time (median and range over alternating repetitions), Ghits/s, the algorithmic bytes per
hit over that time against the H100 SXM data sheet's 3.35 TB/s, the ratio to the trace kernel's time on the same stream, the
cost of the first call after the commit (it uploads the buffers the table reads), and the host rtcInterpolateN on a 1 Mi sample for
contrast.  Prints one JSON line; writes nothing.

Algorithmic bytes per hit (what the kernel must move at least): the hit's u, v, primID, geomID, instID (20 B), its geometry's table
entry (64 B, shared by all hits: 0), the primitive's three indices (12 B), the three vertices' `valueCount` floats each as the
32-byte sectors they lie in (vertices are scattered: 3 x 32 B), and the outputs (4 B per value and output).  Misses read the 20 B
only.

    python scripts/interp_bench.py [--rays N] [--reps R]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
import embree_b200  # noqa: E402
from embree_b200.rtc import (INTERP_OUTPUTS, InterpolateNArguments, RTC_BUFFER_TYPE_VERTEX, RTC_BUFFER_TYPE_VERTEX_ATTRIBUTE,  # noqa: E402
                             RTC_FORMAT_FLOAT, RTC_FORMAT_FLOAT3, _ptr)

HBM = 3.35e12


def algorithmic_bytes(hits, vc, nout):
    return hits * (20 + 12 + 3 * 32 + 4 * vc * nout)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rays", type=int, default=64 << 20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--phi", type=int, default=1581)
    args = ap.parse_args()
    lib = embree_b200.load()
    dev = lib.new_device(None)
    v, t = bench.make_scene(args.phi)
    nv = len(v)
    rng = np.random.RandomState(0)
    uv = rng.uniform(0, 1, (nv, 2)).astype(np.float32)
    nrm = (v / np.linalg.norm(v, axis=1, keepdims=True)).astype(np.float32)
    nrm = np.concatenate([nrm.reshape(-1), np.zeros(4, np.float32)])
    sc = lib.rtcNewScene(dev)
    _gid, keep = lib.add_triangle_mesh(dev, sc, v, t, mask=0xFFFFFFFF)
    g = lib.rtcGetGeometry(sc, 0)
    lib.dll.rtcSetGeometryVertexAttributeCount(C.c_void_p(g), 2)
    lib.rtcSetSharedGeometryBuffer(g, RTC_BUFFER_TYPE_VERTEX_ATTRIBUTE, 0, RTC_FORMAT_FLOAT + 1, _ptr(uv), 0, 8, nv)
    lib.rtcSetSharedGeometryBuffer(g, RTC_BUFFER_TYPE_VERTEX_ATTRIBUTE, 1, RTC_FORMAT_FLOAT3, _ptr(nrm), 0, 12, nv)
    lib.rtcCommitGeometry(g)
    lib.rtcCommitScene(sc)
    lib.check(dev)

    devt = torch.device("cuda:0")
    stream = torch.cuda.current_stream()
    a = lib.args()
    prim = bench.scenes.primary_rays(bench.PRIMARY_W, bench.PRIMARY_H, eye=bench.EYE, look=bench.LOOK, device=devt)
    lib.rtcb200Intersect1MDevice(sc, C.c_void_p(prim.data_ptr()), prim.shape[0], C.byref(a), C.c_void_p(stream.cuda_stream))
    torch.cuda.synchronize()
    n = args.rays
    R = torch.empty((n, 24), dtype=torch.float32, device=devt)
    for c0 in range(0, n, 1 << 22):
        ids = torch.arange(c0, min(c0 + (1 << 22), n), device=devt, dtype=torch.int64)
        R[c0:c0 + len(ids)] = bench.bounce_rays(prim, ids)
    del prim
    rays = R.clone()

    runs = {"vertex": (RTC_BUFFER_TYPE_VERTEX, 0, 3, ("P", "dPdu", "dPdv")),
            "texcoord": (RTC_BUFFER_TYPE_VERTEX_ATTRIBUTE, 0, 2, ("P",)),
            "normal": (RTC_BUFFER_TYPE_VERTEX_ATTRIBUTE, 1, 3, ("P",))}
    outs = {k: {o: torch.empty((vc, n), dtype=torch.float32, device=devt) for o in want} for k, (_b, _s, vc, want) in runs.items()}
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]

    def timed(fn):
        ev[0].record(stream)
        fn()
        ev[1].record(stream)
        ev[1].synchronize()
        return ev[0].elapsed_time(ev[1])

    def trace():
        R.copy_(rays)   # untimed below: the trace is timed alone
        torch.cuda.synchronize()
        return timed(lambda: lib.rtcb200Intersect1MDevice(sc, C.c_void_p(R.data_ptr()), n, C.byref(a), C.c_void_p(stream.cuda_stream)))

    def interp(k):
        bt, slot, vc, want = runs[k]
        return timed(lambda: lib.interpolate_hits(sc, R, bt, slot, vc, want=want, stream=stream, out=outs[k]))

    trace_ms = [trace()]
    first_call = {k: interp(k) for k in runs}   # the first call after the commit builds the table and uploads the buffers
    lib.check(dev)
    for k in runs:
        interp(k)   # warm
    times = {k: [] for k in runs}
    for _ in range(args.reps):
        for k in runs:
            times[k].append(interp(k))
        trace_ms.append(trace())
    lib.check(dev)
    hits = int((R.view(torch.int32)[:, 18] != -1).sum().item())
    tmed = float(np.median(trace_ms[1:]))

    # host rtcInterpolateN on a 1 Mi sample of the hits, for contrast
    sample = R[:: max(1, n // (1 << 20))][: 1 << 20].cpu().numpy().view(np.uint32)
    hit = sample[:, 18] != 0xFFFFFFFF
    prim_ids = np.ascontiguousarray(sample[hit, 17])
    u = np.ascontiguousarray(sample[hit, 15].view(np.float32))
    vv = np.ascontiguousarray(sample[hit, 16].view(np.float32))
    o = {k: np.empty((3, len(u)), np.float32) for k in INTERP_OUTPUTS}
    na = InterpolateNArguments(g, None, prim_ids.ctypes.data, u.ctypes.data, vv.ctypes.data, len(u), RTC_BUFFER_TYPE_VERTEX, 0, o["P"].ctypes.data,
                               o["dPdu"].ctypes.data, o["dPdv"].ctypes.data, None, None, None, 3)
    t0 = time.perf_counter()
    lib.rtcInterpolateN(C.byref(na))
    host_s = time.perf_counter() - t0
    # the device result on the same hits
    dP = outs["vertex"]["P"][:, :: max(1, n // (1 << 20))][:, : 1 << 20].cpu().numpy()[:, hit]
    same = bool((dP.view(np.uint32) == o["P"].view(np.uint32)).all())

    gpu = {}
    try:
        q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], stdout=subprocess.PIPE,
                           stderr=subprocess.DEVNULL, text=True, timeout=10).stdout.strip()
        gpu = dict(zip(("name", "power_limit", "sm_max_clock"), [x.strip() for x in q.split(",")]))
    except Exception:   # noqa: BLE001
        pass
    res = {}
    for k, (_b, _s, vc, want) in runs.items():
        ms = float(np.median(times[k]))
        byts = algorithmic_bytes(hits, vc, len(want)) + (n - hits) * 20
        res[k] = {"kernel_ms_median": ms, "kernel_ms_range": [float(min(times[k])), float(max(times[k]))], "Ghits_per_s": hits / ms * 1e-6,
                  "algorithmic_bytes_per_hit": algorithmic_bytes(1, vc, len(want)), "achieved_TB_per_s": byts / ms * 1e-9,
                  "share_of_hbm_peak": byts / ms * 1e3 / HBM, "ratio_to_trace": ms / tmed, "first_call_ms": first_call[k]}
    print(json.dumps({"metric": "batched interpolation of traced hits", "gpu": gpu, "rays": n, "hits": hits, "reps": args.reps,
                      "trace_ms_median": tmed, "trace_ms_range": [float(min(trace_ms[1:])), float(max(trace_ms[1:]))], "runs": res,
                      "host_rtcInterpolateN": {"hits": int(hit.sum()), "seconds": host_s, "Mhits_per_s": hit.sum() / host_s * 1e-6,
                                               "bit_equal_to_device": same}}))
    lib.rtcReleaseScene(sc)
    lib.rtcReleaseDevice(dev)


if __name__ == "__main__":
    main()
