"""Instances flattened into one BVH against instance traversal (one BVH per instanced scene under a top level over the instances).

  (a) scale    N = 2, 4, 16, 256, 4096, 65536 random instances (rotation, scale 0.5 .. 1, translation) of the 1 M-triangle
               createTriangleSphere(500), at MEDIUM quality: the first commit of a new top-level scene (the instanced scene committed
               before), the scene's node + record bytes, and Mrays/s of 1 Mi camera rays and of 1 Mi diffuse bounces off their hits
               through rtcb200Intersect1MDevice.  The flattened arm runs while its build fits in the card's memory; a commit that fails
               is reported as such.
  (b) edits    re-commit of the N = 16 and N = 4096 scenes after moving 1 % (at least one) and 100 % of the instances.
  (c) records  the two arms' records for the same scene and rays, compared byte for byte (differences at bit-identical t are
               ties: which of two equal-t records wins depends on the traversal order).

rtcb200SetTuning("instance_flatten_max") selects the arm.  The arms alternate: one warm-up each, then --reps repetitions; the
report gives median [min, max], with the card's name, power limit and max SM clock read in the same call.  Commit times are wall
clock around rtcCommitScene (it returns when the build is done); trace times are CUDA events around one launch.  Prints one JSON
line; writes nothing.

    python scripts/instancing_bench.py [--reps R] [--phi P] [--counts 2,4,16,256,4096,65536] [--width W]
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

import embree_b200  # noqa: E402
from embree_b200 import scenes  # noqa: E402
from embree_b200.rtc import RTC_BUILD_QUALITY_MEDIUM, RTC_FORMAT_FLOAT3X4_COLUMN_MAJOR, _ptr  # noqa: E402
from scripts.device_traversal_bench import gpu_info  # noqa: E402

FLAT, INST = "flattened", "instance_traversal"
FORCE = {FLAT: 2**31 - 1, INST: 0}
MAX_PRIMS = 2**31 - 1   # the builder's limit on the primitives of one BVH: a flattened scene beyond it cannot be built


def stat(x):
    return {"median": float(np.median(x)), "range": [float(min(x)), float(max(x))]} if x else "not measured"


def transforms(n, seed):
    rng = np.random.RandomState(seed)
    side = 2.0 * n ** (1.0 / 3.0)
    out = []
    for _ in range(n):
        q, _r = np.linalg.qr(rng.normal(size=(3, 3)))
        m = q * rng.uniform(0.5, 1.0)
        out.append(np.concatenate([m[:, 0], m[:, 1], m[:, 2], rng.uniform(-side, side, 3)]).astype(np.float32))
    return out, side


class Top:
    """A top-level scene of instances of `child`, committed under one arm's threshold."""

    def __init__(self, lib, dev, child, xfms, arm):
        self.lib, self.dev, self.xfms, self.arm = lib, dev, [x.copy() for x in xfms], arm
        self.sc = lib.rtcNewScene(dev)
        lib.rtcSetSceneBuildQuality(self.sc, RTC_BUILD_QUALITY_MEDIUM)
        self.ids = [lib.add_instance(dev, self.sc, child, m) for m in self.xfms]

    def commit(self):
        """wall-clock ms of rtcCommitScene, None when the commit failed"""
        assert self.lib.rtcb200SetTuning(b"instance_flatten_max", FORCE[self.arm]) == 0
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        self.lib.rtcCommitScene(self.sc)
        ms = (time.perf_counter() - t0) * 1e3
        self.error = self.lib.rtcGetDeviceError(self.dev)
        if self.error:
            self.error = f"commit failed (RTCError {self.error}: {self.lib.rtcGetDeviceLastErrorMessage(self.dev).decode()})"
            return None
        # the arm took its path: only instance-traversal scenes refuse device-side queries
        inst = self.lib.scene_device_traversable(self.sc).nodes is None
        self.lib.rtcGetDeviceError(self.dev)
        assert inst == (self.arm == INST), (self.arm, inst)
        return ms

    def move(self, k, step):
        for i in range(k):
            self.xfms[i][9] += np.float32(step)
            g = self.lib.rtcGetGeometry(self.sc, self.ids[i])
            self.lib.rtcSetGeometryTransform(g, 0, RTC_FORMAT_FLOAT3X4_COLUMN_MAJOR, _ptr(self.xfms[i]))
            self.lib.rtcCommitGeometry(g)

    def bytes(self):
        s = self.lib.scene_stats(self.sc)
        return int(s.node_bytes + s.tri_bytes)

    def release(self):
        self.lib.rtcReleaseScene(self.sc)


def trace(lib, sc, rays):
    """(ms of one rtcb200Intersect1MDevice launch, the records it wrote); rays: [n, 24] float32 on the GPU"""
    buf = rays.clone()
    a = lib.args()
    st = torch.cuda.current_stream()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record(st)
    lib.rtcb200Intersect1MDevice(sc, C.c_void_p(buf.data_ptr()), buf.shape[0], C.byref(a), C.c_void_p(st.cuda_stream))
    e1.record(st)
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), buf


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--phi", type=int, default=500)
    ap.add_argument("--counts", default="2,4,16,256,4096,65536")
    ap.add_argument("--width", type=int, default=1024)
    args = ap.parse_args()
    lib = embree_b200.load()
    dev = lib.new_device(None)
    v, t = scenes.triangle_sphere(args.phi)
    child = lib.rtcNewScene(dev)
    lib.rtcSetSceneBuildQuality(child, RTC_BUILD_QUALITY_MEDIUM)
    keep = lib.add_triangle_mesh(dev, child, v, t, mask=0xFFFFFFFF)
    lib.rtcCommitScene(child)
    lib.check(dev)
    shipped = None
    with open(os.path.join(ROOT, "embree_b200", "csrc", "rtk_device.h")) as f:
        for line in f:
            if "int instance_flatten_max" in line:
                shipped = int(line.split("=")[1].split(";")[0])
    out = {"gpu": gpu_info(), "child_triangles": int(len(t)), "reps": args.reps, "instance_flatten_max": shipped, "scale": [], "edits": []}
    for n in [int(x) for x in args.counts.split(",")]:
        xf, side = transforms(n, seed=n)
        cam = scenes.primary_rays(args.width, args.width, eye=(0.0, 0.0, -3.0 * side), look=(0.0, 0.0, 1.0), fov=60.0).cuda()
        row = {"instances": n, "flattened_records": n * int(len(t))}
        res = {arm: {"commit_ms": [], "bytes": None, "camera_ms": [], "bounce_ms": [], "failed": False} for arm in (FLAT, INST)}
        if row["flattened_records"] > MAX_PRIMS:
            res[FLAT]["failed"] = f"cannot be flattened: more than {MAX_PRIMS} records"
        recs = {}
        bounce = None
        for rep in range(args.reps + 1):
            for arm in (INST, FLAT):
                r = res[arm]
                if r["failed"]:
                    continue
                top = Top(lib, dev, child, xf, arm)
                ms = top.commit()
                if ms is None:
                    r["failed"] = top.error
                    top.release()
                    continue
                r["bytes"] = top.bytes()
                cms, chits = trace(lib, top.sc, cam)
                if bounce is None:
                    bounce = scenes.diffuse_bounce_rays(chits.cpu(), seed=1).cuda()
                bms, bhits = trace(lib, top.sc, bounce)
                if rep:
                    r["commit_ms"].append(ms); r["camera_ms"].append(cms); r["bounce_ms"].append(bms)
                else:
                    recs[arm] = (chits.cpu().numpy(), bhits.cpu().numpy())
                top.release()
        nc, nb = cam.shape[0], bounce.shape[0]
        for arm in (FLAT, INST):
            r = res[arm]
            row[arm] = r["failed"] if r["failed"] else {
                "commit_ms": stat(r["commit_ms"]), "scene_bytes": r["bytes"],
                "camera_mrays_s": stat([nc / ms * 1e-3 for ms in r["camera_ms"]]),
                "bounce_mrays_s": stat([nb / ms * 1e-3 for ms in r["bounce_ms"]])}
        if FLAT in recs and INST in recs:   # (c): records of the two arms on the same rays
            cmp = {}
            for k, name in ((0, "camera"), (1, "bounce")):
                a, b = recs[FLAT][k], recs[INST][k]
                diff = (a.view(np.uint32) != b.view(np.uint32)).any(1)
                tie = diff & (a[:, 8].view(np.uint32) == b[:, 8].view(np.uint32))
                cmp[name] = {"rays": int(len(a)), "differ": int(diff.sum()), "of_which_equal_t_ties": int(tie.sum())}
                other = np.nonzero(diff & ~tie)[0][:4]   # tfar, Ng, u, v, primID, geomID, instID of the rest, flattened then instance traversal
                if len(other):
                    cmp[name]["others"] = [[a[i, 8:21].view(np.uint32).tolist(), b[i, 8:21].view(np.uint32).tolist()] for i in other]
            row["records"] = cmp
        else:
            row["records"] = "not measured"
        out["scale"].append(row)
        print(json.dumps(row), file=sys.stderr, flush=True)
        # (b): re-commit after moving some instances
        if n in (16, 4096):   # (b)
            erow = {"instances": n}
            for frac in (0.01, 1.0):
                k = max(1, int(round(frac * n)))
                times = {INST: [], FLAT: []}
                arms = (INST, FLAT) if n * int(len(t)) <= MAX_PRIMS else (INST,)
                tops = {arm: Top(lib, dev, child, xf, arm) for arm in arms}
                ok = {arm: tops[arm].commit() is not None for arm in tops}
                for rep in range(args.reps + 1):
                    for arm in arms:
                        if not ok[arm]:
                            continue
                        tops[arm].move(k, 0.25 if rep % 2 == 0 else -0.25)
                        ms = tops[arm].commit()
                        if ms is None:
                            ok[arm] = False
                        elif rep:
                            times[arm].append(ms)
                erow[f"moved_{k}"] = {arm: (stat(times[arm]) if ok[arm] else tops[arm].error) for arm in tops}
                for arm in tops:
                    tops[arm].release()
            out["edits"].append(erow)
            print(json.dumps(erow), file=sys.stderr, flush=True)
    lib.rtcReleaseScene(child)
    lib.rtcReleaseDevice(dev)
    del keep
    print(json.dumps(out))


if __name__ == "__main__":
    main()
