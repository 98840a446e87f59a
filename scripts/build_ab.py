"""A/B of library builds on what the builder produces: the same scenes must give the same BVHs (test/bench tool).

    python scripts/build_ab.py [--repeat 2] name=lib.so ...

The first library is the baseline.  It runs `--repeat` times and must agree with itself, otherwise the digests below are not
deterministic and the comparison means nothing; every other library must then equal it, scene for scene.  Each run is its own
process (a library is loaded once per process).

Scenes, all from fixed seeds: every primitive kind (triangles, quads, ROBUST triangles, round / flat linear curves, flat and round
cubic curves in the four bases, the three point kinds) alone and under two instance transforms, with invalid primitives (NaN
vertex, index out of range, negative radius, a cubic curve whose box crosses +-FLT_LARGE), with one primitive only, and a REFIT
re-commit after a vertex move; each at LOW (LBVH) and MEDIUM (SAH) build quality.  Then two seeded edit sequences, at both qualities,
on the commit paths that keep BVHs across commits (two_level_sequence, instance_sequence), digested after every commit.

Per scene the digest holds the rtcGetSceneBounds bytes, the record count (the valid primitives), the sorted multiset of records,
a canonical walk of the BVH (depth-first from the root in slot order, each node's 96 bytes with child_base / tri_base zeroed, each
leaf slot's records in leaf-mask order), and the two-level sub-BVH table and top-level room of rtcb200CopySceneArrays.  A commit of
an edit sequence adds its builder (rtcb200GetSceneStats) and the kernels it launched (rtcb200GetLaunchCount).  Node and record
positions come from atomic counters, so the raw arrays differ from run to run while the walk does not.  At MEDIUM the SAH builder's
tree may itself depend on thread timing: the walk, the sub-BVH table and the launches are compared there only where the baseline
agrees with itself on them."""
import ctypes as C
import hashlib
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

BASES = ("bezier", "bspline", "catmull_rom", "hermite")
STRICT = ("bounds", "count", "multiset", "builder")   # digest keys every run must agree on, at MEDIUM too


def _tris(rng, n):
    v = rng.uniform(-1, 1, (3 * n, 3)).astype(np.float32)
    v = (v.reshape(n, 3, 3) * np.float32(0.1) + rng.uniform(-1, 1, (n, 1, 3)).astype(np.float32)).reshape(-1, 3)
    return v, np.arange(3 * n, dtype=np.uint32).reshape(n, 3)


def _quads(rng, n):
    v = (rng.uniform(-0.1, 0.1, (n, 4, 3)) + rng.uniform(-1, 1, (n, 1, 3))).astype(np.float32).reshape(-1, 3)
    return v, np.arange(4 * n, dtype=np.uint32).reshape(n, 4)


def _linear(rng, n):
    v = np.concatenate([rng.uniform(-1, 1, (n + 1, 3)), rng.uniform(0.005, 0.02, (n + 1, 1))], 1).astype(np.float32)
    return v, np.arange(n, dtype=np.uint32)


def _cubic(rng, n):
    cps = (rng.uniform(-1, 1, (n, 1, 3)) + 0.2 * rng.normal(size=(n, 4, 3))).astype(np.float32)
    rad = rng.uniform(0.005, 0.02, (n, 4, 1)).astype(np.float32)
    return np.concatenate([cps, rad], 2).reshape(-1, 4), np.arange(0, 4 * n, 4, dtype=np.uint32)


def _points(rng, n):
    return np.concatenate([rng.uniform(-1, 1, (n, 3)), rng.uniform(0.005, 0.03, (n, 1))], 1).astype(np.float32)


def add_kind(lib, dev, sc, kind, n, rng, invalid):
    """one geometry of `kind` with n primitives (curves for the cubic kinds); `invalid`: some of them made invalid"""
    if kind in ("triangles", "robust"):
        v, t = _tris(rng, n)
        if invalid and n > 2:
            v[1, 0] = np.nan
            t[2, 1] = len(v) + 5
        return lib.add_triangle_mesh(dev, sc, v, t, mask=0xFFFFFFFF)[1]
    if kind == "quads":
        v, q = _quads(rng, n)
        if invalid and n > 2:
            v[4, 2] = np.nan
            q[2, 3] = len(v) + 1
        return lib.add_quad_mesh(dev, sc, v, q, mask=0xFFFFFFFF)[1]
    if kind in ("round_linear", "flat_linear"):
        v, i = _linear(rng, n)
        if invalid and n > 2:
            v[1, 3] = -0.01
            v[3, 1] = np.nan
            i[-1] = len(v) - 1                      # its second vertex is out of range
        return lib.add_round_linear_curves(dev, sc, v, i, mask=0xFFFFFFFF, flat=kind == "flat_linear")[1]
    if kind.startswith(("flat_", "round_")):
        rnd, basis = kind.split("_", 1)[0] == "round", kind.split("_", 1)[1]
        v, i = _cubic(rng, n)
        if invalid and n > 2:
            c = v.reshape(n, 4, 4)
            c[1, :, :3] = np.float32(1.8e18)         # valid control points, box beyond FLT_LARGE
            c[1, :, 3] = np.float32(1e17)
            c[2, 1, 0] = np.nan
            i[-1] = len(v) - 2
        tg = None
        if basis == "hermite":                       # two vertices + two tangents per curve, as tests/test_bvh_structure.py builds them
            tg = (0.3 * rng.normal(size=v.shape)).astype(np.float32)
            tg[:, 3] *= np.float32(0.01)
        return lib.add_flat_cubic_curves(dev, sc, v, i, basis=basis, tangents=tg, mask=0xFFFFFFFF, round=rnd)
    if kind in ("sphere", "disc", "oriented_disc"):
        v = _points(rng, n)
        if invalid and n > 2:
            v[1, 3] = -0.01
            v[2, 0] = np.inf
        nrm = rng.normal(size=(n, 3)).astype(np.float32) if kind == "oriented_disc" else None
        return lib.add_points(dev, sc, v, kind=kind, normals=nrm, mask=0xFFFFFFFF)
    raise ValueError(kind)


KINDS = ["triangles", "robust", "quads", "round_linear", "flat_linear"] + [f"flat_{b}" for b in BASES] + \
        [f"round_{b}" for b in BASES] + ["sphere", "disc", "oriented_disc"]
XFMS = {"xfm1": [0.8, 0.3, -0.1, -0.2, 0.9, 0.25, 0.15, -0.3, 1.1, 0.5, -1.5, 2.0],
        "xfm2": [0.0, 0.0, 3.0, 0.0, 2.5, 0.0, -4.0, 0.0, 0.0, 1.0e3, 20.0, -7.0]}


def walk_digest(arr):
    nodes, recs = arr["nodes"], arr["records"]
    h = hashlib.sha256()
    if len(nodes) == 0:
        return h.hexdigest()
    stack = [0]
    while stack:
        k = stack.pop()
        w = nodes[k].copy()
        imask, child_base, tri_base = int(w[3] >> 24), int(w[4]), int(w[5])
        w[4] = w[5] = 0
        h.update(w.tobytes())
        lm = nodes[k].view(np.uint8)[24:48]
        kids = []
        for sl in range(8):
            if (imask >> sl) & 1:
                kids.append(child_base + bin(imask & ((1 << sl) - 1)).count("1"))
                continue
            m = int(lm[3 * sl]) | int(lm[3 * sl + 1]) << 8 | int(lm[3 * sl + 2]) << 16
            for b in range(24):
                if (m >> b) & 1:
                    h.update(recs[tri_base + b].tobytes())
        stack.extend(reversed(kids))              # children in slot order
    return h.hexdigest()


def digest(lib, sc):
    from embree_b200.rtc import RTCBounds
    b = RTCBounds()
    lib.rtcGetSceneBounds(sc, C.byref(b))
    arr = lib.scene_arrays(sc)
    recs = arr["records"]
    srt = recs[np.lexsort(recs.T[::-1])] if len(recs) else recs
    return {"bounds": bytes(b).hex(), "count": int(arr["num_records"]), "multiset": hashlib.sha256(srt.tobytes()).hexdigest(),
            "walk": walk_digest(arr), "subs": arr["subs"].tolist(), "top_nodes": int(arr["top_nodes"])}


class Mesh:
    """A triangle geometry on shared host buffers that an edit sequence changes in place."""

    def __init__(self, lib, dev, v, t, quality=None):
        from embree_b200.rtc import RTC_BUFFER_TYPE_VERTEX, RTC_FORMAT_FLOAT3, RTC_GEOMETRY_TYPE_TRIANGLE, _ptr
        self.lib, self.n = lib, len(v)
        self.v = np.zeros(v.size + 4, np.float32)     # 16 B of padding after the last vertex
        self.v[:v.size] = np.ascontiguousarray(v, np.float32).ravel()
        self.g = lib.rtcNewGeometry(dev, RTC_GEOMETRY_TYPE_TRIANGLE)
        lib.rtcSetSharedGeometryBuffer(self.g, RTC_BUFFER_TYPE_VERTEX, 0, RTC_FORMAT_FLOAT3, _ptr(self.v), 0, 12, self.n)
        self.set_indices(t)
        if quality is not None:
            lib.rtcSetGeometryBuildQuality(self.g, quality)
        lib.rtcCommitGeometry(self.g)

    def set_indices(self, t):
        from embree_b200.rtc import RTC_BUFFER_TYPE_INDEX, RTC_FORMAT_UINT3, _ptr
        self.t = np.ascontiguousarray(t, np.uint32).reshape(-1, 3)
        keep = self.t if len(self.t) else np.zeros((1, 3), np.uint32)
        self.lib.rtcSetSharedGeometryBuffer(self.g, RTC_BUFFER_TYPE_INDEX, 0, RTC_FORMAT_UINT3, _ptr(keep), 0, 12, len(self.t))
        self.keep = keep

    def move(self, d):
        from embree_b200.rtc import RTC_BUFFER_TYPE_VERTEX
        self.v[:3 * self.n] += np.tile(np.asarray(d, np.float32), self.n)
        self.lib.rtcUpdateGeometryBuffer(self.g, RTC_BUFFER_TYPE_VERTEX, 0)
        self.lib.rtcCommitGeometry(self.g)


def two_level_sequence(lib, dev, quality, commit):
    """A DYNAMIC scene of 12 small meshes (two of them REFIT) and one of ~100 k triangles: a commit that changes one small mesh is
    two-level, one that changes two is a single BVH.  Edits: moves, REFIT deformation, a mesh moved to another geomID, a geomID
    handed to another geometry object of equal size, a mesh emptied, and two meshes moved at once."""
    from embree_b200 import scenes
    rng = np.random.RandomState(11 + quality)
    sc = lib.rtcNewScene(dev)
    lib.rtcSetSceneFlags(sc, 1)                       # RTC_SCENE_FLAG_DYNAMIC
    lib.rtcSetSceneBuildQuality(sc, quality)
    made, ids = [], {}
    for i in range(12):
        v, t = scenes.triangle_sphere(int(rng.randint(6, 14)), rng.uniform(-3, 3, 3), rng.uniform(0.2, 0.8))
        ids[i] = Mesh(lib, dev, v, t, 3 if i in (2, 7) else None)   # RTC_BUILD_QUALITY_REFIT
    v, t = scenes.triangle_sphere(160, (0.0, -5.0, 0.0), 4.0)
    ids[12] = Mesh(lib, dev, v, t)
    made += ids.values()
    for i, m in ids.items():
        lib.rtcAttachGeometryByID(sc, m.g, i)
    commit(sc, "start")
    edits = ["move", "refit", "id_move", "hand_over", "empty", "two_moves"]
    for k in range(24):
        e = edits[k] if k < len(edits) else edits[rng.randint(len(edits))]
        small = sorted(i for i in ids if ids[i].n < 10000)
        i = small[rng.randint(len(small))]
        if e == "move":
            ids[i].move(rng.uniform(-0.3, 0.3, 3))
        elif e == "refit":
            refit = [j for j in small if ids[j] in (made[2], made[7])] or [i]
            ids[refit[rng.randint(len(refit))]].move(rng.uniform(-0.3, 0.3, 3))
        elif e == "id_move":
            m = ids.pop(i)
            lib.rtcDetachGeometry(sc, i)
            j = max(ids) + 1
            lib.rtcAttachGeometryByID(sc, m.g, j)
            ids[j] = m
        elif e == "hand_over":                        # the same vertices and indices in a new geometry object
            m = ids[i]
            ids[i] = Mesh(lib, dev, m.v[:3 * m.n].reshape(-1, 3), m.t)
            made.append(ids[i])
            lib.rtcDetachGeometry(sc, i)
            lib.rtcAttachGeometryByID(sc, ids[i].g, i)
        elif e == "empty":
            ids[i].set_indices(np.zeros((0, 3), np.uint32))
            lib.rtcCommitGeometry(ids[i].g)
        else:
            a, b = rng.choice(small, 2, replace=False)
            ids[a].move(rng.uniform(-0.3, 0.3, 3))
            ids[b].move(rng.uniform(-0.3, 0.3, 3))
        commit(sc, f"{k}/{e}")
    lib.rtcReleaseScene(sc)
    for m in made:
        lib.rtcReleaseGeometry(m.g)


def instance_sequence(lib, dev, quality, commit):
    """A scene of 12 instances of two instanced scenes beside a mesh of its own, committed with instance traversal.  Edits: an
    instance moved, an instance mask changed, an instanced scene re-committed, instances of a third scene added, all of them removed."""
    from embree_b200 import scenes
    from embree_b200.rtc import RTC_FORMAT_FLOAT3X4_COLUMN_MAJOR, _ptr
    rng = np.random.RandomState(21 + quality)
    children, meshes = [], []
    for c in range(3):
        csc = lib.rtcNewScene(dev)
        lib.rtcSetSceneBuildQuality(csc, quality)
        for _ in range(2):
            v, t = scenes.triangle_sphere(int(rng.randint(8, 16)), rng.uniform(-0.5, 0.5, 3), rng.uniform(0.3, 0.6))
            meshes.append(Mesh(lib, dev, v, t))
            lib.rtcAttachGeometry(csc, meshes[-1].g)
        lib.rtcCommitScene(csc)
        lib.check(dev)
        children.append(csc)
    sc = lib.rtcNewScene(dev)
    lib.rtcSetSceneBuildQuality(sc, quality)
    v, t = scenes.triangle_sphere(20, (0.0, -4.0, 0.0), 2.0)
    meshes.append(Mesh(lib, dev, v, t))
    lib.rtcAttachGeometryByID(sc, meshes[-1].g, 0)

    def xfm():
        q, _r = np.linalg.qr(rng.normal(size=(3, 3)))
        return np.concatenate([q.T.ravel(), rng.uniform(-4, 4, 3)]).astype(np.float32)
    insts, keep = {}, []                              # geomID -> (geometry, instanced scene index)
    for gid in range(1, 13):
        m = xfm()
        keep.append(m)
        lib.add_instance(dev, sc, children[gid % 2], m, geom_id=gid)
        insts[gid] = (lib.rtcGetGeometry(sc, gid), gid % 2)
    commit(sc, "start")
    edits = ["inst_move", "mask", "child_recommit", "add_scene", "remove_scene"]
    for k in range(20):
        e = edits[k] if k < len(edits) else edits[rng.randint(len(edits))]
        gid = sorted(insts)[rng.randint(len(insts))]
        if e == "inst_move":
            m = xfm()
            keep.append(m)
            lib.rtcSetGeometryTransform(insts[gid][0], 0, RTC_FORMAT_FLOAT3X4_COLUMN_MAJOR, _ptr(m))
            lib.rtcCommitGeometry(insts[gid][0])
        elif e == "mask":
            lib.rtcSetGeometryMask(insts[gid][0], int(rng.choice([1, 2, 3, 0xFFFFFFFF])))
            lib.rtcCommitGeometry(insts[gid][0])
        elif e == "child_recommit":
            c = insts[gid][1]
            meshes[2 * c].move(rng.uniform(-0.2, 0.2, 3))
            lib.rtcCommitScene(children[c])
            lib.check(dev)
        elif e == "add_scene":
            for _ in range(3):
                j = max(insts) + 1
                m = xfm()
                keep.append(m)
                lib.add_instance(dev, sc, children[2], m, geom_id=j)
                insts[j] = (lib.rtcGetGeometry(sc, j), 2)
        else:                                         # every instance of the scene of `gid`, unless that empties the scene
            c = insts[gid][1]
            gone = [j for j in insts if insts[j][1] == c]
            if len(gone) < len(insts):
                for j in gone:
                    lib.rtcDetachGeometry(sc, j)
                    del insts[j]
        commit(sc, f"{k}/{e}")
    lib.rtcReleaseScene(sc)
    for csc in children:
        lib.rtcReleaseScene(csc)
    for m in meshes:
        lib.rtcReleaseGeometry(m.g)


def worker(lib_path):
    os.environ["EMBREE_B200_LIB"] = os.path.abspath(lib_path)
    import embree_b200
    from embree_b200.rtc import RTC_BUFFER_TYPE_VERTEX
    lib = embree_b200.load()
    dev = lib.new_device(None)
    out = {}

    def commit(name, quality, build, flags=0):
        rng = np.random.RandomState(int(hashlib.md5(name.encode()).hexdigest()[:7], 16))   # the scene name is its seed
        sc = lib.rtcNewScene(dev)
        lib.rtcSetSceneFlags(sc, flags)
        lib.rtcSetSceneBuildQuality(sc, quality)
        keep = build(sc, rng)
        lib.rtcCommitScene(sc)
        lib.check(dev)
        out[f"{name}/q{quality}"] = digest(lib, sc)
        return sc, keep

    for quality in (0, 1):
        for kind in KINDS:
            flags = 4 if kind == "robust" else 0
            for size, inv in (("n300", False), ("invalid", True), ("one", False)):
                n = {"n300": 300, "invalid": 60, "one": 1}[size]
                sc, keep = commit(f"{kind}/{size}", quality, lambda s, r: add_kind(lib, dev, s, kind, n, r, inv), flags)
                if size != "one":
                    for xn, m in XFMS.items():
                        commit(f"{kind}/{size}/{xn}", quality, lambda s, r: lib.add_instance(dev, s, sc, m), flags)
                lib.rtcReleaseScene(sc)
                del keep
        # REFIT: a dynamic triangle scene re-committed after its vertices moved
        from embree_b200.rtc import RTC_BUFFER_TYPE_INDEX, RTC_FORMAT_FLOAT3, RTC_FORMAT_UINT3, RTC_GEOMETRY_TYPE_TRIANGLE, _ptr
        from embree_b200 import scenes
        v, t = scenes.triangle_sphere(40)
        vpad = np.zeros(v.size + 4, np.float32)
        vpad[:v.size] = v.ravel()
        t = np.ascontiguousarray(t, np.uint32)
        sc = lib.rtcNewScene(dev)
        lib.rtcSetSceneFlags(sc, 1)
        lib.rtcSetSceneBuildQuality(sc, quality)
        g = lib.rtcNewGeometry(dev, RTC_GEOMETRY_TYPE_TRIANGLE)
        lib.rtcSetSharedGeometryBuffer(g, RTC_BUFFER_TYPE_VERTEX, 0, RTC_FORMAT_FLOAT3, _ptr(vpad), 0, 12, len(v))
        lib.rtcSetSharedGeometryBuffer(g, RTC_BUFFER_TYPE_INDEX, 0, RTC_FORMAT_UINT3, _ptr(t), 0, 12, len(t))
        lib.rtcSetGeometryBuildQuality(g, 3)
        lib.rtcCommitGeometry(g)
        lib.rtcAttachGeometry(sc, g)
        lib.rtcCommitScene(sc)
        lib.check(dev)
        out[f"refit/before/q{quality}"] = digest(lib, sc)
        rng = np.random.RandomState(5)
        moved = v * np.float32(1.5) + rng.uniform(-0.01, 0.01, v.shape).astype(np.float32)
        moved[7] = np.nan                         # a triangle that becomes invalid keeps its slot with an empty box
        vpad[:v.size] = np.ascontiguousarray(moved, np.float32).ravel()
        lib.rtcUpdateGeometryBuffer(g, RTC_BUFFER_TYPE_VERTEX, 0)
        lib.rtcCommitGeometry(g)
        lib.rtcCommitScene(sc)
        lib.check(dev)
        assert lib.scene_stats(sc).builder == 2, "expected a refit"
        out[f"refit/after/q{quality}"] = digest(lib, sc)
        lib.rtcReleaseGeometry(g)
        lib.rtcReleaseScene(sc)

    # edit sequences on the paths that keep BVHs across commits; each commit also records its builder and its kernel launches
    def commit_edit(prefix, quality):
        def commit(sc, step):
            n0 = lib.rtcb200GetLaunchCount()
            lib.rtcCommitScene(sc)
            lib.check(dev)
            d = digest(lib, sc)
            d.update(builder=int(lib.scene_stats(sc).builder), launches=int(lib.rtcb200GetLaunchCount() - n0))
            out[f"{prefix}/{step}/q{quality}"] = d
        return commit

    for quality in (0, 1):
        two_level_sequence(lib, dev, quality, commit_edit("two_level_edits", quality))
        assert lib.rtcb200SetTuning(b"instance_flatten_max", 0) == 0
        instance_sequence(lib, dev, quality, commit_edit("instance_edits", quality))
        assert lib.rtcb200SetTuning(b"instance_flatten_max", 2147483647) == 0
    lib.rtcReleaseDevice(dev)
    print(json.dumps(out), flush=True)


def run(lib_path):
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", lib_path], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    lines = [l for l in r.stdout.splitlines() if l.startswith("{")]
    if r.returncode != 0 or not lines:
        raise RuntimeError(f"{lib_path}: rc={r.returncode}\n{r.stderr[-3000:]}")
    return json.loads(lines[-1])


def main(args):
    repeat = 2
    if args and args[0] == "--repeat":
        repeat, args = int(args[1]), args[2:]
    specs = [a.split("=", 1) for a in args]
    base_name, base_lib = specs[0]
    runs = [run(base_lib) for _ in range(repeat)]
    base = runs[0]
    ok = True
    stable = {}
    for s, d in base.items():
        for other in runs[1:]:
            for key in d:
                if (key in STRICT or s.endswith("/q0")) and other[s][key] != d[key]:
                    print(f"{base_name} disagrees with itself: {s} {key}")
                    ok = False
        stable[s] = [k for k in d if all(o[s][k] == d[k] for o in runs[1:])]
    n_unstable = sum(len(stable[s]) < len(d) for s, d in base.items())
    print(f"{base_name}: {len(base)} scenes, {repeat} runs; MEDIUM scenes whose walk, sub-BVH table or launches differ between its own runs: {n_unstable}")
    for name, path in specs[1:]:
        got = run(path)
        diff = []
        for s, d in base.items():
            diff += [f"{s} {k}" for k in stable[s] if got.get(s, {}).get(k) != d[k]]
        print(f"{name}: {len(got)} scenes, {len(diff)} differences from {base_name}" + "".join(f"\n  {x}" for x in diff[:40]))
        ok = ok and not diff and len(got) == len(base)
    print("RESULT", "identical" if ok else "DIFFERENT")
    return 0 if ok else 1


if __name__ == "__main__":
    if sys.argv[1:2] == ["--worker"]:
        worker(sys.argv[2])
        sys.exit(0)
    sys.exit(main(sys.argv[1:]))
