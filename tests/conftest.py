import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90a); run with -m gpu")


def load_golden(name, robust=False):
    """tests/golden/<name>.npz -> (meshes, rays_in, intersect_out, occluded_out, bounds); records as structured arrays.
    robust=True returns the reference's outputs for the same scene committed with RTC_SCENE_FLAG_ROBUST."""
    from embree_b200.rtc import RAYHIT_DTYPE, RAY_DTYPE, aligned_empty
    z = np.load(os.path.join(ROOT, "tests", "golden", name + ".npz"))
    meshes = [(z[f"v{i}"], z[f"t{i}"], int(z[f"gid{i}"]), int(z[f"mask{i}"])) for i in range(int(z["n_meshes"]))]

    def rec(a, dt):
        out = aligned_empty(a.shape[0], dt)
        out.view(np.uint8).reshape(a.shape)[:] = a
        return out
    sfx = "_robust" if robust else ""
    return (meshes, rec(z["rays_in"], RAYHIT_DTYPE), rec(z["intersect_out" + sfx], RAYHIT_DTYPE),
            rec(z["occluded_out" + sfx], RAY_DTYPE), z["bounds"])


def load_golden_instances(name="instances"):
    """tests/golden/instances.npz -> dict(child=[meshes], top=[meshes], xfms[n,12], inst_masks, first_inst, rays_in,
    intersect_out, occluded_out, bounds): the two-level scene of make_golden.run_instances and the reference's outputs."""
    from embree_b200.rtc import RAYHIT_DTYPE, RAY_DTYPE, aligned_empty
    z = np.load(os.path.join(ROOT, "tests", "golden", name + ".npz"))

    def rec(a, dt):
        out = aligned_empty(a.shape[0], dt)
        out.view(np.uint8).reshape(a.shape)[:] = a
        return out

    def meshes(pre, n):
        return [(z[f"{pre}v{i}"], z[f"{pre}t{i}"], int(z[f"{pre}gid{i}"]), int(z[f"{pre}mask{i}"])) for i in range(n)]
    return dict(child=meshes("c", int(z["n_child"])), top=meshes("m", int(z["n_top"])), xfms=z["xfms"],
                inst_masks=z["inst_masks"], first_inst=int(z["first_inst"]), rays_in=rec(z["rays_in"], RAYHIT_DTYPE),
                intersect_out=rec(z["intersect_out"], RAYHIT_DTYPE), occluded_out=rec(z["occluded_out"], RAY_DTYPE),
                bounds=z["bounds"])


def load_golden_curves(name="curves"):
    """tests/golden/curves.npz -> dict(meshes, curves=[(verts4, idx, flags or None, geomID, mask)], rays_in, intersect_out,
    occluded_out, bounds): triangle meshes + round linear curve sets and the reference's outputs (make_golden.run_curves)."""
    from embree_b200.rtc import RAYHIT_DTYPE, RAY_DTYPE, aligned_empty
    z = np.load(os.path.join(ROOT, "tests", "golden", name + ".npz"))

    def rec(a, dt):
        out = aligned_empty(a.shape[0], dt)
        out.view(np.uint8).reshape(a.shape)[:] = a
        return out
    meshes = [(z[f"v{i}"], z[f"t{i}"], int(z[f"gid{i}"]), int(z[f"mask{i}"])) for i in range(int(z["n_meshes"]))]
    curves = [(z[f"cv{i}"], z[f"ci{i}"], z[f"cf{i}"] if z[f"cf{i}"].size else None, int(z[f"cgid{i}"]), int(z[f"cmask{i}"]),
               bool(int(z[f"cflat{i}"])) if f"cflat{i}" in z else False) for i in range(int(z["n_curves"]))]
    return dict(meshes=meshes, curves=curves, rays_in=rec(z["rays_in"], RAYHIT_DTYPE), intersect_out=rec(z["intersect_out"], RAYHIT_DTYPE),
                occluded_out=rec(z["occluded_out"], RAY_DTYPE), bounds=z["bounds"])


def load_golden_cubic(name="curves_cubic"):
    """tests/golden/curves_cubic.npz -> dict(meshes, cubics=[(verts4, idx, geomID, mask, basis, tess or None, tangents or None)],
    rays_in, intersect_out, occluded_out, bounds): flat Bezier / B-spline / Catmull-Rom / Hermite curve sets around a triangle
    sphere and the reference's outputs (make_golden.main_cubic_curves)."""
    from embree_b200.rtc import RAYHIT_DTYPE, RAY_DTYPE, aligned_empty
    from tests.golden.make_golden_sets import CUBIC_SETS
    z = np.load(os.path.join(ROOT, "tests", "golden", name + ".npz"))

    def rec(a, dt):
        out = aligned_empty(a.shape[0], dt)
        out.view(np.uint8).reshape(a.shape)[:] = a
        return out
    cubics = []
    for i in range(int(z["n_sets"])):
        tess = int(z[f"ctess{i}"])
        tg = z[f"ctang{i}"]
        cubics.append((z[f"cv{i}"], z[f"ci{i}"], int(z[f"cgid{i}"]), int(z[f"cmask{i}"]), CUBIC_SETS[i][0], tess if tess else None,
                       tg if tg.size else None, bool(int(z["round"])) if "round" in z else False))
    return dict(meshes=[(z["v0"], z["t0"], 0, 0xFFFFFFFF)], cubics=cubics, rays_in=rec(z["rays_in"], RAYHIT_DTYPE),
                intersect_out=rec(z["intersect_out"], RAYHIT_DTYPE), occluded_out=rec(z["occluded_out"], RAY_DTYPE), bounds=z["bounds"])


def load_golden_points(name="points"):
    """tests/golden/points.npz -> dict(meshes, points=[(verts4, kind, normals or None, geomID, mask)], rays_in, intersect_out,
    occluded_out, bounds): sphere / disc / oriented-disc point sets around a triangle sphere (the scene is rebuilt from its seed by
    make_golden.point_scene, the file holds the rays and the reference's outputs)."""
    from embree_b200.rtc import RAYHIT_DTYPE, RAY_DTYPE, aligned_empty
    from tests.golden.make_golden_sets import point_scene
    z = np.load(os.path.join(ROOT, "tests", "golden", name + ".npz"))

    def rec(a, dt):
        out = aligned_empty(a.shape[0], dt)
        out.view(np.uint8).reshape(a.shape)[:] = a
        return out
    meshes, sets, rays = point_scene()
    rays_in = rec(z["rays_in"], RAYHIT_DTYPE)
    assert rays_in.tobytes() == rays.tobytes(), "point_scene() no longer reproduces the rays of the committed fixture"
    return dict(meshes=meshes, points=sets, rays_in=rays_in, intersect_out=rec(z["intersect_out"], RAYHIT_DTYPE),
                occluded_out=rec(z["occluded_out"], RAY_DTYPE), bounds=z["bounds"])


GOLDEN = ["cube_ground", "sphere21", "terrain_masks"]
GOLDEN_QUADS = ["quads"]   # meshes with [n,4] indices are RTC_GEOMETRY_TYPE_QUAD


@pytest.fixture(scope="session")
def oracle():
    import subprocess
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle")])
    from tests.parity import load_oracle
    return load_oracle()


@pytest.fixture(scope="session")
def emu():
    import ctypes as C
    import subprocess
    subprocess.check_call([os.path.join(ROOT, "tests", "emu", "build.sh")])
    e = C.CDLL(os.path.join(ROOT, "tests", "emu", "_build", "libemu.so"))
    e.emu_build.restype = C.c_void_p
    e.emu_build.argtypes = [C.c_void_p, C.c_uint, C.c_void_p, C.c_uint, C.c_uint, C.c_uint, C.c_int]
    e.emu_trace.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_int, C.c_void_p]
    e.emu_free.argtypes = [C.c_void_p]
    e.emu_num_nodes.argtypes = [C.c_void_p]
    e.emu_depth.argtypes = [C.c_void_p]
    return e


@pytest.fixture(scope="session")
def b200():
    """The product library + a device on cuda:0 (GPU tests only)."""
    import embree_b200
    lib = embree_b200.load()
    dev = lib.new_device(None)
    yield lib, dev
    lib.rtcReleaseDevice(dev)
