"""rtcInterpolate arithmetic on the CPU: the host instantiation of embree_b200/csrc/interp.cuh (tests/interp_emu, emu_interpolate) against
the unmodified reference's answers for every curve type (tests/golden/reference/interpolate_curves.npz) and for the triangle / quad
meshes of the golden quads fixture (interpolate_quads.npz), bit for bit, plus the reference verify suite's own interpolation
formulas (InterpolateTrianglesTest / InterpolateHairTest, tutorials/verify/verify.cpp:2181-2440) within their 1e-4."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from embree_b200.rtc import RTC_BUFFER_TYPE_VERTEX
from tests.conftest import load_golden
from tests.interp_cases import BUFFERS, CURVE_TYPES, SENTINEL, curve_case, host_answers, make_geometry
from tests.parity import REFERENCE_GOLDEN, reference_outputs

LINEAR = ("round_linear", "flat_linear")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def interp_emu():
    """tests/interp_emu/_build/libinterp_emu.so, (re)built here as the `emu` fixture builds tests/emu."""
    subprocess.check_call([os.path.join(ROOT, "tests", "interp_emu", "build.sh")])
    return C.CDLL(os.path.join(ROOT, "tests", "interp_emu", "_build", "libinterp_emu.so"))


def _emu_fn(interp_emu):
    f = interp_emu.emu_interpolate
    f.argtypes = [C.c_uint, C.c_uint, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p,
                  C.c_void_p, C.c_uint64, C.c_uint] + [C.c_void_p] * 6
    return f


def reference_curve_answers():
    """{type: {P, dPdu, ddPdudu[, dPdu_alone]}} of the reference's rtcInterpolate on curve_case(type) (flattened per query)."""
    def run(R):
        dev = R.new_device(None)
        out = {}
        for name in CURVE_TYPES:
            case = curve_case(name)
            g, keep = make_geometry(R, dev, name, case)
            a = host_answers(R, g, case)
            for k, x in a.items():
                out[f"{name}__{k}"] = x
            if name in LINEAR:   # the reference loses dPdu when ddPdudu is asked for: record dPdu asked for alone too
                out[f"{name}__dPdu_alone"] = host_answers(R, g, case, dpdu_only=True)["dPdu"]
            R.check(dev)
            R.rtcReleaseGeometry(g)
        R.rtcReleaseDevice(dev)
        return out
    flat = reference_outputs("interpolate_curves", run)[0]
    res = {}
    for k, x in flat.items():
        name, _, f = k.partition("__")
        res.setdefault(name, {})[f] = x
    return res


def emu_answers(interp_emu, name, case, outputs=("P", "dPdu", "ddPdudu")):
    """emu_interpolate of every query of `case`, flattened as host_answers() flattens (value k of query q at offs[q] + k)."""
    f = _emu_fn(interp_emu)
    _t, kind_v, kind_a, basis = CURVE_TYPES[name]
    offs = np.concatenate([[0], np.cumsum(case["vc"])])
    res = {k: np.full(offs[-1], SENTINEL, np.float32) for k in ("P", "dPdu", "ddPdudu")}
    tang = case["tangents"]
    for b, (btype, _slot, floats, _fmt, counts) in enumerate(BUFFERS):
        data = case["verts"] if b == 0 else case["attr0"] if b == 1 else case["attr1"]
        kind = kind_v if btype == RTC_BUFFER_TYPE_VERTEX else kind_a
        for vc in counts:
            q = np.nonzero((case["buf"] == b) & (case["vc"] == vc))[0]
            prim = np.ascontiguousarray(case["prim"][q])
            u = np.ascontiguousarray(case["u"][q])
            v = np.zeros_like(u)
            out = {k: np.zeros((vc, len(q)), np.float32) for k in ("P", "dPdu", "ddPdudu")}
            dv, d2 = np.zeros((vc, len(q)), np.float32), np.zeros((3, vc, len(q)), np.float32)
            ptr = lambda k: out[k].ctypes.data if k in outputs else None
            f(kind, basis, case["idx"].ctypes.data, 4, data.ctypes.data, 4 * floats, tang.ctypes.data if tang is not None else None, 16,
              prim.ctypes.data, u.ctypes.data, v.ctypes.data, len(q), vc, ptr("P"), ptr("dPdu"), dv.ctypes.data if "dPdu" in outputs else None,
              ptr("ddPdudu"), d2[1].ctypes.data if "ddPdudu" in outputs else None, d2[2].ctypes.data if "ddPdudu" in outputs else None)
            assert not dv.any() and not d2.any()      # a curve has no v-derivatives
            for j, qi in enumerate(q):
                for k in outputs:
                    res[k][offs[qi]:offs[qi + 1]] = out[k][:, j]
    return res


@pytest.fixture(scope="module")
def reference_curves():
    return reference_curve_answers()


@pytest.mark.parametrize("name", list(CURVE_TYPES))
def test_emu_curve_interpolation_matches_the_reference(interp_emu, reference_curves, name):
    case = curve_case(name)
    assert len(case["u"]) >= 2000 and (case["u"] == 0).any() and (case["u"] == 1).any()
    ref, mine = reference_curves[name], emu_answers(interp_emu, name, case)
    assert (ref["P"].view(np.uint32) == mine["P"].view(np.uint32)).all()
    if name not in LINEAR:
        for k in ("dPdu", "ddPdudu"):
            assert (ref[k].view(np.uint32) == mine[k].view(np.uint32)).all(), k
        return
    # The one deliberate difference (scene_line_segments.h:73): asked for dPdu and ddPdudu together, the reference writes zeros into
    # dPdu and leaves ddPdudu unwritten.  Here dPdu is p1 - p0, as the reference computes it when dPdu is asked for alone, and
    # ddPdudu is 0.
    assert (ref["dPdu"] == 0).all() and (ref["ddPdudu"].view(np.uint32) == SENTINEL.view(np.uint32)).all()
    assert (ref["dPdu_alone"].view(np.uint32) == mine["dPdu"].view(np.uint32)).all()
    assert (mine["ddPdudu"] == 0).all() and (mine["dPdu"] != 0).any()


def _basis64(name, u):
    """Basis weights in float64 (bezier_curve.h / bspline_curve.h / catmullrom_curve.h, as the verify suite writes them out)."""
    t, s = u, 1.0 - u
    if "bspline" in name:
        return np.stack([s ** 3, 4 * s ** 3 + t ** 3 + 12 * s * t * s + 6 * t * s * t, 4 * t ** 3 + s ** 3 + 12 * t * s * t + 6 * s * t * s, t ** 3]) / 6
    if "catmull_rom" in name:
        return np.stack([-t * s * s, 2 + t * t * (3 * t - 5), 2 + s * s * (3 * s - 5), -s * t * t]) / 2
    return np.stack([s ** 3, 3 * t * s * s, 3 * t * t * s, t ** 3])


@pytest.mark.parametrize("name", list(CURVE_TYPES))
def test_emu_curve_interpolation_restates_the_verify_formulas(interp_emu, name):
    """InterpolateHairTest (verify.cpp:2356-2440) checks P against the curve evaluated from its control points within 1e-4; so does this,
    for every curve type, buffer and valueCount of curve_case(), relative to the size of the control values."""
    case = curve_case(name)
    mine = emu_answers(interp_emu, name, case, outputs=("P",))
    offs = np.concatenate([[0], np.cumsum(case["vc"])])
    for q in range(0, len(case["vc"]), 7):
        b, vc, i, u = case["buf"][q], int(case["vc"][q]), int(case["idx"][case["prim"][q]]), float(case["u"][q])
        data = (case["verts"] if b == 0 else case["attr0"] if b == 1 else case["attr1"]).reshape(-1).astype(np.float64)
        floats = BUFFERS[b][2]
        row = lambda r: data[r * floats:r * floats + vc]
        if "linear" in name or ("hermite" in name and b != 0):
            want = (1 - u) * row(i) + u * row(i + 1)
            scale = np.abs(np.stack([row(i), row(i + 1)])).max()
        elif "hermite" in name:
            t0, t1 = case["tangents"][i, :vc].astype(np.float64), case["tangents"][i + 1, :vc].astype(np.float64)
            cps = np.stack([row(i), row(i) + t0 / 3, row(i + 1) - t1 / 3, row(i + 1)])
            want = _basis64(name, u) @ cps
            scale = np.abs(cps).max()
        else:
            cps = np.stack([row(i + k) for k in range(4)])
            want = _basis64(name, u) @ cps
            scale = np.abs(cps).max()
        got = mine["P"][offs[q]:offs[q + 1]]
        assert np.abs(got - want).max() <= 1e-4 * max(1.0, scale), (q, got, want)


def test_emu_triangle_and_quad_interpolation_matches_the_reference(interp_emu):
    """The stored reference answers of test_interpolate_matches_the_reference (P, dPdu, dPdv of the vertex buffer at the reference's
    own hits of the golden quads fixture) are what the host instantiation of interp.cuh computes, bit for bit."""
    meshes, _rin, want_i, _o, _b = load_golden("quads")
    queries = want_i[np.nonzero(want_i["geomID"] != 0xFFFFFFFF)[0][:400]]
    ref = np.load(os.path.join(REFERENCE_GOLDEN, "interpolate_quads.npz"))["interp"]
    assert len(ref) == len(queries) > 200
    f = _emu_fn(interp_emu)
    by_id = {gid: (np.ascontiguousarray(v, np.float32), np.ascontiguousarray(t, np.uint32)) for (v, t, gid, _m) in meshes}
    for j, q in enumerate(queries):
        v, t = by_id[int(q["geomID"])]
        kind = 2 if t.shape[1] == 4 else 1
        prim, uu, vv = (np.array([q[k]], dt) for k, dt in (("primID", np.uint32), ("u", np.float32), ("v", np.float32)))
        P, du, dv = (np.zeros(3, np.float32) for _ in range(3))
        f(kind, 0, t.ctypes.data, 4 * t.shape[1], v.ctypes.data, 12, None, 0, prim.ctypes.data, uu.ctypes.data, vv.ctypes.data, 1, 3,
          P.ctypes.data, du.ctypes.data, dv.ctypes.data, None, None, None)
        assert (ref[j].view(np.uint32) == np.stack([P, du, dv]).view(np.uint32)).all(), j
