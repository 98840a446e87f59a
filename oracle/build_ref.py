#!/usr/bin/env python3
"""Build the UNMODIFIED reference (Embree 4.4.1) CPU library into oracle/_ref/.

TEST INFRASTRUCTURE ONLY.  The product (embree_b200/) never links or loads
anything produced here; only tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs may use it, as the checker / CPU baseline.

This does NOT run the reference's own build system (CMake).  It compiles the
reference sources *where they lie* under $EMBREE_REFERENCE with g++ through a
ninja file that this script writes, following the source lists in
kernels/CMakeLists.txt:33-195 and common/*/CMakeLists.txt, and the flags in
common/cmake/gnu.cmake:12-92.  Nothing is copied out of the reference tree: the
three headers the reference's CMake would *generate* (rtcore_config.h,
config.h, hash.h; templates kernels/rtcore_config.h.in, kernels/config.h.in,
kernels/hash.h.in) are produced here by substituting the template variables
and written under oracle/_ref/gen/ (git-ignored).

Configuration (all are supported reference build options, CMakeLists.txt:185-214):
  tasking   = INTERNAL        (no TBB in this image)
  ISAs      = SSE2 (base) + AVX + AVX2 + AVX512   (runtime-selected by cpuid)
  geometry  = triangles + quads + curves + points + instances (EMBREE_GEOMETRY_TRIANGLE / QUAD / CURVE / POINT / INSTANCE), ray packets ON,
              ray masks ON, filter functions ON, backface culling OFF  -- the
              reference defaults for every switch that reaches the hot path.

Output: oracle/_ref/libembree4.so.4   (+ libembree4_stat.so.4 with --stat:
        EMBREE_STAT_COUNTERS=ON, used to derive nodes/leaves visited per ray).
"""
import argparse
import os
import re
import subprocess
import sys

REF = os.environ.get("EMBREE_REFERENCE", "")
HERE = os.path.dirname(os.path.abspath(__file__))

MAIN_FILES = """
common/device.cpp common/stat.cpp common/acceln.cpp common/accelset.cpp common/state.cpp
common/rtcore.cpp common/rtcore_builder.cpp common/scene.cpp common/scene_verify.cpp common/alloc.cpp
common/geometry.cpp common/scene_user_geometry.cpp common/scene_instance.cpp common/scene_instance_array.cpp
common/scene_triangle_mesh.cpp common/scene_quad_mesh.cpp common/scene_curves.cpp common/scene_line_segments.cpp
common/scene_grid_mesh.cpp common/scene_points.cpp common/motion_derivative.cpp
subdiv/bezier_curve.cpp subdiv/bspline_curve.cpp subdiv/catmullrom_curve.cpp
geometry/primitive4.cpp geometry/instance_intersector.cpp geometry/instance_array_intersector.cpp
geometry/curve_intersector_virtual_4v.cpp geometry/curve_intersector_virtual_4i.cpp
geometry/curve_intersector_virtual_4i_mb.cpp geometry/curve_intersector_virtual_8v.cpp
geometry/curve_intersector_virtual_8i.cpp geometry/curve_intersector_virtual_8i_mb.cpp
builders/primrefgen.cpp
bvh/bvh.cpp bvh/bvh_statistics.cpp bvh/bvh4_factory.cpp bvh/bvh8_factory.cpp
bvh/bvh_collider.cpp bvh/bvh_rotate.cpp bvh/bvh_refit.cpp bvh/bvh_builder.cpp bvh/bvh_builder_hair.cpp
bvh/bvh_builder_hair_mb.cpp bvh/bvh_builder_morton.cpp bvh/bvh_builder_sah.cpp bvh/bvh_builder_sah_spatial.cpp
bvh/bvh_builder_sah_mb.cpp bvh/bvh_builder_twolevel.cpp bvh/bvh_intersector1_bvh4.cpp
bvh/bvh_intersector_hybrid4_bvh4.cpp
""".split()

COMMON_FILES = """
sys/sysinfo.cpp sys/alloc.cpp sys/filename.cpp sys/library.cpp sys/thread.cpp sys/estring.cpp
sys/regression.cpp sys/mutex.cpp sys/condition.cpp sys/barrier.cpp
math/constants.cpp simd/sse.cpp lexers/stringstream.cpp lexers/tokenstream.cpp
tasking/taskschedulerinternal.cpp
""".split()

SSE2, SSE42, AVX, AVX2, AVX512 = range(5)
ISA_FLAGS = {
    SSE2: "-msse2",
    AVX: "-mavx",
    AVX2: "-mf16c -mavx2 -mfma -mlzcnt -mbmi -mbmi2",
    AVX512: "-march=skylake-avx512",
}
ISA_NAME = {SSE2: "sse2", AVX: "avx", AVX2: "avx2", AVX512: "avx512"}


def isa_files(isa, lowest=SSE2, lowest_avx=AVX):
    """kernels/CMakeLists.txt:122-195 (macro embree_files), packets ON, subdiv OFF."""
    f = """geometry/instance_intersector.cpp geometry/instance_array_intersector.cpp
    geometry/curve_intersector_virtual_4v.cpp geometry/curve_intersector_virtual_4i.cpp
    geometry/curve_intersector_virtual_4i_mb.cpp geometry/curve_intersector_virtual_8v.cpp
    geometry/curve_intersector_virtual_8i.cpp geometry/curve_intersector_virtual_8i_mb.cpp
    bvh/bvh_intersector1_bvh4.cpp""".split()
    if isa == lowest_avx:
        f.append("geometry/primitive8.cpp")
    if isa in (SSE2, AVX, AVX2, AVX512) or isa == lowest:
        f += """common/scene_user_geometry.cpp common/scene_instance.cpp common/scene_instance_array.cpp
        common/scene_triangle_mesh.cpp common/scene_quad_mesh.cpp common/scene_curves.cpp
        common/scene_line_segments.cpp common/scene_grid_mesh.cpp common/scene_points.cpp
        bvh/bvh_collider.cpp bvh/bvh_refit.cpp bvh/bvh_builder.cpp bvh/bvh_builder_hair.cpp
        bvh/bvh_builder_hair_mb.cpp bvh/bvh_builder_sah.cpp bvh/bvh_builder_sah_spatial.cpp
        bvh/bvh_builder_sah_mb.cpp bvh/bvh_builder_twolevel.cpp""".split()
    if isa in (SSE2, AVX, AVX2) or isa == lowest:
        f += "bvh/bvh_builder_morton.cpp bvh/bvh_rotate.cpp builders/primrefgen.cpp".split()
    if isa > SSE42:
        f.append("bvh/bvh_intersector1_bvh8.cpp")
    if isa == AVX:
        f += "bvh/bvh.cpp bvh/bvh_statistics.cpp".split()
    f.append("bvh/bvh_intersector_hybrid4_bvh4.cpp")
    if isa > SSE42:
        f += """bvh/bvh_intersector_hybrid8_bvh4.cpp bvh/bvh_intersector_hybrid4_bvh8.cpp
        bvh/bvh_intersector_hybrid8_bvh8.cpp""".split()
    if isa > AVX2:
        f += "bvh/bvh_intersector_hybrid16_bvh8.cpp bvh/bvh_intersector_hybrid16_bvh4.cpp".split()
    return f


def write_if_changed(path, text):
    """Generated headers keep their time stamp when their content is unchanged, so that a second run rebuilds nothing."""
    if os.path.exists(path) and open(path).read() == text:
        return
    open(path, "w").write(text)


def gen_headers(gen, stat):
    os.makedirs(f"{gen}/include/embree4", exist_ok=True)
    os.makedirs(f"{gen}/kernels/common", exist_ok=True)  # so that "../config.h" resolves via -I
    # --- rtcore_config.h from kernels/rtcore_config.h.in
    t = open(f"{REF}/kernels/rtcore_config.h.in").read()
    subst = {
        "EMBREE_VERSION_MAJOR": "4", "EMBREE_VERSION_MINOR": "4", "EMBREE_VERSION_PATCH": "1",
        "EMBREE_VERSION_NUMBER": "40401", "EMBREE_VERSION_NOTE": "",
        "EMBREE_MAX_INSTANCE_LEVEL_COUNT": "1", "EMBREE_API_NAMESPACE": "",
    }
    defined = {"EMBREE_GEOMETRY_INSTANCE_ARRAY"}  # default ON; fixes RTCHit layout (instPrimID present)
    on01 = {"EMBREE_SYCL_GEOMETRY_CALLBACK": 0, "EMBREE_MIN_WIDTH": 0}

    def cmdef(m):
        name = m.group(1)
        return f"#define {name}" if name in defined else f"/* #undef {name} */"

    def cmdef01(m):
        return f"#define {m.group(1)} {on01.get(m.group(1), 0)}"

    t = re.sub(r"#cmakedefine01 (\w+)", cmdef01, t)
    t = re.sub(r"#cmakedefine (\w+)", cmdef, t)
    t = re.sub(r"@(\w+)@", lambda m: subst[m.group(1)], t)
    write_if_changed(f"{gen}/include/embree4/rtcore_config.h", t)
    # --- config.h from kernels/config.h.in
    t = open(f"{REF}/kernels/config.h.in").read()
    cfg_on = {"EMBREE_RAY_MASK", "EMBREE_FILTER_FUNCTION", "EMBREE_GEOMETRY_TRIANGLE", "EMBREE_GEOMETRY_QUAD", "EMBREE_GEOMETRY_CURVE",
              "EMBREE_GEOMETRY_INSTANCE", "EMBREE_GEOMETRY_POINT", "EMBREE_RAY_PACKETS"}
    if stat:
        cfg_on.add("EMBREE_STAT_COUNTERS")
    t = re.sub(r"#cmakedefine (\w+)",
               lambda m: f"#define {m.group(1)}" if m.group(1) in cfg_on else f"/* #undef {m.group(1)} */", t)
    t = t.replace("@EMBREE_CURVE_SELF_INTERSECTION_AVOIDANCE_FACTOR@", "2.0")
    t = t.replace('#include "../include/embree4/rtcore_config.h"',
                  f'#include "{gen}/include/embree4/rtcore_config.h"')
    write_if_changed(f"{gen}/kernels/config.h", t)
    write_if_changed(f"{gen}/kernels/hash.h", '#define RTC_HASH "0"\n')


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--stat", action="store_true", help="build the EMBREE_STAT_COUNTERS variant")
    ap.add_argument("-j", type=int, default=os.cpu_count())
    a = ap.parse_args()
    if not os.path.isdir(REF):
        print(f"[build_ref] EMBREE_REFERENCE={REF!r} is not a directory -- using prebuilt oracle/_ref if any")
        return 0
    tag = "stat" if a.stat else "rel"
    out = os.path.join(HERE, "_ref")
    gen = os.path.join(out, f"gen_{tag}")
    bld = os.path.join(out, f"build_{tag}")
    os.makedirs(bld, exist_ok=True)
    gen_headers(gen, a.stat)
    lib = os.path.join(out, "libembree4_stat.so.4" if a.stat else "libembree4.so.4")

    base = ("-O3 -DNDEBUG -std=c++11 -fPIC -fvisibility=hidden -fvisibility-inlines-hidden "
            "-fno-strict-aliasing -fno-tree-vectorize -fno-strict-overflow -fno-delete-null-pointer-checks "
            "-fwrapv -fsigned-char -w "
            "-DTASKING_INTERNAL -DEMBREE_TARGET_SSE2 -DEMBREE_TARGET_AVX -DEMBREE_TARGET_AVX2 "
            "-DEMBREE_TARGET_AVX512 "
            f"-I{gen}/include/embree4 -I{gen}/kernels/common -I{gen}/kernels -I{REF}/include")
    n = ["cxx = g++", f"base = {base}",
         "rule cc", "  command = $cxx $base $flags -MMD -MF $out.d -c $in -o $out", "  depfile = $out.d",
         "  deps = gcc", "  description = CC $out",
         "rule link", f"  command = $cxx -shared -o $out $in -Wl,--version-script={REF}/kernels/export.linux.map "
         "-Wl,--no-undefined -Wl,-soname,libembree4.so.4 -lpthread -ldl", "  description = LINK $out",
         "rule ar", "  command = rm -f $out && ar rcs $out $in", "  description = AR $out", ""]
    objs = []

    def add(src, obj, flags, dst=None):
        n.append(f"build {bld}/{obj}: cc {src}")
        n.append(f"  flags = {flags}")
        (objs if dst is None else dst).append(f"{bld}/{obj}")

    for f in COMMON_FILES:
        add(f"{REF}/common/{f}", "c_" + f.replace("/", "_") + ".o", ISA_FLAGS[SSE2])
    for f in MAIN_FILES:
        add(f"{REF}/kernels/{f}", "k_" + f.replace("/", "_") + ".o",
            ISA_FLAGS[SSE2] + " -DEMBREE_LOWEST_ISA -DRTC_EXPORT_API")
    # per-ISA static archives, as the reference does (kernels/CMakeLists.txt:283-352): members that nothing
    # references (e.g. the AVX-512 builders, which have no AVX-512 primrefgen) are dropped by the linker
    archives = []
    for isa in (AVX, AVX2, AVX512):
        iobjs = []
        for f in isa_files(isa):
            add(f"{REF}/kernels/{f}", f"{ISA_NAME[isa]}_" + f.replace("/", "_") + ".o", ISA_FLAGS[isa], iobjs)
        arc = f"{bld}/libembree_{ISA_NAME[isa]}.a"
        n.append(f"build {arc}: ar " + " ".join(iobjs))
        archives.append(arc)
    n.append(f"build {lib}: link " + " ".join(objs) + " " + " ".join(archives))
    n.append(f"default {lib}")
    open(f"{bld}/build.ninja", "w").write("\n".join(n) + "\n")
    r = subprocess.call(["ninja", "-C", bld, f"-j{a.j}"])
    if r == 0:
        subprocess.call(["strip", "--strip-unneeded", lib])
        print(f"[build_ref] built {lib} ({os.path.getsize(lib) >> 20} MiB)")
    return r


if __name__ == "__main__":
    sys.exit(main())
