"""In-tree builds: the CUDA C-ABI library (nvcc, sm_90a), the CPU oracle and the host-emulation
harness used by the CPU-only logic tests.  Artefacts stay next to the sources."""
from __future__ import annotations

import os
import subprocess
import sys

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
CSRC = os.path.join(_HERE, "csrc")
LIB = os.path.join(_HERE, "libimmesh_b200.so")
EMU = os.path.join(_ROOT, "tests", "emu", "libimmesh_emu.so")
ORACLE = os.path.join(_ROOT, "oracle", "liborc.so")
REF_IKD = os.path.join(_ROOT, "oracle", "_ref", "libref_ikd.so")
# where the reference checkout lies (oracle/Makefile.ref compiles its ikd-Tree from there when it is present)
REFERENCE = os.environ.get("IMMESH_REFERENCE", "/root/reference")
GXX = "/usr/bin/g++"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-fmad=false",            # numerics contract: no FMA contraction (bit parity with the reference's SSE2 build)
    "-Xcompiler", "-fPIC", "-shared",
]


def _newer(target, sources):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(s) > t for s in sources)


def _sources(dirpath, exts):
    return sorted(os.path.join(dirpath, f) for f in os.listdir(dirpath) if f.endswith(exts))


def build_cuda(force=False, verbose=False):
    cu = _sources(CSRC, (".cu",))
    # this file is a dependency too: a library built with other NVCC_FLAGS (another architecture) is rebuilt
    deps = cu + _sources(CSRC, (".cuh", ".hpp")) + [os.path.join(_ROOT, "include", "immesh_b200.h"), os.path.abspath(__file__)]
    if force or _newer(LIB, deps):
        cmd = ["nvcc", *NVCC_FLAGS, "-ccbin", GXX, "-o", LIB, *cu]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        subprocess.check_call(cmd, cwd=_ROOT)
    return LIB


def build_oracle(force=False):
    src = _sources(os.path.join(_ROOT, "oracle"), (".cpp", ".hpp"))
    if force or _newer(ORACLE, src):
        subprocess.check_call(["make", "-C", os.path.join(_ROOT, "oracle"), "-B"])
    return ORACLE


def build_emu(force=False):
    emu_dir = os.path.join(_ROOT, "tests", "emu")
    src = _sources(emu_dir, (".cpp",))
    deps = src + _sources(CSRC, (".cuh", ".hpp"))
    if force or _newer(EMU, deps):
        cmd = [GXX, "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-Wno-unknown-pragmas", "-I/usr/local/cuda/include", "-shared", "-o", EMU]
        for s in src:
            cmd += ["-x", "c++", s]
        subprocess.check_call(cmd)
    return EMU


PUBMAP_DIR = os.path.join(_ROOT, "tests", "pubmap")
EMU_PUB = os.path.join(PUBMAP_DIR, "libimmesh_emu_pub.so")
ORACLE_PUB = os.path.join(PUBMAP_DIR, "liborc_pub.so")


def _emu_ext(src, out, force, extra=()):
    """a file that includes a tests/emu/ source and extends it, built on its own with the emulation's flags (extra: further
    translation units linked in unchanged)"""
    deps = [src] + _sources(os.path.join(_ROOT, "tests", "emu"), (".cpp",)) + _sources(CSRC, (".cuh", ".hpp"))
    if force or _newer(out, deps):
        cmd = [GXX, "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-Wno-unknown-pragmas", "-I/usr/local/cuda/include", "-shared",
               "-o", out, "-x", "c++", src]
        for e in extra:
            cmd += ["-x", "c++", e]
        subprocess.check_call(cmd)
    return out


def _oracle_ext(src, out, force):
    """a file that includes oracle/orc_capi.cpp and extends it, built on its own with oracle/Makefile's flags"""
    deps = [src] + _sources(os.path.join(_ROOT, "oracle"), (".cpp", ".hpp"))
    if force or _newer(out, deps):
        subprocess.check_call([GXX, "-O3", "-std=c++17", "-fPIC", "-fopenmp", "-ffp-contract=off", "-fno-fast-math", "-Wall", "-Wno-unused-variable",
                               "-shared", "-o", out, src])
    return out


def build_pubmap(force=False):
    """tests/pubmap: the host emulation with the plane-map publisher state attached, and the oracle extended by pubPlaneMap"""
    return (_emu_ext(os.path.join(PUBMAP_DIR, "emu_pub.cpp"), EMU_PUB, force),
            _oracle_ext(os.path.join(PUBMAP_DIR, "orc_pub.cpp"), ORACLE_PUB, force))


EMU_SCANPUB = os.path.join(PUBMAP_DIR, "libimmesh_emu_scanpub.so")
ORACLE_SCANPUB = os.path.join(PUBMAP_DIR, "liborc_scanpub.so")


def build_scanpub(force=False):
    """tests/pubmap: the host emulation with the IESKF weights kept and the two scan publishers (effect / registered cloud), and
    the oracle extended by publish_effect_world / publish_frame_world"""
    return (_emu_ext(os.path.join(PUBMAP_DIR, "emu_scan_pub.cpp"), EMU_SCANPUB, force),
            _oracle_ext(os.path.join(PUBMAP_DIR, "orc_scan_pub.cpp"), ORACLE_SCANPUB, force))


EMU_REGIONBUF = os.path.join(PUBMAP_DIR, "libimmesh_emu_regionbuf.so")
ORACLE_REGIONBUF = os.path.join(PUBMAP_DIR, "liborc_regionbuf.so")


def build_regionbuf(force=False):
    """tests/pubmap: the host emulation of the mesher with the m_smoothed flags and the viewer's region buffers, and the oracle
    extended by the viewer's walk (unparse_triangle_set_to_vector + get_axis_min_max)"""
    return (_emu_ext(os.path.join(PUBMAP_DIR, "emu_region_buf.cpp"), EMU_REGIONBUF, force, extra=[os.path.join(_ROOT, "tests", "emu", "emu_lio.cpp")]),
            _oracle_ext(os.path.join(PUBMAP_DIR, "orc_region_buf.cpp"), ORACLE_REGIONBUF, force))


EMU_BATCHED = os.path.join(_ROOT, "tests", "batched", "libimmesh_emu_batched.so")


def build_batched(force=False):
    """tests/batched: the host emulation of the mesher with the m_smoothed flags and the batched frame's orchestration (the
    localization emulation linked in unchanged: api.load_library binds both handles' entry points)"""
    return _emu_ext(os.path.join(_ROOT, "tests", "batched", "emu_batched.cpp"), EMU_BATCHED, force, extra=[os.path.join(_ROOT, "tests", "emu", "emu_lio.cpp")])


EMU_GROWTH = os.path.join(_ROOT, "tests", "growth", "libimmesh_emu_growth.so")


def build_growth(force=False):
    """tests/growth: the host emulation with the plane-map publisher's state and the pool growth of immesh_lio_reserve /
    immesh_lio_set_growth (the migration bodies and the growth policy of immesh_b200/csrc/pool_growth.cuh)"""
    return _emu_ext(os.path.join(_ROOT, "tests", "growth", "emu_growth.cpp"), EMU_GROWTH, force)


EMU_IMU_CHAIN = os.path.join(_ROOT, "tests", "imu_chain", "libimmesh_emu_imu_chain.so")


def build_imu_chain(force=False):
    """tests/imu_chain: the device interval plan and IMU_init's host body of the IMU-enabled scan loop, built for the host"""
    return _emu_ext(os.path.join(_ROOT, "tests", "imu_chain", "emu_imu_chain.cpp"), EMU_IMU_CHAIN, force)


EMU_DEPTH_IMU = os.path.join(_ROOT, "tests", "depth_imu", "libimmesh_emu_depth_imu.so")


def build_depth_imu(force=False):
    """tests/depth_imu: the depth IMU chain's device decision (sync_packages' drop and carry, the branch, IMU_init) built for the host"""
    return _emu_ext(os.path.join(_ROOT, "tests", "depth_imu", "emu_depth_imu.cpp"), EMU_DEPTH_IMU, force)


EMU_REINFORCE = os.path.join(_ROOT, "tests", "reinforce", "libimmesh_emu_reinforce.so")


def build_reinforce(force=False):
    """tests/reinforce: the reinforcement's camera pose and tiled rasteriser bodies (immesh_b200/csrc/reinforce.cuh), built for the host"""
    return _emu_ext(os.path.join(_ROOT, "tests", "reinforce", "emu_reinforce.cpp"), EMU_REINFORCE, force)


EMU_VIEW = os.path.join(_ROOT, "tests", "view", "libimmesh_emu_view.so")


def build_view(force=False):
    """tests/view: the shaded view's visibility, shading and height-colour bodies and its camera sources (immesh_b200/csrc/reinforce.cuh)
    in the tiled rasteriser's orchestration, built for the host"""
    return _emu_ext(os.path.join(_ROOT, "tests", "view", "emu_view.cpp"), EMU_VIEW, force)


EMU_TEXTURE = os.path.join(_ROOT, "tests", "texture", "libimmesh_emu_texture.so")


def build_texture(force=False):
    """tests/texture: the texture selection's bodies (immesh_b200/csrc/texture_core.cuh, with the rasteriser's of reinforce.cuh) in the
    device chain's orchestration -- binning, tiles, the per-facet test and the rows -- built for the host"""
    src = os.path.join(_ROOT, "tests", "texture", "emu_texture.cpp")
    deps = [src] + _sources(CSRC, (".cuh",)) + [os.path.join(_ROOT, "include", "immesh_b200.h")]
    if force or _newer(EMU_TEXTURE, deps):
        subprocess.check_call([GXX, "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-Wall", "-Wno-unknown-pragmas", "-I/usr/local/cuda/include", "-shared",
                               "-o", EMU_TEXTURE, src])
    return EMU_TEXTURE


EMU_TEXTURE_ONLINE = os.path.join(_ROOT, "tests", "texture_online", "libimmesh_emu_texture_online.so")


def build_texture_online(force=False):
    """tests/texture_online: the queued texturing's bodies (immesh_b200/csrc/texture_core.cuh, with the rasteriser's of reinforce.cuh)
    in the device stage's orchestration -- the frame's camera, the per-slot counts, the update, the state's growth, the rows and the
    frames list -- built for the host"""
    src = os.path.join(_ROOT, "tests", "texture_online", "emu_texture_online.cpp")
    deps = [src] + _sources(CSRC, (".cuh",)) + [os.path.join(_ROOT, "include", "immesh_b200.h")]
    if force or _newer(EMU_TEXTURE_ONLINE, deps):
        subprocess.check_call([GXX, "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-Wall", "-Wno-unknown-pragmas", "-I/usr/local/cuda/include", "-shared",
                               "-o", EMU_TEXTURE_ONLINE, src])
    return EMU_TEXTURE_ONLINE


EMU_TEXTURE_BAKE = os.path.join(_ROOT, "tests", "texture_bake", "libimmesh_emu_texture_bake.so")


def build_texture_bake(force=False):
    """tests/texture_bake: the texture atlas's bodies and argument check (immesh_b200/csrc/texture_bake_core.cuh) in the device call's
    orchestration -- class and key, the stable sort, the class table, placement and the texels of every slot -- built for the host"""
    src = os.path.join(_ROOT, "tests", "texture_bake", "emu_texture_bake.cpp")
    deps = [src] + _sources(CSRC, (".cuh",)) + [os.path.join(_ROOT, "include", "immesh_b200.h")]
    if force or _newer(EMU_TEXTURE_BAKE, deps):
        subprocess.check_call([GXX, "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-Wall", "-Wno-unknown-pragmas", "-shared",
                               "-o", EMU_TEXTURE_BAKE, src])
    return EMU_TEXTURE_BAKE


EMU_TEXTURE_RENDER = os.path.join(_ROOT, "tests", "texture_render", "libimmesh_emu_texture_render.so")


def build_texture_render(force=False):
    """tests/texture_render: the textured render's bodies and argument check (immesh_b200/csrc/texture_render_core.cuh, with the bake's
    scaling, bilinear sample and batch plan and the rasteriser's bodies) in the device call's orchestration -- binning, tiles, the
    needed check, pass B per host-image batch and the score -- built for the host"""
    src = os.path.join(_ROOT, "tests", "texture_render", "emu_texture_render.cpp")
    deps = [src] + _sources(CSRC, (".cuh",)) + [os.path.join(_ROOT, "include", "immesh_b200.h")]
    if force or _newer(EMU_TEXTURE_RENDER, deps):
        subprocess.check_call([GXX, "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-Wall", "-Wno-unknown-pragmas", "-I/usr/local/cuda/include", "-shared",
                               "-o", EMU_TEXTURE_RENDER, src])
    return EMU_TEXTURE_RENDER


EMU_TEXTURE_GAINS = os.path.join(_ROOT, "tests", "texture_gains", "libimmesh_emu_texture_gains.so")


def build_texture_gains(force=False):
    """tests/texture_gains: the colour equalisation's bodies, argument check and host solve (immesh_b200/csrc/texture_gains_core.cuh, with
    the bake's scaling and batch plan, the selection's "seen" test and the rasteriser's bodies) in the device call's orchestration --
    chosen side, observer passes per host-image batch, compaction and solve -- and the gains' host apply, built for the host"""
    src = os.path.join(_ROOT, "tests", "texture_gains", "emu_texture_gains.cpp")
    deps = [src] + _sources(CSRC, (".cuh",)) + [os.path.join(_ROOT, "include", "immesh_b200.h")]
    if force or _newer(EMU_TEXTURE_GAINS, deps):
        subprocess.check_call([GXX, "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-Wall", "-Wno-unknown-pragmas", "-I/usr/local/cuda/include", "-shared",
                               "-o", EMU_TEXTURE_GAINS, src])
    return EMU_TEXTURE_GAINS


EMU_VIEW_OVERLAY = os.path.join(_ROOT, "tests", "view_overlay", "libimmesh_emu_view_overlay.so")


def build_view_overlay(force=False):
    """tests/view_overlay: the queued view's overlay bodies (immesh_b200/csrc/view_overlay.cuh) -- points, clipped wide lines, the
    wireframe, the frustum, the trajectory ring and the layered key -- in the device chain's orchestration, built for the host"""
    return _emu_ext(os.path.join(_ROOT, "tests", "view_overlay", "emu_view_overlay.cpp"), EMU_VIEW_OVERLAY, force)


EMU_CHANGES = os.path.join(_ROOT, "tests", "changes", "libimmesh_emu_changes.so")


def build_changes(force=False):
    """tests/changes: the host emulation of the mesher and the batched frame with the change feed's bodies (mesh_changes.cuh) run in
    the device's order (the localization emulation linked in unchanged)"""
    return _emu_ext(os.path.join(_ROOT, "tests", "changes", "emu_changes.cpp"), EMU_CHANGES, force,
                    extra=[os.path.join(_ROOT, "tests", "emu", "emu_lio.cpp")])


EMU_LIO_FEED = os.path.join(_ROOT, "tests", "lio_feed", "libimmesh_emu_lio_feed.so")


def build_lio_feed(force=False):
    """tests/lio_feed: the scan feed's ring bookkeeping and read (immesh_b200/csrc/lio_feed.cuh) with the device kernels' order restated
    on the host"""
    return _emu_ext(os.path.join(_ROOT, "tests", "lio_feed", "emu_lio_feed.cpp"), EMU_LIO_FEED, force)


EMU_LIO_FEED_MARKERS = os.path.join(_ROOT, "tests", "lio_feed", "libimmesh_emu_lio_feed_markers.so")


def build_lio_feed_markers(force=False):
    """tests/lio_feed: the scan feed's plane-marker rings (marker_append, plane_pub_at, feed_read on marker_rings) with the device
    kernels' order restated on the host"""
    return _emu_ext(os.path.join(_ROOT, "tests", "lio_feed", "emu_lio_feed_markers.cpp"), EMU_LIO_FEED_MARKERS, force)


EMU_MESH_FEED = os.path.join(_ROOT, "tests", "mesh_feed", "libimmesh_emu_mesh_feed.so")


def build_mesh_feed(force=False):
    """tests/mesh_feed: the frame feed's ring bookkeeping (immesh_b200/csrc/mesh_feed.cuh) and the shared read (feed_read) with the
    device kernels' order restated on the host"""
    return _emu_ext(os.path.join(_ROOT, "tests", "mesh_feed", "emu_mesh_feed.cpp"), EMU_MESH_FEED, force)


RS_CHECK = os.path.join(_ROOT, "tests", "radix_sort", "librs_check.so")


def build_rs_check(force=False):
    """tests/radix_sort: the radix sort (immesh_b200/csrc/radix_sort.cuh) with a host count and with a device count on a chosen grid"""
    src = os.path.join(_ROOT, "tests", "radix_sort", "rs_check.cu")
    if force or _newer(RS_CHECK, [src, os.path.join(CSRC, "radix_sort.cuh"), os.path.abspath(__file__)]):
        subprocess.check_call(["nvcc", *NVCC_FLAGS, "-ccbin", GXX, "-o", RS_CHECK, src], cwd=_ROOT)
    return RS_CHECK


EMU_EVAL = os.path.join(_ROOT, "tests", "eval", "libimmesh_emu_eval.so")


def build_eval(force=False):
    """tests/eval: the evaluation's per-element bodies (immesh_b200/csrc/mesh_eval.cuh) in a sequential host evaluator"""
    src = os.path.join(_ROOT, "tests", "eval", "emu_eval.cpp")
    if force or _newer(EMU_EVAL, [src, os.path.join(CSRC, "mesh_eval.cuh"), os.path.join(CSRC, "hd_math.cuh")]):
        subprocess.check_call([GXX, "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-Wall", "-Wno-unknown-pragmas", "-I/usr/local/cuda/include", "-shared", "-o", EMU_EVAL, src])
    return EMU_EVAL


EMU_DEPTH_FRAME = os.path.join(_ROOT, "tests", "depth_frame", "libimmesh_emu_depth_frame.so")


def build_depth_frame(force=False):
    """tests/depth_frame: the depth frame's unprojection and append-step bodies (immesh_b200/csrc/depth_frame.cuh) with the device
    kernels' compaction restated on the host"""
    src = os.path.join(_ROOT, "tests", "depth_frame", "emu_depth_frame.cpp")
    deps = [src, os.path.join(CSRC, "depth_frame.cuh"), os.path.join(CSRC, "hd_math.cuh"), os.path.join(_ROOT, "include", "immesh_b200.h")]
    if force or _newer(EMU_DEPTH_FRAME, deps):
        subprocess.check_call([GXX, "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-Wall", "-Wno-unknown-pragmas", "-I/usr/local/cuda/include", "-shared",
                               "-o", EMU_DEPTH_FRAME, src])
    return EMU_DEPTH_FRAME


EMU_DEPTH_LIO = os.path.join(_ROOT, "tests", "depth_lio", "libimmesh_emu_depth_lio.so")


def build_depth_lio(force=False):
    """tests/depth_lio: the localization's depth filter (immesh_b200/csrc/depth_frame.cuh: depth_point, depth_keep) with the front-end
    kernels' multi-pass block compaction restated on the host"""
    src = os.path.join(_ROOT, "tests", "depth_lio", "emu_depth_lio.cpp")
    deps = [src, os.path.join(CSRC, "depth_frame.cuh"), os.path.join(CSRC, "hd_math.cuh"), os.path.join(_ROOT, "include", "immesh_b200.h")]
    if force or _newer(EMU_DEPTH_LIO, deps):
        subprocess.check_call([GXX, "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-Wall", "-Wno-unknown-pragmas", "-I/usr/local/cuda/include", "-shared",
                               "-o", EMU_DEPTH_LIO, src])
    return EMU_DEPTH_LIO


LOCAL_MAP_DIR = os.path.join(_ROOT, "tests", "local_map")
EMU_LOCAL_MAP = os.path.join(LOCAL_MAP_DIR, "libimmesh_emu_local_map.so")
ORACLE_LOCAL_MAP = os.path.join(LOCAL_MAP_DIR, "liborc_local_map.so")


def build_local_map(force=False):
    """tests/local_map: the host emulation with the local map's box rule, eviction sweep and purge (immesh_b200/csrc/local_map.cuh),
    and the oracle extended by laser_map_fov_segment and the deletion of the boxes it leaves behind"""
    return (_emu_ext(os.path.join(LOCAL_MAP_DIR, "emu_local_map.cpp"), EMU_LOCAL_MAP, force),
            _oracle_ext(os.path.join(LOCAL_MAP_DIR, "orc_local_map.cpp"), ORACLE_LOCAL_MAP, force))


DEV_MEM_DIR = os.path.join(_ROOT, "tests", "dev_mem")
EMU_DEV_MEM = os.path.join(DEV_MEM_DIR, "libdev_mem_emu.so")


def build_dev_mem(force=False):
    """tests/dev_mem: the handles' memory owner (immesh_b200/csrc/dev_mem.hpp) built for the host against allocation stubs that
    can fail on demand (-Bsymbolic: the stubs, not a CUDA runtime loaded earlier in the process, serve its calls)"""
    src = os.path.join(DEV_MEM_DIR, "emu_dev_mem.cpp")
    if force or _newer(EMU_DEV_MEM, [src, os.path.join(CSRC, "dev_mem.hpp")]):
        subprocess.check_call([GXX, "-O2", "-std=c++17", "-fPIC", "-Wall", "-I/usr/local/cuda/include", "-shared", "-Wl,-Bsymbolic", "-o", EMU_DEV_MEM, src])
    return EMU_DEV_MEM


def build_ref():
    """oracle/_ref: the reference's own ikd-Tree compiled unmodified from the reference checkout, where one is present;
    elsewhere a library built earlier is used, and the tests that need it skip when there is none."""
    if os.path.isdir(os.path.join(REFERENCE, "include", "ikd-Tree")):
        subprocess.check_call(["make", "-s", "-C", os.path.join(_ROOT, "oracle"), "-f", "Makefile.ref", f"REF={REFERENCE}"])
    return REF_IKD


def build_all(force=False):
    build_cuda(force)
    build_oracle(force)
    build_emu(force)
    build_pubmap(force)
    build_scanpub(force)
    build_regionbuf(force)
    build_batched(force)
    build_growth(force)
    build_imu_chain(force)
    build_depth_imu(force)
    build_reinforce(force)
    build_view(force)
    build_view_overlay(force)
    build_texture(force)
    build_texture_bake(force)
    build_texture_online(force)
    build_texture_render(force)
    build_texture_gains(force)
    build_changes(force)
    build_lio_feed(force)
    build_lio_feed_markers(force)
    build_mesh_feed(force)
    build_rs_check(force)
    build_eval(force)
    build_depth_frame(force)
    build_depth_lio(force)
    build_local_map(force)
    build_dev_mem(force)
    build_ref()


if __name__ == "__main__":
    build_all(force="--force" in sys.argv)
    print("built:", LIB, ORACLE, EMU)
