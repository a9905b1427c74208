"""Cost of a "rebuild tlas" that changes the instance list, the case the device build (kajiya_b200/csrc/kjb_bvh_build.cuh) serves.

For Cornell, the atrium and the ruins it prints one JSON line with, per scene:
  - device_build_ms: CUDA-event time of kjb_rebuild_tlas alternating between the scene's instance list and the same list plus one
    single-triangle instance (every call is a full device build of the whole scene), median of --runs;
  - host_reference_ms: the host binned-SAH builder this project ran before (kajiya_b200/csrc/kjb_bvh.cpp, exported by the emulator
    library) over the same world-space triangles on this machine's CPU, median of --host-runs (flatten and uploads not included);
  - steady_frame_ms / add_frame_ms / remove_frame_ms: wall time of a 480x270 full-path frame (rtdgi, irradiance cache, reflections,
    TAA) ended by a synchronise, with nothing changed, after adding one instance, after removing it again (medians).
It also prints the GPU's name and power limit.  Needs a CUDA device: there is no CPU fallback.

    python tools/bvh_build_bench.py [--scenes cornell,atrium,ruins] [--runs 20]
"""
import argparse, ctypes as C, json, os, subprocess, sys, time
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import kajiya_b200
from kajiya_b200 import scenes
from kajiya_b200.world import World

EMU_SO = os.path.join(ROOT, "tests", "emu", "_build", "libkjb_emu.so")


class Instance(C.Structure):   # kjb_instance (kjb.h)
    _fields_ = [("transform", C.c_float * 12), ("mesh_index", C.c_uint32), ("emissive_multiplier", C.c_float)]


def world_triangles(scene):
    """gid-ordered world-space triangles float32[n, 9], with the library's xform_point (((m0 x + m1 y) + m2 z) + m3, float32)"""
    out = []
    for mesh, transforms in scene:
        p = np.asarray(mesh["positions"], np.float32)[np.asarray(mesh["indices"], np.int64)]
        for t in transforms:
            m = np.asarray(t, np.float32).reshape(12)
            w = np.empty_like(p)
            for r in range(3):
                w[:, r] = ((m[4 * r] * p[:, 0] + m[4 * r + 1] * p[:, 1]) + m[4 * r + 2] * p[:, 2]) + m[4 * r + 3]
            out.append(w.reshape(-1, 9))
    return np.ascontiguousarray(np.concatenate(out))


def host_reference_ms(world_tris, runs):
    d = C.CDLL(EMU_SO)
    d.kjb_ref_bvh_build.restype = C.c_void_p; d.kjb_ref_bvh_build.argtypes = [C.c_void_p, C.c_uint32]
    d.kjb_ref_bvh_free.argtypes = [C.c_void_p]
    ts = []
    for _ in range(runs):
        t0 = time.perf_counter(); h = d.kjb_ref_bvh_build(world_tris.ctypes.data, len(world_tris)); ts.append((time.perf_counter() - t0) * 1e3)
        d.kjb_ref_bvh_free(h)
    return float(np.median(ts))


def instance_array(items):
    arr = (Instance * len(items))()
    for i, (t, mesh) in enumerate(items):
        arr[i].transform[:] = list(np.asarray(t, np.float32).reshape(12)); arr[i].mesh_index = mesh; arr[i].emissive_multiplier = 1.0
    return arr


def tri_mesh():
    p = np.array([[0, 0.05, 0], [0.05, 0.05, 0], [0, 0.1, 0.05]], np.float32)
    return dict(positions=p, normals=np.tile(np.array([[0, 0, 1]], np.float32), (3, 1)), indices=np.arange(3, dtype=np.uint32),
                material_ids=np.zeros(3, np.uint32), materials=[dict(base_color=[0.8, 0.8, 0.8, 1.0], roughness=0.5)])


def measure(lib, name, scene, view, runs, host_runs):
    d = lib.dll
    d.kjb_rebuild_tlas.argtypes, d.kjb_rebuild_tlas.restype = [C.c_void_p, C.c_void_p, C.c_uint32], C.c_int
    kw = dict(enable_ircache=True, enable_rtr=True, enable_taa=True, spatial_reuse_pass_count=2)
    w = World(lib, 480, 270, **kw)
    items = []
    for mesh, transforms in scene:
        h = w.add_mesh(mesh)
        for t in transforms:
            w.add_instance(h, t); items.append((t, h))
    ht = w.add_mesh(tri_mesh())
    w.set_blue_noise(scenes.blue_noise()); w.set_spatial_resolve_offsets(scenes.spatial_resolve_offsets())
    extra = (np.eye(3, 4, dtype=np.float32), ht)
    lists = [instance_array(items), instance_array(items + [extra])]
    for _ in range(6):                      # warm up: modules loaded, capacities for the larger list reserved, graphs instantiated
        w.render_frame(**view)
    w.sync()
    # device build: one rebuild per call, alternating lists; the world's own list is restored below by its next frame
    for k in range(2):
        d.kjb_rebuild_tlas(w.ctx, C.cast(lists[k], C.c_void_p), len(lists[k]))
    ms = []
    for r in range(runs):
        lst = lists[r & 1]
        w.timer_record(0)
        if d.kjb_rebuild_tlas(w.ctx, C.cast(lst, C.c_void_p), len(lst)):
            raise RuntimeError((d.kjb_last_error(w.ctx) or b"").decode())
        w.timer_record(1)
        ms.append(w.timer_elapsed_ms(0, 1))
    # frames: steady, then one that adds an instance, then one that removes it
    steady, add, remove = [], [], []
    for r in range(max(3, runs // 4)):
        for bucket, action in ((steady, None), (add, "add"), (remove, "remove")):
            if action == "add":
                hid = w.add_instance(ht, extra[0])
            elif action == "remove":
                w.remove_instance(hid)
            w.sync()
            t0 = time.perf_counter(); w.render_frame(**view); w.sync(); bucket.append((time.perf_counter() - t0) * 1e3)
    wt = world_triangles(scene)
    out = dict(scene=name, triangles=int(len(wt)), device_build_ms=float(np.median(ms)), device_build_ms_min=float(np.min(ms)),
               host_reference_ms=host_reference_ms(wt, host_runs), steady_frame_ms=float(np.median(steady)),
               add_frame_ms=float(np.median(add)), remove_frame_ms=float(np.median(remove)), tlas_stats=w.tlas_stats())
    w.close()
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--scenes", default="cornell,atrium,ruins")
    ap.add_argument("--runs", type=int, default=20)
    ap.add_argument("--host-runs", type=int, default=3)
    args = ap.parse_args()
    lib = kajiya_b200.lib()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    makers = dict(cornell=scenes.cornell_box, atrium=scenes.atrium, ruins=scenes.ruins)
    results = []
    for name in args.scenes.split(","):
        scene, view = makers[name]()
        results.append(measure(lib, name, scene, view, args.runs, args.host_runs))
    print(json.dumps(dict(gpu=gpu, results=results)))


if __name__ == "__main__":
    main()
