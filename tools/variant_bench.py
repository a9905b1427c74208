"""A/B timing of compile-time kernel variants on cuda:0 (tuning aid, not a bench line).

    python tools/variant_bench.py build  name=-DKJB_OCC_RESTIR_SPATIAL=4,-DKJB_OCC_RESTIR_RESOLVE=5 ...   # here (nvcc cross-compiles)
    python tools/variant_bench.py run [--frames 48] [--spatial 1]                                          # on the GPU box

`build` compiles kajiya_b200/csrc/_variants/libkjb_<name>.so from the same sources with extra -D flags; `run` renders the Cornell 1080p
workload with every variant found there plus the shipping library, interleaved (A B C A B C ...) so clock drift hits all alike, and prints
per-pass device times (kjb_world_set_profiling) for each."""
import os, subprocess, sys, glob, json
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
VAR = os.path.join(ROOT, "kajiya_b200", "csrc", "_variants")


def build(specs):
    import __graft_entry__ as g
    os.makedirs(VAR, exist_ok=True)
    for spec in specs:
        name, flags = spec.split("=", 1)
        flags = [f for f in flags.split(",") if f]
        objs = []
        procs = []
        for src in g.CU_SOURCES + g.CPP_SOURCES:
            obj = os.path.join(VAR, f"{name}_{os.path.basename(src)}.o"); objs.append(obj)
            cmd = [g.NVCC] + [f for f in g.NVCC_FLAGS if f not in ("-Xptxas", "-v")] + flags + ["-x", "cu" if src.endswith(".cu") else "c++", "-c", os.path.join(g.CSRC, src), "-o", obj]
            procs.append(subprocess.Popen(cmd))
        assert all(p.wait() == 0 for p in procs)
        subprocess.check_call([g.NVCC, "-shared", "-o", os.path.join(VAR, f"libkjb_{name}.so")] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-lcudart"])
        for o in objs: os.remove(o)
        print("built", name, flags)


def run(frames, spatial, rounds=3, workload=None):
    import numpy as np
    import kajiya_b200
    from kajiya_b200._abi import KjbLib
    from kajiya_b200.world import World
    from kajiya_b200 import scenes
    libs = [("shipping", os.path.join(ROOT, "kajiya_b200", "csrc", "libkjb.so"))] + [(os.path.basename(p)[7:-3], p) for p in sorted(glob.glob(os.path.join(VAR, "libkjb_*.so")))]
    import bench
    scene, view = scenes.cornell_box()
    worlds = []
    for name, path in libs:
        if workload:   # a bench.py workload (e.g. atrium_1080p_full): replayed G-buffers, like the bench
            w, view, _, _ = bench.build_world(KjbLib(path), workload)
            for i in range(4): w.render_frame(capture_slot=i + 1, **view)
            view = dict(view, replay_slot=1)
        else:
            w = World(KjbLib(path), 1920, 1080, spatial_reuse_pass_count=spatial); scenes.populate(w, scene)
        for _ in range(8): w.render_frame(**view)
        w.sync(); worlds.append((name, w))
    acc = {name: {} for name, _ in worlds}
    for r in range(rounds):
        for name, w in worlds:
            w.set_profiling(True)
            for _ in range(frames): w.render_frame(**view)
            for label, (calls, ms) in w.pass_timings().items():
                acc[name].setdefault(label, []).append(ms / calls)
            w.set_profiling(False)
    labels = sorted(acc["shipping"], key=lambda l: -np.median(acc["shipping"][l]))
    print(f"{'pass':26s}" + "".join(f"{n[:14]:>15s}" for n, _ in worlds))
    tot = {n: 0.0 for n, _ in worlds}
    for l in labels:
        row = f"{l:26s}"
        for n, _ in worlds:
            v = float(np.median(acc[n].get(l, [0.0]))); tot[n] += v; row += f"{v * 1000:15.1f}"
        print(row)
    print(f"{'sum (us/frame)':26s}" + "".join(f"{tot[n] * 1000:15.1f}" for n, _ in worlds))
    print(json.dumps({"variant_us_per_frame": {n: round(tot[n] * 1000, 2) for n, _ in worlds}}))


if __name__ == "__main__":
    if sys.argv[1] == "build":
        build(sys.argv[2:])
    else:
        import argparse
        ap = argparse.ArgumentParser(); ap.add_argument("cmd"); ap.add_argument("--frames", type=int, default=48); ap.add_argument("--spatial", type=int, default=1); ap.add_argument("--workload", default=None)
        a = ap.parse_args(); run(a.frames, a.spatial, workload=a.workload)
