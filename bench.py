#!/usr/bin/env python
"""bench.py — benchmark of the H100-native kajiya ReSTIR-GI hot path (rtdgi + irradiance cache + rtr + taa).

    python bench.py --gpus N --steps K --warmup W            # this implementation (CUDA, sm_90a)
    python bench.py --impl reference --gpus N --steps K ...  # the CPU restatement of the reference's path, all host threads

A "step" is one frame of the hot path over one synthetic batch of G-buffer inputs.  The headline workload is the WHOLE path on the
Sponza-class atrium at 1080p (BASELINE.json configs[2] — rtdgi with two spatial passes + irradiance cache + ray-traced reflections —
plus the TAA passes): ~40 kernels per frame.  The line also carries `configs`: one entry per BASELINE.json configuration
(configs[0] Cornell 256^2 reference path tracer, configs[1] Cornell 1080p rtdgi 1 spatial + 1 temporal, configs[2] the headline,
configs[3] atrium 1440p full path + TAA, configs[4] 2 M-triangle ruins rendered at 2560x1440 and temporally upsampled to 4K), each with
its own `roofline`, `e2e` and `cpu_baseline`.  Metric: GI rays/s (closest-hit + any-hit rays actually traced, counted on the device)
with ms/frame as `ms_per_step`.

`value`    : inputs (the frame's G-buffer/depth/normal/velocity) already resident in HBM (a ring of distinct jittered G-buffers larger
             than L2, captured untimed).
`e2e`      : the same frames through the public host-buffer call (kjb_world_render_frame with pinned HOST G-buffer inputs uploaded and
             the result image downloaded inside the timed region).
`roofline` : achieved HBM GB/s of the dominant kernel = algorithmic bytes of that pass (SURVEY.md §8a per-pixel figures x pixels) / its
             mean launch duration (CUDA events on the launch stream, a profiling pass over the same K frames); `traffic` = ncu DRAM
             bytes per launch of that kernel, read from the table named in `traffic_source` (profiles/, made by tools/ncu_table.py).
`cpu_baseline`: the oracle (CPU port of the reference shaders, every host thread, cache passes on the parallel schedule) on a bounded
             sample of the same workload — replayed G-buffers, i.e. exactly the passes the GPU arm times.
At N > 1 ONE frame is tile-sharded over the ranks (strong scaling); `parity` compares every rank's band with an untiled render of the
same frames on that rank.
`--dump-outputs DIR`: after the timed steps, the headline's result image of the last timed frame (what the host-buffer call hands its
caller) is written as DIR/<image name>.npy in float32, so that two builds can be compared output for output; the inputs of a run depend
only on its arguments.
"""
import argparse, ctypes as C, hashlib, json, os, subprocess, sys, threading, time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

FULL = dict(enable_ircache=True, enable_rtr=True, enable_taa=True)
WORKLOADS = {
    # name: (scene fn name, kwargs, render width, render height, spatial passes, world flags)
    "cornell_256_reference_pt": ("cornell_box", {}, 256, 256, 1, {}),                         # BASELINE configs[0]: the reference path tracer (paths/s)
    "cornell_1080p_rtdgi_1s1t": ("cornell_box", {}, 1920, 1080, 1, {}),                       # BASELINE configs[1]
    "cornell_256_rtdgi": ("cornell_box", {}, 256, 256, 1, {}),
    "atrium_1080p_rtdgi": ("atrium", {}, 1920, 1080, 2, {}),
    "atrium_1080p_gi_ircache_rtr": ("atrium", {}, 1920, 1080, 2, dict(enable_ircache=True, enable_rtr=True)),
    "atrium_1080p_full": ("atrium", {}, 1920, 1080, 2, dict(FULL)),                           # BASELINE configs[2] (Sponza-class) + TAA: the whole hot path — HEADLINE
    "atrium_1440p_full_taa": ("atrium", {}, 2560, 1440, 2, dict(FULL)),                       # BASELINE configs[3] (the driver's 2/4/8-GPU runs shard the headline; this is its 1-GPU number)
    # BASELINE configs[4]: 2 M-triangle ruins, `--temporal-upsampling 1.5` at 4K = rendered at 2560x1440 and upsampled to 3840x2160 by the TAA
    # pass (crates/lib/kajiya-simple/src/main_loop.rs:222-233), full GI + SSAO guide + lit composite
    "ruins_4k_upsampled_full": ("ruins", {}, 2560, 1440, 2, dict(FULL, enable_ssao=True, enable_lighting=True, upscale=(3840, 2160))),
}
BASELINE_CONFIG = {"cornell_256_reference_pt": 0, "cornell_1080p_rtdgi_1s1t": 1, "atrium_1080p_full": 2, "atrium_1440p_full_taa": 3, "ruins_4k_upsampled_full": 4}
HEADLINE = "atrium_1080p_full"
CONFIG_SET = ["cornell_256_reference_pt", "cornell_1080p_rtdgi_1s1t", "atrium_1080p_full", "atrium_1440p_full_taa", "ruins_4k_upsampled_full"]

# compulsory bytes per pixel of each pass at its own grid (SURVEY.md §8a; F = render-res px, Hh = half-res px, O = TAA output px)
PASS_BYTES = {
    "rtdgi reproject": ("F", 24), "extract ssao/2": ("Hh", 2), "extract half-res inputs": ("Hh", 30), "extract half depth": ("Hh", 8), "extract view normal/2": ("Hh", 20),
    "rtdgi validate": ("Hh", 5), "rtdgi trace": ("Hh", 38), "validity integrate": ("Hh", 21), "restir temporal": ("Hh", 160),
    "restir spatial": ("Hh", 41), "restir resolve": ("F+Hh", (29, 56)), "rtdgi temporal": ("F+Hh", (48, 4)), "rtdgi spatial": ("F", 25),
    # rtr (SURVEY §8a: 44 + 45 + 152 Hh; 36 F + 60 Hh; 52 F + 1 Hh; 20 F)
    "reflection trace": ("Hh", 44), "reflection validate": ("Hh", 45), "rtr restir temporal": ("Hh", 152), "reflection resolve": ("F+Hh", (36, 60)),
    "reflection temporal": ("F+Hh", (52, 1)), "reflection cleanup": ("F", 20),
    # taa (SURVEY §8a: 80 O + 120 I in total; split per pass from the images each kernel binds)
    "reproject taa": ("O+F", (20, 12)), "taa filter input": ("F", 28), "taa filter history": ("O+F", (8, 8)), "taa input prob": ("F", 46), "taa prob filter": ("F", 4),
    "taa prob filter2": ("F", 4), "taa": ("O+F", (52, 18)),
    # irradiance cache (SURVEY §8a: 6.3 MB of grid + 1548 B per live entry; the entry count lives on the device, so only the fixed part is
    # charged here) and the other small passes of the frame
    "clear ircache pool": ("const", 0), "scroll cascades": ("const", 6291456), "age ircache entries": ("const", 0), "_prefix scan": ("const", 524288), "ircache compact": ("const", 0), "_ircache dispatch args": ("const", 0),
    "ircache reset": ("const", 0), "ircache trace access": ("const", 0), "ircache validate": ("const", 0), "ircache trace": ("const", 0), "ircache sum": ("const", 0),
    "restir check": ("Hh", 28), "reprojection map": ("F", 28), "copy depth": ("F", 8),
    # lit composite (N4): bound texels of trace_sun_shadow_mask.rgen / the three shadow_denoise shaders / light_gbuffer.hlsl, once each
    "trace shadow mask": ("F", 9), "shadow bitpack": ("F", 1.125), "shadow temporal": ("F", 33.25), "shadow spatial": ("F", 16), "light gbuffer": ("F", 52), "sample lights": ("Hh", 32), "spatial reuse lights": ("F+Hh", (28, 36)),
    # SSAO guide (N3): ssgi.hlsl + spatial + upsample + temporal (ssgi.rs:41-243)
    "ssao": ("Hh", 30), "ssao spatial": ("Hh", 12), "ssao upsample": ("F+Hh", (10, 10)), "ssao temporal": ("F", 14),
    "tile border all-gather": ("const", 0), "tile gi all-gather": ("const", 0), "tile input all-gather": ("const", 0), "tile ircache all-gather": ("const", 0),
}
NCU_TABLE = os.path.join("profiles", "ncu_kernel_table.json")   # {workload: {pass label: {"dram_bytes": .., "warp_inst": .., "source": "profiles/<csv>"}}}, made by tools/ncu_table.py


def load_ncu_table():
    p = os.path.join(ROOT, NCU_TABLE)
    try:
        return json.load(open(p))
    except Exception:
        return {}


def pass_bytes(label, F, Hh, O=None, validation_frame_fraction=1.0 / 3.0):
    O = F if O is None else O
    kind, b = PASS_BYTES[label]
    if label == "rtdgi validate":
        return Hh * (5 + 61 * validation_frame_fraction)
    if kind == "const":
        return b
    if kind == "F":
        return F * b
    if kind == "Hh":
        return Hh * b
    if kind == "O+F":
        return O * b[0] + F * b[1]
    return F * b[0] + Hh * b[1]


class ClockSampler:
    """nvidia-smi clocks/throttle reasons sampled DURING the timed region."""

    def __init__(self, gpu_index):
        self.samples, self.proc, self.gpu = [], None, gpu_index

    def start(self):
        q = "clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap"
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--id={self.gpu}", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-lms", "100"],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.thread = threading.Thread(target=self._read, daemon=True); self.thread.start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.samples.append([x.strip() for x in line.split(",")] + [time.perf_counter()])

    def stop(self, windows=None):
        """median SM clock / reasons over the samples taken inside the [begin, end] perf_counter windows, i.e. while timed loops ran"""
        if not self.proc:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        time.sleep(0.15)
        self.proc.terminate()
        smp = self.samples
        if windows:
            smp = [s for s in smp if any(a <= s[-1] <= b + 0.1 for a, b in windows)]
        sm = sorted(int(float(s[0])) for s in smp if s and s[0].replace(".", "").isdigit())
        reasons = set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for s in smp:
            for i, n in enumerate(names):
                if len(s) > 3 + i and s[3 + i].lower().startswith("active"):
                    reasons.add(n)
        mx = None
        for s in self.samples:
            if len(s) > 1 and s[1].replace(".", "").isdigit():
                mx = int(float(s[1]))
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": mx, "reasons": sorted(reasons), "samples": len(sm)}


def load_peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        return json.load(open(p)).get("hbm_gbs", 6650.0), "measured (MEASURED_PEAKS.json)"
    return 3350.0, "fallback (H100 SXM data sheet: 3.35 TB/s HBM3)"


def build_world(lib, workload, device=0, tile=None):
    from kajiya_b200 import scenes
    from kajiya_b200.world import World
    fn, kw, W, H, spatial, flags = WORKLOADS[workload]
    scene, view = getattr(scenes, fn)(**kw)
    w = World(lib, W, H, device=device, spatial_reuse_pass_count=spatial, tile=tile, **flags)
    scenes.populate(w, scene)
    return w, view, W, H


def config_of(workload):
    """The workload description both arms print (identical keys and values for `--impl reference`, independent of N)."""
    fn, kw, W, H, spatial, flags = WORKLOADS[workload]
    out = flags.get("upscale") or (W, H)
    return {"workload": workload, "baseline_config": BASELINE_CONFIG.get(workload), "scene": fn, "resolution": [W, H], "output_resolution": list(out),
            "spatial_reuse_passes": spatial, "features": sorted(k for k, v in flags.items() if v and k != "upscale"),
            "inputs": "a ring of distinct jittered G-buffers larger than L2 (50 MB), replayed; e2e uploads them from pinned host memory"}


def pinned_empty(torch, nbytes):
    return torch.empty(nbytes, dtype=torch.uint8).pin_memory()


def result_image_name(workload):
    flags = WORKLOADS[workload][5]
    return "taa.this_frame_out" if flags.get("enable_taa") else ("debug_out" if flags.get("enable_lighting") else "rtdgi.spatial_filtered")


# ---------------------------------------------------------------------------------------------------------------- GPU arm
def measure_frames(lib, torch, dist, workload, K, Wm, rank, world_size, local_rank, nslots, streaming=True, dump=None):
    """device-resident, per-pass and end-to-end legs of one frame workload; returns a dict on every rank (reduced over ranks).
    `dump`: a dict that receives the result image of the last timed frame"""
    w, view, W, H = build_world(lib, workload, device=local_rank, tile=(rank, world_size) if world_size > 1 else None)
    if world_size > 1:
        uid = [None]
        if rank == 0:
            buf = C.create_string_buffer(128)
            assert lib.dll.kjb_comm_nccl_unique_id(buf) == 0, "ncclGetUniqueId failed"
            uid[0] = buf.raw
        dist.broadcast_object_list(uid, src=0)
        w.comm_init_nccl(uid[0], rank, world_size)
    flags = WORKLOADS[workload][5]
    OW, OH = flags.get("upscale") or (W, H)
    F, Hh, O = W * H, ((W + 1) // 2) * ((H + 1) // 2), OW * OH
    nslots = max(2, min(K, nslots))

    # ---- untimed: produce the G-buffer ring on the device (the raster stand-in is an input producer, not the hot path)
    for i in range(nslots):
        w.render_frame(capture_slot=i + 1, **view)
    w.sync()
    host_ring = []
    for i in range(nslots):
        bufs = []
        for name in ("gbuffer", "depth", "geometric_normal", "velocity"):
            img = w.image_handle(f"slot{i + 1}.{name}")
            t = pinned_empty(torch, img.width * img.height * lib.dll.kjb_format_texel_bytes(img.format))
            w._check(lib.dll.kjb_image_download(w.ctx, C.byref(img), t.data_ptr()))
            bufs.append(t)
        host_ring.append(bufs)
    w.sync()
    res_img = w.image_handle(result_image_name(workload))
    res_bytes = res_img.width * res_img.height * lib.dll.kjb_format_texel_bytes(res_img.format)
    host_results = [pinned_empty(torch, res_bytes), pinned_empty(torch, res_bytes)]   # streaming mode alternates between two result buffers

    def barrier():
        if dist is not None:
            dist.barrier()
        torch.cuda.synchronize()

    def step_device(i):
        w.render_frame(replay_slot=(i % nslots) + 1, **view)

    def step_e2e(i):
        b = host_ring[i % nslots]
        w.render_frame(host_inputs=(b[0].data_ptr(), b[1].data_ptr(), b[2].data_ptr(), b[3].data_ptr()), host_result=host_results[i & 1].data_ptr(), streaming=streaming, **view)

    # ---- device-resident leg
    for i in range(Wm):
        step_device(i)
    w.sync(); w.stats()          # reset ray counters
    launches0 = lib.dll.kjb_launch_count(w.ctx)
    barrier()
    t_begin = time.perf_counter()
    w.timer_record(1000)
    for i in range(K):
        step_device(Wm + i)
    w.timer_record(1001)
    ms_total = w.timer_elapsed_ms(1000, 1001)
    barrier()
    st = w.stats()
    if dump is not None:
        dump[result_image_name(workload)] = w.image(result_image_name(workload))
    rays = st["closest_rays"] + st["any_hit_rays"]
    closest_share = st["closest_rays"] / max(rays, 1)
    launches = lib.dll.kjb_launch_count(w.ctx) - launches0

    # ---- per-pass timing (CUDA events around every pass, same K frames)
    w.set_profiling(True)
    for i in range(K):
        step_device(Wm + K + i)
    timings = w.pass_timings()
    w.set_profiling(False)

    # ---- e2e leg: host G-buffer in, result out
    for i in range(max(4, Wm // 2)):
        step_e2e(i)
    w.wait(); w.stats()
    barrier()
    t0 = time.perf_counter()
    w.timer_record(1002)
    for i in range(K):
        step_e2e(i)
    w.wait()                     # the last results have landed in host memory
    w.timer_record(1003)
    ms_e2e = w.timer_elapsed_ms(1002, 1003)
    wall_e2e = (time.perf_counter() - t0) * 1e3
    barrier()
    windows = [(t_begin, time.perf_counter())]
    st2 = w.stats()
    rays_e2e = st2["closest_rays"] + st2["any_hit_rays"]
    ms_e2e = max(ms_e2e, wall_e2e)   # the call blocks on the download: wall clock is the honest end-to-end figure
    h2d = sum(int(t.numel()) for t in host_ring[0]) // world_size + 1216    # a rank of a tile-sharded frame uploads its band only (the bands travel over NVLink)
    res_bytes = res_bytes // world_size
    w.close()
    del host_ring, host_results

    # ---- reduce over ranks: max time, summed rays
    rays_traced = rays
    per_pass = {k: v[1] / max(v[0], 1) for k, v in timings.items() if k in PASS_BYTES}
    calls = {k: v[0] for k, v in timings.items() if k in PASS_BYTES}
    if dist is not None:
        t = torch.tensor([ms_total, ms_e2e], device="cuda", dtype=torch.float64); dist.all_reduce(t, op=dist.ReduceOp.MAX)
        r = torch.tensor([rays, rays_e2e, launches], device="cuda", dtype=torch.float64); dist.all_reduce(r, op=dist.ReduceOp.SUM)
        ms_total, ms_e2e = t.tolist(); rays_traced, _, launches = r.tolist()
        labels = sorted(per_pass)   # every rank runs the same pass list
        pm = torch.tensor([per_pass[k] for k in labels], device="cuda", dtype=torch.float64); dist.all_reduce(pm, op=dist.ReduceOp.MAX)
        per_pass = dict(zip(labels, pm.tolist()))   # slowest rank per pass
    return dict(workload=workload, W=W, H=H, F=F, Hh=Hh, O=O, K=K, ms_total=ms_total, ms_e2e=ms_e2e, rays=rays, rays_e2e=rays_e2e, rays_traced=rays_traced, launches=launches,
                per_pass=per_pass, calls=calls, h2d=h2d, d2h=res_bytes, closest_share=closest_share, nslots=nslots, windows=windows, view=view, streaming=streaming)


def frame_rays_untiled(lib, workload, K, Wm, local_rank, nslots):
    """rays one GPU traces for the same K frames: at N > 1 the metric counts the frame's rays once (the tiles also trace rays for their halos)"""
    w1, view, _, _ = build_world(lib, workload, device=local_rank, tile=None)
    n1 = max(2, min(K, nslots, 4))
    for i in range(n1):
        w1.render_frame(capture_slot=i + 1, **view)
    for i in range(Wm):
        w1.render_frame(replay_slot=(i % n1) + 1, **view)
    w1.sync(); w1.stats()
    for i in range(K):
        w1.render_frame(replay_slot=((Wm + i) % n1) + 1, **view)
    s1 = w1.stats(); w1.close()
    return s1["closest_rays"] + s1["any_hit_rays"]


def band_compare(a, b, H, rank, world_size, statistical):
    """compare this rank's band (rows of the result image) of an untiled render `a` and a tiled render `b` (numpy arrays, storage dtype)"""
    import numpy as np
    HH = (H + 1) // 2
    y0, y1 = 2 * (HH * rank // world_size), 2 * (HH * (rank + 1) // world_size)
    scale = max(1, a.shape[0] // H)
    ba, bb = a[y0 * scale:y1 * scale], b[y0 * scale:y1 * scale]
    exact = bool(np.array_equal(ba, bb))
    if ba.dtype == np.uint16:   # RGBA16F storage
        fa, fb = ba.view(np.float16).astype(np.float32)[..., :3], bb.view(np.float16).astype(np.float32)[..., :3]
    else:
        fa, fb = ba.astype(np.float32)[..., :3], bb.astype(np.float32)[..., :3]
    mean_a, mean_b = float(fa.mean()), float(fb.mean())
    rel_mean = abs(mean_b / max(mean_a, 1e-12) - 1.0)
    # Texel-wise RMS says little once the two renders have run for a while: both are realisations of the same racy process and their noise has decorrelated
    # (per-texel difference = sqrt(2) x the noise level, 20-30 % after 24 frames), and both grow a few isolated bright texels over time, at different places (the
    # oracle does too: 1080p atrium, taa max 1.9 after 12 frames, 5.1 after 24).  The structural comparison is made on 16x16 block means of values clipped at
    # 4x the band mean; the texel-wise figure is reported beside it.
    cap = 4.0 * max(mean_a, 1e-12)
    ca, cb = np.minimum(fa, cap), np.minimum(fb, cap)
    hb, wb = ca.shape[0] // 16 * 16, ca.shape[1] // 16 * 16
    if hb and wb:
        ba_, bb_ = (x[:hb, :wb].reshape(hb // 16, 16, wb // 16, 16, -1).mean(axis=(1, 3)) for x in (ca, cb))
        rel_rms = float(np.sqrt(((ba_ - bb_) ** 2).mean())) / max(mean_a, 1e-12)
    else:
        rel_rms = float(np.sqrt(((ca - cb) ** 2).mean())) / max(mean_a, 1e-12)
    ok = exact if not statistical else (rel_mean < 0.08 and rel_rms < 0.25)
    band_compare.last_detail = {"max_abs_diff": float(np.abs(fa - fb).max()), "max_untiled": float(fa.max()), "max_tiled": float(fb.max()),
                                "rel_rms_unclipped": float(np.sqrt(((fa - fb) ** 2).mean())) / max(mean_a, 1e-12), "nonfinite": int((~np.isfinite(fb)).sum() + (~np.isfinite(fa)).sum())}
    return ok, exact, rel_mean, rel_rms, hashlib.sha256(bb.tobytes()).hexdigest()[:16]


def parity_check(lib, torch, dist, workload, rank, world_size, local_rank, frames=6):
    """every rank renders `frames` frames tiled (its band, NCCL exchange) AND untiled on its own GPU and compares its band of the result.
    Without the irradiance cache the band must be bit-identical.  With it (racy by design; per-rank replicas that exchange their rays' requests every
    frame, so a request reaches the other replicas one frame late) the comparison is statistical and made after 24 frames, when the cold-start transient of
    that one-frame lag has decayed: band mean within 8 %, RMS difference of 16x16 block means below 25 % of the mean (tests/test_multigpu_gloo.py and DESIGN §7 give the
    emulator's numbers: without the exchange some bands stay 20 % off for good, with it every band is within 6 % after 20 frames)."""
    if WORKLOADS[workload][5].get("enable_ircache"):
        frames = 24
    wt, view, W, H = build_world(lib, workload, device=local_rank, tile=(rank, world_size))
    uid = [None]
    if rank == 0:
        buf = C.create_string_buffer(128); assert lib.dll.kjb_comm_nccl_unique_id(buf) == 0; uid[0] = buf.raw
    dist.broadcast_object_list(uid, src=0)
    wt.comm_init_nccl(uid[0], rank, world_size)
    wu, _, _, _ = build_world(lib, workload, device=local_rank, tile=None)
    statistical = bool(WORKLOADS[workload][5].get("enable_ircache"))
    # statistical mode: a SECOND untiled world rendered alongside gives the run-to-run spread of the single-GPU renderer itself (same racy kernels, same frames) —
    # the yardstick the tiled-vs-untiled difference is held against
    wu2 = build_world(lib, workload, device=local_rank, tile=None)[0] if statistical else None
    for _ in range(frames):
        wt.render_frame(**view); wu.render_frame(**view)
        if wu2 is not None:
            wu2.render_frame(**view)
    name = result_image_name(workload)
    floor_mean = floor_rms = 0.0
    if wu2 is not None:
        _, _, floor_mean, floor_rms, _ = band_compare(wu.image(name), wu2.image(name), H, rank, world_size, True)
        wu2.close()
    ok, exact, rel_mean, rel_rms, sha = band_compare(wu.image(name), wt.image(name), H, rank, world_size, statistical)
    if statistical:
        ok = rel_mean < 0.08 and rel_rms < max(0.25, 1.5 * floor_rms)
    wt.close(); wu.close()
    det = band_compare.last_detail
    v = torch.tensor([1.0 if ok else 0.0, 1.0 if exact else 0.0, rel_mean, rel_rms, det["rel_rms_unclipped"], det["max_untiled"], det["max_tiled"], float(det["nonfinite"]), floor_mean, floor_rms], device="cuda", dtype=torch.float64)
    lo = v.clone(); dist.all_reduce(lo, op=dist.ReduceOp.MIN)
    hi = v.clone(); dist.all_reduce(hi, op=dist.ReduceOp.MAX)
    return {"ok": bool(lo[0].item() > 0.5), "mode": "statistical (irradiance cache: per-rank replicas exchanging their requests, racy by design; band mean within 8 %, RMS of 16x16 block means below max(25 %, 1.5 x the spread of two single-GPU renders))" if statistical else "bit-exact (every rank's band of the tiled frame == the untiled frame)",
            "bands_bit_identical": bool(lo[1].item() > 0.5), "worst_band_mean_rel_diff": hi[2].item(), "worst_band_rel_rms": hi[3].item(), "worst_band_rel_rms_unclipped": hi[4].item(),
            "max_texel_untiled": hi[5].item(), "max_texel_tiled": hi[6].item(), "nonfinite_texels": int(hi[7].item()),
            "untiled_vs_untiled": {"worst_band_mean_rel_diff": hi[8].item(), "worst_band_rel_rms": hi[9].item(), "note": "two single-GPU renders of the same frames on this rank: the renderer's own run-to-run spread"} if statistical else None,
            "frames": frames,
            "band_sha256_rank0": sha, "image": name}


def summarize(m, world_size, peak, ncu_table):
    """bench-line fields of one measured frame workload"""
    F, Hh, O, K = m["F"], m["Hh"], m["O"], m["K"]
    per_pass, calls = m["per_pass"], m["calls"]
    share = {k: per_pass[k] * calls.get(k, K) for k in per_pass}
    kernels = [k for k in share if not k.startswith("tile ")]   # the exchange entries are waits on the communication queue, not one of our kernels
    dom = max(kernels, key=share.get)
    dom_bytes = pass_bytes(dom, F, Hh, O)
    # at N > 1 the frame's algorithmic bytes are counted ONCE (halo recompute is not credited) against N x the per-GPU peak
    achieved = dom_bytes / (per_pass[dom] * 1e-3) / 1e9
    frame_bytes = sum(pass_bytes(k, F, Hh, O) * (calls.get(k, K) / K) for k in per_pass)
    frame_ms = m["ms_total"] / K
    tab = (ncu_table.get(m["workload"]) or {}).get(dom) if world_size == 1 else None
    roof = {"bound": "hbm", "kernel": dom, "achieved": achieved, "peak": peak * world_size, "unit": "GB/s", "frac": achieved / (peak * world_size),
            "traffic": tab.get("dram_bytes") if tab else None, "traffic_source": (tab.get("source") if tab else None),
            "kernel_ms": per_pass[dom], "kernel_share_of_step": share[dom] / sum(share.values()), "algorithmic_bytes_per_launch": dom_bytes,
            "frame": {"algorithmic_bytes": frame_bytes, "achieved_gbs": frame_bytes / (frame_ms * 1e-3) / 1e9, "frac": frame_bytes / (frame_ms * 1e-3) / 1e9 / (peak * world_size)},
            "per_pass_ms": {k: round(v, 5) for k, v in sorted(per_pass.items(), key=lambda kv: -share[kv[0]])}}
    if tab and tab.get("warp_inst"):
        # these kernels are bound by instruction issue, not DRAM: also report the dominant kernel against 132 SMs x 4 schedulers x SM clock
        sm_mhz = 1980.0
        ach = tab["warp_inst"] / (per_pass[dom] * 1e-3) / 1e9
        roof["issue_slots"] = {"warp_inst_per_launch": tab["warp_inst"], "achieved_ginst_s": ach, "peak_ginst_s": 132 * 4 * sm_mhz * 1e-3, "frac": ach / (132 * 4 * sm_mhz * 1e-3), "source": tab.get("source")}
    return {"ms_per_step": frame_ms, "value": m["rays"] / (m["ms_total"] * 1e-3), "unit": "rays/s", "rays_per_frame": m["rays"] / K,
            "ray_kinds": {"closest_hit_per_frame": m["rays"] / K * m.get("closest_share", 0.0), "any_hit_per_frame": m["rays"] / K * (1.0 - m.get("closest_share", 0.0)),
                          "note": "closest-hit rays carry shading (material fetch, sun shadow ray, cache lookup); any-hit rays are visibility only"},
            "e2e": {"value": m["rays_e2e"] / (m["ms_e2e"] * 1e-3), "unit": "rays/s", "ms_per_step": m["ms_e2e"] / K, "h2d_bytes_per_step": int(m["h2d"]), "d2h_bytes_per_step": int(m["d2h"]),
                    "mode": "streaming: upload/compute/download queues, 2 frames in flight" if m["streaming"] else "blocking call per frame"},
            "gpu_launches": int(m["launches"]), "roofline": roof,
            "submission": ("frames submitted back to back; " + ("tile-sharded: direct launches, exchange on the comm queue" if world_size > 1 else
                           "CUDA graph recordings per frame" + ("; irradiance-cache chain of frame N+1 on the async pass queue under the reflection filters + TAA of frame N "
                           "(kjb_world_set_async_compute; per_pass_ms is measured with it off, one queue, direct launches)" if "enable_ircache" in WORKLOADS[m["workload"]][5] and not os.environ.get("KJB_NO_ASYNC") else "")))}


def measure_fast_math(torch, workload, K, Wm, local_rank, nslots=8):
    """the same frames through libkjb_fast.so (-DKJB_FAST -use_fast_math: MUFU transcendentals, approximate division / sqrt, FMA contraction) — NOT parity-valid
    (tests/test_gpu_fast.py states how close it stays), reported next to the exact build so that the cost of the numeric contract is a measured number"""
    import kajiya_b200
    try:
        lib = kajiya_b200.lib_fast()
    except Exception as e:
        return {"unavailable": str(e)[:120]}
    w, view, W, H = build_world(lib, workload, device=local_rank)
    n = max(2, min(K, nslots))
    for i in range(n):
        w.render_frame(capture_slot=i + 1, **view)
    for i in range(Wm):
        w.render_frame(replay_slot=(i % n) + 1, **view)
    w.sync(); w.stats()
    torch.cuda.synchronize()
    w.timer_record(1000)
    for i in range(K):
        w.render_frame(replay_slot=((Wm + i) % n) + 1, **view)
    w.timer_record(1001)
    ms = w.timer_elapsed_ms(1000, 1001)
    st = w.stats(); w.close()
    return {"ms_per_step": ms / K, "value": (st["closest_rays"] + st["any_hit_rays"]) / (ms * 1e-3), "unit": "rays/s", "steps": K,
            "build": "libkjb_fast.so: same sources, -DKJB_FAST -use_fast_math", "parity": "not bit-compatible with the oracle; tolerances in tests/test_gpu_fast.py"}


def measure_reference_pt(lib, torch, workload, K, Wm, local_rank):
    """BASELINE configs[0]: the reference path tracer (rt/reference_path_trace.rgen.hlsl), 1 path per pixel per frame, on the GPU"""
    w, view, W, H = build_world(lib, workload, device=local_rank)
    for _ in range(Wm):
        w.render_reference(**view)
    w.sync(); w.stats()
    l0 = lib.dll.kjb_launch_count(w.ctx)
    torch.cuda.synchronize()
    w.timer_record(1000)
    for _ in range(K):
        w.render_reference(**view)
    w.timer_record(1001)
    ms = w.timer_elapsed_ms(1000, 1001)
    st = w.stats()
    launches = lib.dll.kjb_launch_count(w.ctx) - l0
    res = pinned_empty(torch, W * H * 16)   # e2e: each frame downloads the accumulated image
    t0 = time.perf_counter()
    for _ in range(K):
        w.render_reference(host_result=res.data_ptr(), **view)
    w.sync()
    ms_e2e = (time.perf_counter() - t0) * 1e3
    st2 = w.stats(); w.close()
    rays = st["closest_rays"] + st["any_hit_rays"]
    return {"ms_per_step": ms / K, "value": rays / (ms * 1e-3), "unit": "rays/s", "paths_per_sec": W * H * K / (ms * 1e-3), "rays_per_frame": rays / K,
            "e2e": {"value": (st2["closest_rays"] + st2["any_hit_rays"]) / (ms_e2e * 1e-3), "unit": "rays/s", "ms_per_step": ms_e2e / K, "h2d_bytes_per_step": 1216, "d2h_bytes_per_step": W * H * 16, "mode": "blocking call per frame"},
            "gpu_launches": int(launches),
            "roofline": {"bound": "hbm", "kernel": "reference pt", "achieved": None, "peak": None, "unit": "GB/s", "frac": None, "traffic": None,
                         "note": "BVH traversal of a 32-triangle scene: L1-resident, no HBM roofline applies (SURVEY.md §8d: ray traversal is reported as rays/s)"}}


def run_cuda(args):
    import torch
    import kajiya_b200
    rank = int(os.environ.get("RANK", "0")); world_size = int(os.environ.get("WORLD_SIZE", "1")); local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    dist = None
    if world_size > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
    torch.cuda.set_device(local_rank)
    lib = kajiya_b200.lib()   # raises without the CUDA extension: no fallback
    if args.dump_outputs and world_size > 1:   # a rank of a tile-sharded frame holds only its band of the result
        raise SystemExit("--dump-outputs: the result image is written by single-GPU runs only")
    K, Wm = args.steps, args.warmup
    peak, peak_src = load_peaks()
    ncu_table = load_ncu_table()
    headline = args.workload
    if args.configs == "all":
        names = [headline] + [c for c in CONFIG_SET if c != headline]
    elif args.configs == "auto":   # N = 1: every BASELINE configuration; N > 1: the frame configurations that shard (not configs[0], the 256x256 path tracer, nor the lit composite of configs[4])
        names = [headline] + [c for c in CONFIG_SET if c != headline and (world_size == 1 or not (c == "cornell_256_reference_pt" or WORKLOADS[c][5].get("enable_lighting")))]   # the lit composite does not shard
    else:
        names = [headline]
    clocks = ClockSampler(local_rank); clocks.start()
    windows, entries, head, dump = [], [], None, {}
    for name in names:
        Kc = K if name == headline else min(K, 16)   # secondary configurations: a shorter timed region keeps the default run within minutes
        Wc = Wm if name == headline else max(3, min(Wm, 4))
        if name == "cornell_256_reference_pt":
            if rank == 0:
                e = measure_reference_pt(lib, torch, name, Kc, Wc, local_rank)
                e.update(config=config_of(name), steps=Kc, warmup=Wc)
                e["metric_note"] = "paths/s = pixels x frames / time (1 path per pixel per frame, up to 16 bounces)"
                if not args.no_cpu_baseline:
                    e["cpu_baseline"] = cpu_baseline_pt(name, seconds=min(args.cpu_seconds, 4.0))
                entries.append(e)
            if dist is not None:
                dist.barrier()
            continue
        m = measure_frames(lib, torch, dist, name, Kc, Wc, rank, world_size, local_rank, nslots=16 if name == headline else 6, streaming=not args.no_streaming,
                           dump=dump if args.dump_outputs and name == headline else None)
        windows += m["windows"]
        par = None
        if world_size > 1:
            m["rays_traced_all_ranks"] = m["rays_traced"]
            if rank == 0:
                m["rays"] = m["rays_e2e"] = frame_rays_untiled(lib, name, Kc, Wc, local_rank, 4)
            par = parity_check(lib, torch, dist, name, rank, world_size, local_rank)
        if rank == 0:
            e = summarize(m, world_size, peak, ncu_table)
            e.update(config=config_of(name), steps=Kc, warmup=Wc)
            e["roofline"]["peak_source"] = peak_src + (f" x {world_size} GPUs; the frame's algorithmic bytes counted once, slowest rank's kernel time" if world_size > 1 else "")
            if world_size > 1:
                e["multi_gpu"] = (f"one frame tile-sharded into {world_size} bands of half-res rows, NCCL all-gather of band borders per frame; `value` counts the frame's rays once "
                                  f"(the ranks actually traced {m['rays_traced_all_ranks'] / Kc:.0f} per frame including halo recompute)")
                e["parity"] = par
            if world_size == 1 and name in (headline, "cornell_1080p_rtdgi_1s1t") and not args.no_fast_math:
                e["fast_math"] = measure_fast_math(torch, name, min(Kc, 16), Wc, local_rank)
                if "ms_per_step" in e["fast_math"]:
                    e["fast_math"]["exact_over_fast"] = e["ms_per_step"] / e["fast_math"]["ms_per_step"]
            if world_size == 1 and not args.no_cpu_baseline:
                e["cpu_baseline"] = cpu_baseline(name, seconds=args.cpu_seconds if name == headline else min(args.cpu_seconds, 4.0), reduced=name != headline)
            entries.append(e)
            if name == headline:
                head = e
    clock_info = clocks.stop(windows)
    if rank == 0 and args.dump_outputs:
        dump_outputs(args.dump_outputs, dump)
    if rank != 0:
        if dist is not None:
            dist.destroy_process_group()
        return
    out = {"metric": "gi_rays_per_sec", "value": head["value"], "unit": "rays/s", "n_gpus": world_size, "steps": K, "warmup": Wm, "ms_per_step": head["ms_per_step"],
           "higher_is_better": True, "scaling": "strong", "vs_baseline": None, "dtype": "f32", "data": "synthetic", "config": head["config"],
           "e2e": head["e2e"], "gpu_launches": head["gpu_launches"], "clocks": clock_info, "roofline": head["roofline"]}
    for k in ("cpu_baseline", "parity", "multi_gpu", "fast_math"):
        if k in head:
            out[k] = head[k]
    out["configs"] = entries
    print(json.dumps(out))
    if dist is not None:
        dist.destroy_process_group()


DUMP_BYTES = 64 << 20


def dump_outputs(dirname, arrays):
    """DIR/<name>.npy in float32, at most DUMP_BYTES in all: an array over its share is replaced by a fixed, seeded sample of its rows"""
    import numpy as np
    os.makedirs(dirname, exist_ok=True)
    share = (DUMP_BYTES - 4096 * len(arrays)) // max(len(arrays), 1)   # 4 KiB per file for the .npy header
    for name, a in arrays.items():
        a = np.asarray(a, dtype=np.float32)
        if a.nbytes > share:
            rows = np.random.default_rng(0).choice(a.shape[0], share // (a.nbytes // a.shape[0]), replace=False)
            a = a[np.sort(rows)]
        np.save(os.path.join(dirname, name + ".npy"), a)


# ---------------------------------------------------------------------------------------------------------------- CPU arms
def oracle_lib():
    from kajiya_b200._abi import KjbLib
    return KjbLib(os.path.join(ROOT, "oracle", "_build", "libkj_oracle.so"))


def cpu_frames(workload, steps=None, seconds=None, warmup=1, reduced=False):
    """The oracle (CPU port of the reference shaders) on the host cores: the same scene and pass list over replayed G-buffers (the raster
    stand-in is outside the timed region on both arms), cache passes on the parallel schedule so every host thread is used.
    `reduced`: secondary configurations run at 1/4 of the width and height (scene-complexity-matched sample, SURVEY.md §8d)."""
    from kajiya_b200 import scenes
    from kajiya_b200.world import World
    lib = oracle_lib()
    fn, kw, W, H, spatial, flags = WORKLOADS[workload]
    fl = dict(flags)
    if reduced:
        W, H = max(64, W // 4) & ~1, max(64, H // 4) & ~1
        if fl.get("upscale"):
            fl["upscale"] = ((fl["upscale"][0] // 4) & ~1, (fl["upscale"][1] // 4) & ~1)
    scene, view = getattr(scenes, fn)(**kw)
    w = World(lib, W, H, spatial_reuse_pass_count=spatial, **fl)
    scenes.populate(w, scene)
    w.set_debug_serial(False)   # oracle: cache-touching passes on all threads (racy, like the reference's GPU dispatch)
    nslots = 2
    for i in range(nslots):
        w.render_frame(capture_slot=i + 1, **view)
    for i in range(warmup):
        w.render_frame(replay_slot=(i % nslots) + 1, **view)
    w.stats()
    per_frame, n, t0 = [], 0, time.perf_counter()
    while True:
        t1 = time.perf_counter()
        w.render_frame(replay_slot=((warmup + n) % nslots) + 1, **view); n += 1
        per_frame.append(time.perf_counter() - t1)
        el = time.perf_counter() - t0
        if (steps is not None and n >= steps) or (steps is None and ((el > seconds and n >= 3) or n >= 64)):
            break
    st = w.stats(); w.close()
    rays = st["closest_rays"] + st["any_hit_rays"]
    pf = sorted(per_frame)
    return {"value": rays / el, "unit": "rays/s", "cores": os.cpu_count(), "kind": "port", "ms_per_step": el / n * 1e3,
            "spread_ms": {"min": pf[0] * 1e3, "median": pf[len(pf) // 2] * 1e3, "max": pf[-1] * 1e3, "frames": n},
            "sample": f"{n} replayed frames of {workload} at {W}x{H}" + (" (1/4 of the configuration's width and height)" if reduced else "") +
                      f" after {warmup} warm-up, {os.cpu_count()} host threads, G-buffers captured beforehand (the same passes the GPU arm times)"}


def cpu_baseline(workload, seconds=12.0, reduced=False):
    return cpu_frames(workload, seconds=seconds, reduced=reduced)


def cpu_baseline_pt(workload, seconds=4.0):
    from kajiya_b200 import scenes
    from kajiya_b200.world import World
    lib = oracle_lib()
    fn, kw, W, H, spatial, flags = WORKLOADS[workload]
    scene, view = getattr(scenes, fn)(**kw)
    w = World(lib, W, H, spatial_reuse_pass_count=spatial, **flags)
    scenes.populate(w, scene)
    w.render_reference(**view); w.stats()
    n, t0 = 0, time.perf_counter()
    while True:
        w.render_reference(**view); n += 1
        el = time.perf_counter() - t0
        if el > seconds or n >= 256:
            break
    st = w.stats(); w.close()
    rays = st["closest_rays"] + st["any_hit_rays"]
    return {"value": rays / el, "unit": "rays/s", "paths_per_sec": W * H * n / el, "cores": os.cpu_count(), "kind": "port", "ms_per_step": el / n * 1e3,
            "sample": f"{n} frames of the reference path tracer at {W}x{H} (1 path per pixel per frame), {os.cpu_count()} host threads"}


def run_reference(args):
    """--impl reference: the reference's own implementation of the path cannot run here (Rust + Vulkan RT, SURVEY.md §8c);
    its CPU restatement (oracle port) is timed on the host cores on the same config/metric/unit: W warm-up and EXACTLY K timed steps,
    each step one replayed frame of the headline workload."""
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    world_size = int(os.environ.get("WORLD_SIZE", "1"))
    K, Wm = args.steps, args.warmup
    cb = cpu_frames(args.workload, steps=K, warmup=Wm)
    out = {"impl": "reference", "metric": "gi_rays_per_sec", "value": cb["value"], "unit": "rays/s", "n_gpus": world_size, "steps": K, "warmup": Wm,
           "ms_per_step": cb["ms_per_step"], "higher_is_better": True, "scaling": "strong", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
           "config": config_of(args.workload),
           "cpu_baseline": cb, "e2e": {"value": cb["value"], "unit": "rays/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}, "gpu_launches": 0}
    print(json.dumps(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=32, help="timed frames of the headline; the secondary configurations and the fast-math leg time min(steps, 16)")
    ap.add_argument("--warmup", type=int, default=6)
    ap.add_argument("--impl", default="kajiya_b200", choices=["kajiya_b200", "reference"])
    ap.add_argument("--workload", default=HEADLINE, choices=sorted(WORKLOADS), help="the headline workload of the line")
    ap.add_argument("--configs", default="auto", choices=["auto", "all", "headline"], help="which BASELINE configurations ride along in `configs`")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-fast-math", action="store_true", help="skip the libkjb_fast.so leg (the price of the exact numeric contract)")
    ap.add_argument("--no-streaming", action="store_true", help="e2e leg with the blocking call (upload, passes, download serialised)")
    ap.add_argument("--cpu-seconds", type=float, default=12.0)
    ap.add_argument("--dump-outputs", metavar="DIR", help="write the headline's result image of the last timed frame to DIR/<name>.npy (float32); one GPU only")
    args = ap.parse_args()
    args.warmup = max(args.warmup, 3)
    if args.impl == "reference":
        run_reference(args)
    else:
        run_cuda(args)


if __name__ == "__main__":
    main()
