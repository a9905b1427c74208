"""GPU parity tests proper: the CUDA library (through the C-ABI) against the CPU oracle on the same seeded inputs.
Bar: bit-exact for every image, integer AND float (the numeric contract pins the transcendentals; no FMA contraction)."""
import numpy as np, pytest
import parity
from parity import glossy
from kajiya_b200 import scenes

pytestmark = pytest.mark.gpu


def _assert_clean(report):
    bad = [(f, b) for f, frame in enumerate(report) for b in frame]
    assert not bad, f"images differ from the oracle (frame, (image, texels, max abs err)): {bad[:10]}"


def test_backend_is_cuda(cuda_lib):
    assert cuda_lib.backend == "cuda-sm90a"


def test_cornell_rtdgi_lockstep(oracle_lib, cuda_lib):
    scene, view = scenes.cornell_box()
    wa, wb, report = parity.run_lockstep(oracle_lib, cuda_lib, scene, view, 192, 108, 8)
    _assert_clean(report)
    s = wb.stats()
    assert s["launches"] > 0 and s["closest_rays"] > 0


def test_cornell_odd_extent(oracle_lib, cuda_lib):
    scene, view = scenes.cornell_box()
    _, _, report = parity.run_lockstep(oracle_lib, cuda_lib, scene, view, 101, 67, 7)
    _assert_clean(report)


def test_atrium_rtdgi_lockstep(oracle_lib, cuda_lib):
    scene, view = scenes.atrium(target_tris=30000)
    _, _, report = parity.run_lockstep(oracle_lib, cuda_lib, scene, view, 160, 90, 5)
    _assert_clean(report)


def test_single_spatial_pass_config(oracle_lib, cuda_lib):
    # BASELINE config 2: "ReSTIR GI 1 spatial + 1 temporal pass"
    scene, view = scenes.cornell_box()
    _, _, report = parity.run_lockstep(oracle_lib, cuda_lib, scene, view, 128, 72, 5, spatial_reuse_pass_count=1)
    _assert_clean(report)


def test_reference_path_tracer(oracle_lib, cuda_lib):
    scene, view = scenes.cornell_box()
    wa, wb = parity.make_world(oracle_lib, scene, 64, 64), parity.make_world(cuda_lib, scene, 64, 64)
    for _ in range(3):
        wa.render_reference(**view); wb.render_reference(**view)
    a, b = wa.image("refpt.accum"), wb.image("refpt.accum")
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))


def test_full_size_properties(cuda_lib):
    """At BASELINE's 1080p size the oracle is too slow for lockstep; check size-independent properties instead:
    determinism (two contexts, identical bits), sky pixels produce exactly zero irradiance, no NaN/Inf, payloads in range."""
    scene, view = scenes.cornell_box()
    w1, w2 = parity.make_world(cuda_lib, scene, 1920, 1080), parity.make_world(cuda_lib, scene, 1920, 1080)
    for _ in range(4):
        w1.render_frame(**view); w2.render_frame(**view)
    assert not parity.compare_images(w1, w2)
    irr = w1.image("rtdgi.spatial_filtered").astype(np.float32)
    depth = w1.image("depth")[..., 0]
    assert np.isfinite(irr).all()
    assert (irr[..., :3][depth == 0] == 0).all()
    res = w1.image("rtdgi.reservoir_output0")
    px, py = res[..., 0] & 0xffff, res[..., 0] >> 16
    assert (px < 960).all() and (py < 540).all()


def test_taa_native_and_upscaled(oracle_lib, cuda_lib):
    scene, view = scenes.cornell_box()
    for kw in (dict(enable_taa=True), dict(enable_taa=True, upscale=(240, 135))):
        _, wb, report = parity.run_lockstep(oracle_lib, cuda_lib, scene, view, 160, 90, 6, **kw)
        _assert_clean(report)
        assert "taa.this_frame_out" in wb.image_names()


def _moving_views(view, frames):
    cp = np.array(view["camera_position"], np.float32)
    for f in range(frames):
        v = dict(view); v["camera_position"] = tuple(cp + np.array([0.07 * f, 0.013 * f, -0.09 * f], np.float32))
        if f >= 8:
            v["camera_rotation"] = (0.0, float(np.sin(0.6)), 0.0, float(np.cos(0.6)))
        yield v


def test_ircache_serial_schedule_bit_exact(oracle_lib, cuda_lib):
    """The irradiance cache is racy by design upstream (ircache.rs:68-76); the default parallel schedule decides differently from the
    oracle's (kjb_ircache.cuh).  With kjb_set_debug_serial the CUDA kernels that touch the cache run on one device thread in launch order — the schedule the
    oracle restates — and then EVERYTHING (images + grid/pool/reservoir/SH buffers) must be bit-identical, including cascade
    scrolling, deallocation, aging and recycling under a moving camera."""
    scene, view = scenes.cornell_box()
    kw = dict(enable_ircache=True, spatial_reuse_pass_count=1)
    wa, wb = parity.make_world(oracle_lib, scene, 80, 48, **kw), parity.make_world(cuda_lib, scene, 80, 48, **kw)
    wb.set_debug_serial(True)
    for f, v in enumerate(_moving_views(view, 16)):
        wa.render_frame(**v); wb.render_frame(**v)
        bad = parity.compare_images(wa, wb)
        assert not bad, (f, bad[:5])
    meta = wb.image("ircache.meta_buf").ravel()
    assert meta[3] > 100 and meta[2] > meta[3]


def _cache_summary(w):
    meta = w.image("ircache.meta_buf").ravel()
    life = w.image("ircache.life_buf").ravel()
    irr = w.image("ircache.irradiance_buf").reshape(-1, 3, 4)
    valid = life < 12
    return dict(alloc=int(meta[3]), entries=int(meta[2]), valid=valid, r0=irr[valid][:, :, 0])


def test_ircache_parallel_statistical(oracle_lib, cuda_lib):
    """Normal (parallel) execution against the oracle's serial schedule: entry assignment, keep-alive and reposition votes are decided
    differently (kjb_ircache.cuh), so parity is statistical.  Tolerances: live entry count 3 %, occupied-cell sets Jaccard >= 0.9 (either buffer
    parity), mean L0 irradiance over the live entries 12 % (a few hundred entries after 12 frames: observed spread between GPU runs ~6 %), mean of the final GI image 6 % (observed up to 3 % between racy runs), and the final image within 0.05 RMS of the oracle's."""
    scene, view = scenes.cornell_box()
    kw = dict(enable_ircache=True)
    wa, wb = parity.make_world(oracle_lib, scene, 192, 108, **kw), parity.make_world(cuda_lib, scene, 192, 108, **kw)
    for f in range(12):
        wa.render_frame(**view); wb.render_frame(**view)
    a, b = _cache_summary(wa), _cache_summary(wb)
    assert abs(a["alloc"] - b["alloc"]) <= 0.03 * a["alloc"] + 2, (a["alloc"], b["alloc"])
    # occupied cells: the ping-pong parity is the same on both sides, compare the current grid
    def occupied(w):
        best = None
        for n in ("ircache.grid_meta_buf", "ircache.grid_meta_buf2"):
            g = w.image(n).reshape(-1, 2)
            occ = set(np.nonzero(g[:, 1] & 1)[0].tolist())
            if best is None or len(occ) > len(best): best = occ
        return best
    oa, ob = occupied(wa), occupied(wb)
    jac = len(oa & ob) / max(1, len(oa | ob))
    assert jac >= 0.9, jac
    ma, mb = float(a["r0"].mean()), float(b["r0"].mean())
    assert abs(ma - mb) <= 0.12 * abs(ma), (ma, mb)
    ia, ib = wa.image("rtdgi.spatial_filtered").astype(np.float64)[..., :3], wb.image("rtdgi.spatial_filtered").astype(np.float64)[..., :3]
    assert np.isfinite(ib).all()
    assert abs(ia.mean() - ib.mean()) <= 0.06 * ia.mean(), (ia.mean(), ib.mean())
    assert np.sqrt(((ia - ib) ** 2).mean()) <= 0.05 * max(ia.mean(), 1e-6) + 0.05, np.sqrt(((ia - ib) ** 2).mean())


def test_rtr_lockstep(oracle_lib, cuda_lib):
    """Reflections R1-R6 on glossy Cornell, camera in motion: every image bit for bit."""
    scene, view = scenes.cornell_box()
    scene = glossy(scene)
    kw = dict(enable_rtr=True)
    wa, wb = parity.make_world(oracle_lib, scene, 160, 90, **kw), parity.make_world(cuda_lib, scene, 160, 90, **kw)
    cp = np.array(view["camera_position"], np.float32)
    for f in range(7):
        v = dict(view); v["camera_position"] = tuple(cp + np.array([0.03 * f, 0.01 * f, -0.04 * f], np.float32))
        wa.render_frame(**v); wb.render_frame(**v)
        bad = parity.compare_images(wa, wb)
        assert not bad, (f, bad[:5])
    assert (wb.image("rtr.rng:0") != 0).mean() > 0.2


def test_full_pipeline_serial_schedule_bit_exact(oracle_lib, cuda_lib):
    """rtdgi + ircache + rtr + taa with the cache passes on the serial schedule: everything bit for bit on the real GPU."""
    scene, view = scenes.cornell_box()
    kw = dict(enable_rtr=True, enable_ircache=True, enable_taa=True)
    wa, wb = parity.make_world(oracle_lib, glossy(scene), 80, 48, **kw), parity.make_world(cuda_lib, glossy(scene), 80, 48, **kw)
    wb.set_debug_serial(True)
    for f in range(6):
        wa.render_frame(**view); wb.render_frame(**view)
        bad = parity.compare_images(wa, wb)
        assert not bad, (f, bad[:5])


def test_streaming_frames_match_blocking_frames(cuda_lib):
    """Streaming mode (upload / compute / download queues, two frames in flight) delivers the same bits as the blocking call,
    also when frames are submitted back to back without waiting (1080p so that copies and passes really overlap)."""
    scene, view = scenes.cornell_box()
    W, H, N = 1920, 1080, 6
    wa = parity.make_world(cuda_lib, scene, W, H, spatial_reuse_pass_count=1)
    host = []
    for i in range(N):
        wa.render_frame(**view)
        host.append([wa.image(n).copy() for n in ("gbuffer", "depth", "geometric_normal", "velocity")])
    wa.close()
    wb, wc = parity.make_world(cuda_lib, scene, W, H, spatial_reuse_pass_count=1), parity.make_world(cuda_lib, scene, W, H, spatial_reuse_pass_count=1)
    res_b = [np.zeros((H, W, 4), np.float16) for _ in range(N)]; res_s = [np.zeros((H, W, 4), np.float16) for _ in range(N)]
    for i in range(N):
        wb.render_frame(host_inputs=tuple(a.ctypes.data for a in host[i]), host_result=res_b[i].ctypes.data, **view)
    for i in range(N):
        wc.render_frame(host_inputs=tuple(a.ctypes.data for a in host[i]), host_result=res_s[i].ctypes.data, streaming=True, **view)
    wc.wait()
    for i in range(N):
        assert np.array_equal(res_b[i].view(np.uint16), res_s[i].view(np.uint16)), i


def test_atrium_full_pipeline_serial_schedule(oracle_lib, cuda_lib):
    """Sponza-class procedural scene (many materials, 1x1 placeholder textures, NaN validation rays from empty reservoirs):
    rtdgi + ircache + rtr, cache passes on the serial schedule, everything bit for bit."""
    scene, view = scenes.atrium(target_tris=12000)
    kw = dict(enable_rtr=True, enable_ircache=True, spatial_reuse_pass_count=2)
    wa, wb = parity.make_world(oracle_lib, scene, 96, 54, **kw), parity.make_world(cuda_lib, scene, 96, 54, **kw)
    wb.set_debug_serial(True)
    for f in range(5):
        wa.render_frame(**view); wb.render_frame(**view)
        bad = parity.compare_images(wa, wb)
        assert not bad, (f, bad[:5])


def test_ssao_guide(oracle_lib, cuda_lib):
    """SsgiRenderer (ssao, spatial, upsample, temporal) feeding rtdgi + rtr, camera in motion: every image bit for bit."""
    scene, view = scenes.cornell_box()
    kw = dict(enable_ssao=True, enable_rtr=True)
    wa, wb = parity.make_world(oracle_lib, scene, 160, 90, **kw), parity.make_world(cuda_lib, scene, 160, 90, **kw)
    cp = np.array(view["camera_position"], np.float32)
    for f in range(6):
        v = dict(view); v["camera_position"] = tuple(cp + np.array([0.02 * f, 0.0, -0.03 * f], np.float32))
        wa.render_frame(**v); wb.render_frame(**v)
        bad = parity.compare_images(wa, wb)
        assert not bad, (f, bad[:5])


@pytest.mark.gpu
def test_position_cache_is_invisible_on_gpu(cuda_lib):
    scene, view = scenes.cornell_box()
    wa, wb = parity.make_world(cuda_lib, scene, 320, 180), parity.make_world(cuda_lib, scene, 320, 180)
    wb.set_option(1, 0)
    for f in range(4):
        wa.render_frame(**view); wb.render_frame(**view)
        assert not parity.compare_images(wa, wb), f


@pytest.mark.gpu
def test_shadow_denoiser_on_gpu(oracle_lib, cuda_lib):
    """soft sun: trace shadow mask -> bitpack -> temporal -> 3 x spatial -> light gbuffer, camera in motion; every image bit for bit"""
    import math
    scene, view = scenes.cornell_box()
    wa, wb = parity.make_world(oracle_lib, scene, 200, 120, enable_lighting=True, enable_taa=True), parity.make_world(cuda_lib, scene, 200, 120, enable_lighting=True, enable_taa=True)
    for f in range(5):
        v = dict(view); px, py, pz = view["camera_position"]; v["camera_position"] = (px + 0.25 * math.sin(0.7 * f), py + 0.05 * f, pz - 0.1 * f)
        wa.render_frame(**v); wb.render_frame(**v)
        assert not parity.compare_images(wa, wb), f
    den = wb.image("shadow_denoise.spatial_input")[..., 0].astype(np.float32); geo = wb.image("depth")[..., 0] != 0
    assert ((den[geo] > 0.02) & (den[geo] < 0.98)).mean() > 0.01


# ------------------------------------------------------------------ BASELINE sizes (1080p): the oracle on the box's host threads takes a few seconds per frame
def test_cornell_1080p_lockstep_config2(oracle_lib, cuda_lib):
    """BASELINE configs[1] at its real size: Cornell 1920x1080, 1 spatial + 1 temporal pass, 4 frames, EVERY image bit for bit (the
    production kernels with their TMA tile staging — the small lockstep tests never have 16-byte aligned rows everywhere)."""
    scene, view = scenes.cornell_box()
    _, wb, report = parity.run_lockstep(oracle_lib, cuda_lib, scene, view, 1920, 1080, 4, spatial_reuse_pass_count=1)
    _assert_clean(report)
    assert wb.stats()["closest_rays"] > 100000


def test_atrium_1080p_rtdgi_rtr_taa_lockstep(oracle_lib, cuda_lib):
    """BASELINE configs[2]'s scene and size without the cache (whose ordered schedule the oracle does not restate): the 260 k-triangle atrium at 1920x1080, rtdgi with two spatial passes +
    reflections + TAA, camera in motion — the parallel production kernels of every pass but the cache's, every image bit for bit."""
    scene, view = scenes.atrium()
    kw = dict(enable_rtr=True, enable_taa=True, spatial_reuse_pass_count=2)
    wa, wb = parity.make_world(oracle_lib, scene, 1920, 1080, **kw), parity.make_world(cuda_lib, scene, 1920, 1080, **kw)
    cp = np.array(view["camera_position"], np.float32)
    for f in range(3):
        v = dict(view); v["camera_position"] = tuple(cp + np.array([0.05 * f, 0.01 * f, 0.02 * f], np.float32))
        wa.render_frame(**v); wb.render_frame(**v)
        bad = parity.compare_images(wa, wb)
        assert not bad, (f, bad[:5])


def test_atrium_full_path_serial_schedule_480x270(oracle_lib, cuda_lib):
    """the whole path (rtdgi + ircache + rtr + taa) on the full atrium with the cache passes on the serial schedule: bit for bit.  (One GPU thread
    walking 1080p would take minutes per pass; 480x270 exercises the same code on the same scene.)"""
    scene, view = scenes.atrium()
    kw = dict(enable_rtr=True, enable_ircache=True, enable_taa=True, spatial_reuse_pass_count=2)
    wa, wb = parity.make_world(oracle_lib, scene, 480, 270, **kw), parity.make_world(cuda_lib, scene, 480, 270, **kw)
    wb.set_debug_serial(True)
    for f in range(3):
        wa.render_frame(**view); wb.render_frame(**view)
        bad = parity.compare_images(wa, wb)
        assert not bad, (f, bad[:5])


def test_atrium_1080p_full_path_parallel_statistical(oracle_lib, cuda_lib):
    """BASELINE configs[2] exactly as bench.py times it — atrium 1080p, rtdgi + ircache + rtr + taa, the PARALLEL cache kernels — against the
    oracle's serial schedule.  Statistical by necessity (entries are assigned in cell order at the next chain, reposition votes go to the smallest
    hash, and no pixel sees an entry allocated earlier in the SAME pass): live cache entries within 5 %, mean of the GI / final images within 15 %, per-image RMS difference below 20 % of the
    image mean, mean L0 irradiance of the live entries within 40 % after 8 frames (a few samples per entry: the serial schedule lets late
    pixels of a pass hit entries the early ones just allocated, the parallel one does not)."""
    scene, view = scenes.atrium()
    kw = dict(enable_rtr=True, enable_ircache=True, enable_taa=True, spatial_reuse_pass_count=2)
    wa, wb = parity.make_world(oracle_lib, scene, 1920, 1080, **kw), parity.make_world(cuda_lib, scene, 1920, 1080, **kw)
    for f in range(12):
        wa.render_frame(**view); wb.render_frame(**view)
    a, b = _cache_summary(wa), _cache_summary(wb)
    m = {"alloc": (a["alloc"], b["alloc"]), "r0": (float(a["r0"].mean()), float(b["r0"].mean()))}
    for name in ("rtdgi.spatial_filtered", "taa.this_frame_out"):
        ia, ib = wa.image(name).astype(np.float64)[..., :3], wb.image(name).astype(np.float64)[..., :3]
        assert np.isfinite(ib).all(), name
        m[name] = (float(ia.mean()), float(ib.mean()), float(np.sqrt(((ia - ib) ** 2).mean())))
    print("atrium 1080p parallel-vs-serial:", m)
    assert abs(m["alloc"][0] - m["alloc"][1]) <= 0.05 * m["alloc"][0] + 2, m
    assert abs(m["r0"][0] - m["r0"][1]) <= 0.30 * abs(m["r0"][0]), m
    for name in ("rtdgi.spatial_filtered", "taa.this_frame_out"):
        ma, mb, rms = m[name]
        assert abs(ma - mb) <= 0.15 * ma, m     # the parallel schedule runs brighter while the cache fills
        assert rms <= 0.20 * ma, m
    # images that never see the cache are still exact: the G-buffer side and the reprojection map
    assert not parity.compare_images(wa, wb, names=["depth", "gbuffer", "reprojection_map", "half_depth", "half_view_normal"])


def test_parallel_cache_schedule_is_deterministic(cuda_lib):
    """The default (parallel) schedule of the irradiance cache decides independently of the order its threads run in: two worlds rendering the
    same frames of the full path — cache filling from cold, cells claimed, entries assigned, aged and moved by votes — hold the same bits in every
    image and buffer, the cache's included."""
    scene, view = scenes.atrium()
    kw = dict(enable_rtr=True, enable_ircache=True, enable_taa=True, spatial_reuse_pass_count=2)
    wa, wb = parity.make_world(cuda_lib, scene, 480, 270, **kw), parity.make_world(cuda_lib, scene, 480, 270, **kw)
    for f in range(12):
        wa.render_frame(**view); wb.render_frame(**view)
        bad = parity.compare_images(wa, wb)
        assert not bad, (f, bad[:8])
    assert int(wb.image("ircache.meta_buf").ravel()[3]) > 100


def test_async_cache_chain_matches_in_order_submission(cuda_lib):
    """From the fifth frame on the irradiance-cache chain of a frame runs on the async pass queue, under the previous frame's reflection filters + TAA
    (kjb_world_set_async_compute), and the frame is submitted as three graph recordings around the two ordering points.  The cache's ordered schedule
    makes the same decisions whatever the order its threads run in, so against the same frames submitted in program order on one queue every image
    and cache buffer is bit-identical after every frame; a difference means a missing dependency between the queues."""
    scene, view = scenes.atrium()
    kw = dict(enable_rtr=True, enable_ircache=True, enable_taa=True, spatial_reuse_pass_count=2)
    wa, wb = parity.make_world(cuda_lib, scene, 960, 540, **kw), parity.make_world(cuda_lib, scene, 960, 540, **kw)
    wb.set_async_compute(False)
    for f in range(16):
        wa.render_frame(**view); wb.render_frame(**view)
        bad = parity.compare_images(wa, wb)
        assert not bad, (f, bad[:8])
    ga, gb = wa.graph_stats(), wb.graph_stats()
    assert ga["launches"] == 3 * 12 and gb["launches"] == 12, (ga, gb)     # frames 4..15: three recordings per async frame, one per in-order frame
    assert ga["instantiations"] <= 4 and gb["instantiations"] <= 2, (ga, gb)
    assert {"ircache.aux_buf", "ircache.life_buf", "ircache.grid_meta_buf2", "taa.this_frame_out"} <= set(wa.image_names())
    assert int(wa.image("ircache.meta_buf").ravel()[3]) > 100


def test_cuda_graph_frames_match_directly_launched_frames(cuda_lib):
    """From the fifth frame on a frame's ~40 passes are recorded and submitted as ONE CUDA graph launch whose kernel-node parameters are updated
    in place every frame (ping-pong halves, frame constants).  Same bits as launching the kernels one by one — full path, camera in motion,
    and also through the streaming host-buffer call."""
    scene, view = scenes.cornell_box()
    kw = dict(enable_rtr=True, enable_ircache=False, enable_taa=True)
    wa, wb = parity.make_world(cuda_lib, glossy(scene), 320, 180, **kw), parity.make_world(cuda_lib, glossy(scene), 320, 180, **kw)
    wb.set_cuda_graph(False)
    cp = np.array(view["camera_position"], np.float32)
    for f in range(12):
        v = dict(view); v["camera_position"] = tuple(cp + np.array([0.02 * f, 0.0, -0.03 * f], np.float32))
        wa.render_frame(**v); wb.render_frame(**v)
        assert not parity.compare_images(wa, wb), f
    ga, gb = wa.graph_stats(), wb.graph_stats()
    assert ga["launches"] == 8 and ga["instantiations"] <= 2 and gb["launches"] == 0, (ga, gb)   # frames 4..11; one instance, updated in place
