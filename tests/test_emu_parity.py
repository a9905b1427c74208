"""Kernel LOGIC parity without a GPU: the unmodified .cu sources compiled for the CPU by the launch emulator
(tests/emu) against the oracle, frame by frame, every image bit-for-bit.  (The real CUDA build is checked by test_gpu_parity.py.)"""
import numpy as np
import parity
from kajiya_b200 import scenes


def _clean(report):
    bad = [(f, b) for f, frame in enumerate(report) for b in frame]
    assert not bad, bad[:10]


def test_cornell_lockstep(oracle_lib, emu_lib):
    scene, view = scenes.cornell_box()
    wa, wb, report = parity.run_lockstep(oracle_lib, emu_lib, scene, view, 96, 64, 7)
    _clean(report)
    assert wb.stats()["launches"] == 13 and len(wb.image_names()) >= 40


def test_cornell_odd_extent_single_spatial_pass(oracle_lib, emu_lib):
    scene, view = scenes.cornell_box()
    _, _, report = parity.run_lockstep(oracle_lib, emu_lib, scene, view, 53, 37, 5, spatial_reuse_pass_count=1)
    _clean(report)


def test_atrium_lockstep(oracle_lib, emu_lib):
    scene, view = scenes.atrium(target_tris=8000)
    _, _, report = parity.run_lockstep(oracle_lib, emu_lib, scene, view, 80, 48, 4)
    _clean(report)


def test_reference_path_tracer(oracle_lib, emu_lib):
    import numpy as np
    scene, view = scenes.cornell_box()
    wa, wb = parity.make_world(oracle_lib, scene, 40, 40), parity.make_world(emu_lib, scene, 40, 40)
    for _ in range(2):
        wa.render_reference(**view); wb.render_reference(**view)
    assert np.array_equal(wa.image("refpt.accum").view(np.uint32), wb.image("refpt.accum").view(np.uint32))


def test_gbuffer_ring_replay_and_host_upload_match(emu_lib):
    """The two bench legs feed the hot path differently — device-resident ring (`value`) vs host buffers uploaded inside the
    call (`e2e`) — and must produce identical frames."""
    import numpy as np
    scene, view = scenes.cornell_box()
    wc, wd = parity.make_world(emu_lib, scene, 64, 40), parity.make_world(emu_lib, scene, 64, 40)
    for i in range(3):
        wc.render_frame(capture_slot=i + 1, **view)
        wd.render_frame(**view)
    host = [[np.ascontiguousarray(wc.image(f"slot{i + 1}.{n}")) for n in ("gbuffer", "depth", "geometric_normal", "velocity")] for i in range(3)]
    result = np.zeros((40, 64, 4), np.float16)
    for i in range(3):
        wc.render_frame(replay_slot=i + 1, **view)
        wd.render_frame(host_inputs=tuple(a.ctypes.data for a in host[i]), host_result=result.ctypes.data, **view)
    names = [n for n in wc.image_names() if n.startswith("rtdgi.")]
    assert len(names) > 25 and not parity.compare_images(wc, wd, names)
    assert np.array_equal(result.view(np.uint16), wd.image("rtdgi.spatial_filtered").view(np.uint16))


def test_taa_native_and_upscaled(oracle_lib, emu_lib):
    """T1-T7 (taa.rs:41-185) at native resolution and with 1.5x temporal super-resolution"""
    scene, view = scenes.cornell_box()
    for kw in (dict(enable_taa=True), dict(enable_taa=True, upscale=(150, 96))):
        wa, wb, report = parity.run_lockstep(oracle_lib, emu_lib, scene, view, 100, 64, 5, **kw)
        _clean(report)
        assert "taa.this_frame_out" in wb.image_names() and wb.stats()["launches"] == 20


def _moving_views(view, frames):
    cp = np.array(view["camera_position"], np.float32)
    for f in range(frames):
        v = dict(view); v["camera_position"] = tuple(cp + np.array([0.07 * f, 0.013 * f, -0.09 * f], np.float32))
        if f >= 8:
            v["camera_rotation"] = (0.0, float(np.sin(0.6)), 0.0, float(np.cos(0.6)))   # turn away: entries age out and are recycled
        yield v


def test_ircache_lockstep(oracle_lib, emu_lib):
    """Irradiance cache on (ircache.rs): the emulator runs the cache-touching kernels block after block in launch order, the schedule
    the oracle restates, so every image AND every cache buffer (grid, pool, reservoirs, SH) must agree bit for bit."""
    scene, view = scenes.cornell_box()
    wa, wb, report = parity.run_lockstep(oracle_lib, emu_lib, scene, view, 96, 64, 6, enable_ircache=True)
    assert not [(f, b) for f, fr in enumerate(report) for b in fr]
    meta = wb.image("ircache.meta_buf").ravel()
    assert meta[3] > 100 and meta[2] >= meta[3]          # entries were allocated; entry_count >= alloc_count
    assert np.abs(wb.image("ircache.irradiance_buf")).max() > 0
    assert {"ircache.grid_meta_buf", "ircache.aux_buf", "ircache.entry_indirection_buf"} <= set(wb.image_names())


def test_ircache_moving_camera_scroll_and_recycle(oracle_lib, emu_lib):
    """Cascade scrolling (scroll_cascades.hlsl), deallocation of scrolled-out cells, aging and pool recycling, through the
    serial forms of the cache-touching kernels (kjb_set_debug_serial) on the kernel side — once with the cache alone, once with
    glossy reflections on, so that the reflection trace and validate passes run their serial forms too."""
    scene, view = scenes.cornell_box()
    for sc, rtr in ((scene, False), (_glossy(scene), True)):
        kw = dict(enable_ircache=True, enable_rtr=rtr, spatial_reuse_pass_count=1)
        wa, wb = parity.make_world(oracle_lib, sc, 80, 48, **kw), parity.make_world(emu_lib, sc, 80, 48, **kw)
        wb.set_debug_serial(True)
        peak = 0
        for f, v in enumerate(_moving_views(view, 16)):
            wa.render_frame(**v); wb.render_frame(**v)
            bad = parity.compare_images(wa, wb)
            assert not bad, (rtr, f, bad[:5])
            peak = max(peak, int(wb.image("ircache.meta_buf").ravel()[3]))
        meta = wb.image("ircache.meta_buf").ravel()
        assert meta[3] < peak and meta[2] > meta[3]       # entries were recycled: alloc_count fell below its peak and below entry_count


def _glossy(scene):
    import copy
    s = copy.deepcopy(scene)
    for i, m in enumerate(s[0][0]["materials"]):
        m["roughness"] = [0.05, 0.2, 0.35, 0.5, 0.8][i % 5]; m["metallic"] = [1.0, 0.0, 0.5][i % 3]
    return s


def test_rtr_lockstep(oracle_lib, emu_lib):
    """Reflections (rtr.rs): trace (only below roughness 0.6, else the diffuse candidates are reused), validate, temporal ReSTIR,
    resolve, temporal filter, cleanup — with glossy Cornell materials so that every branch runs, camera in motion so the
    reprojection search does too."""
    scene, view = scenes.cornell_box()
    scene = _glossy(scene)
    kw = dict(enable_rtr=True, spatial_reuse_pass_count=1)
    wa, wb = parity.make_world(oracle_lib, scene, 88, 56, **kw), parity.make_world(emu_lib, scene, 88, 56, **kw)
    cp = np.array(view["camera_position"], np.float32)
    for f in range(7):
        v = dict(view); v["camera_position"] = tuple(cp + np.array([0.03 * f, 0.01 * f, -0.04 * f], np.float32))
        wa.render_frame(**v); wb.render_frame(**v)
        bad = parity.compare_images(wa, wb)
        assert not bad, (f, bad[:5])
    names = set(wb.image_names())
    assert {"rtr.resolved", "rtr.temporal:0", "rtr.ray_len:0", "rtr.reservoir:0", "rtr.rng:0", "rtr.restir_invalidity"} <= names
    assert (wb.image("rtr.rng:0") != 0).mean() > 0.2          # reflection rays were traced (roughness <= 0.6)
    assert (wb.image("rtr.resolved") != 0).mean() > 0.3
    t = wb.image("rtr.temporal:0").astype(np.float32)
    assert np.isfinite(t[wb.image("depth")[..., 0] != 0]).all()


def test_rtr_with_ircache_and_taa(oracle_lib, emu_lib):
    """BASELINE config 3/4 shape: rtdgi + ircache + rtr (+ taa), every image and cache buffer bit for bit (serial cache schedule)."""
    scene, view = scenes.cornell_box()
    _, wb, report = parity.run_lockstep(oracle_lib, emu_lib, _glossy(scene), view, 80, 48, 6, enable_rtr=True, enable_ircache=True, enable_taa=True)
    _clean(report)
    assert wb.image("ircache.meta_buf").ravel()[3] > 50


def test_streaming_frames_match_blocking_frames(emu_lib):
    """kjb_world_frame.streaming (two input sets / result stages, copy queues): same bits as the blocking call."""
    scene, view = scenes.cornell_box()
    wa, wb = parity.make_world(emu_lib, scene, 64, 40), parity.make_world(emu_lib, scene, 64, 40)
    host = []
    for i in range(5):   # produce 5 frames' worth of host G-buffers with a third world
        wa.render_frame(**view)
        host.append([wa.image(n).copy() for n in ("gbuffer", "depth", "geometric_normal", "velocity")])
    wc = parity.make_world(emu_lib, scene, 64, 40)
    res_b = [np.zeros((40, 64, 4), np.float16) for _ in range(5)]; res_s = [np.zeros((40, 64, 4), np.float16) for _ in range(5)]
    for i in range(5):
        wb.render_frame(host_inputs=tuple(a.ctypes.data for a in host[i]), host_result=res_b[i].ctypes.data, **view)
        wc.render_frame(host_inputs=tuple(a.ctypes.data for a in host[i]), host_result=res_s[i].ctypes.data, streaming=True, **view)
    wc.wait()
    for i in range(5):
        assert np.array_equal(res_b[i].view(np.uint16), res_s[i].view(np.uint16)), i
    assert {"in0.gbuffer", "in1.gbuffer", "result.stage0", "result.stage1"} <= set(wc.image_names())


def test_restir_check_optional_pass(oracle_lib, emu_lib):
    """RtdgiRenderer::use_raytraced_reservoir_visibility: the optional "restir check" ray pass + importance-only ray march."""
    scene, view = scenes.cornell_box()
    wa, wb, report = parity.run_lockstep(oracle_lib, emu_lib, scene, view, 72, 44, 5, use_raytraced_reservoir_visibility=True)
    _clean(report)
    wc = parity.make_world(emu_lib, scene, 72, 44)
    for _ in range(5): wc.render_frame(**view)
    assert parity.compare_images(wb, wc, names=["rtdgi.irradiance"])   # the pass does change the result


def test_ssao_guide(oracle_lib, emu_lib):
    """SsgiRenderer (SURVEY §8f N3): the real screen-space occlusion guide instead of the constant 1 — ssao, spatial, upsample,
    temporal — feeding the rtdgi kernels, camera in motion (history reprojection)."""
    scene, view = scenes.cornell_box()
    kw = dict(enable_ssao=True, enable_rtr=True)
    wa, wb = parity.make_world(oracle_lib, scene, 96, 60, **kw), parity.make_world(emu_lib, scene, 96, 60, **kw)
    cp = np.array(view["camera_position"], np.float32)
    for f in range(6):
        v = dict(view); v["camera_position"] = tuple(cp + np.array([0.02 * f, 0.0, -0.03 * f], np.float32))
        wa.render_frame(**v); wb.render_frame(**v)
        bad = parity.compare_images(wa, wb)
        assert not bad, (f, bad[:5])
    ao = wb.image("ssao")[..., 0]; depth = wb.image("depth")[..., 0]
    assert {"ssgi.raw", "ssgi.spatial", "ssgi.upsampled", "ssgi:0", "ssgi:1"} <= set(wb.image_names())
    geo = ao[depth != 0]
    assert geo.min() < 200 and geo.max() > 230          # corners are occluded, open walls are not
    wc = parity.make_world(emu_lib, scene, 96, 60, enable_rtr=True)
    for f in range(6):
        v = dict(view); v["camera_position"] = tuple(cp + np.array([0.02 * f, 0.0, -0.03 * f], np.float32))
        wc.render_frame(**v)
    assert parity.compare_images(wb, wc, names=["rtdgi.irradiance"])   # the guide does steer the GI kernels


def test_lighting_composite_feeds_taa(oracle_lib, emu_lib):
    """SURVEY §8f N4: sun shadow mask trace + light_gbuffer (direct sun, emissive, rtdgi * albedo, rtr * FG, sky with the sun disk),
    whose output is what TAA then consumes; full path around it."""
    scene, view = scenes.cornell_box()
    kw = dict(enable_lighting=True, enable_rtr=True, enable_ircache=True, enable_taa=True, enable_ssao=True)
    wa, wb, report = parity.run_lockstep(oracle_lib, emu_lib, _glossy(scene), view, 96, 60, 5, **kw)
    _clean(report)
    out = wb.image("debug_out").astype(np.float32); gi = wb.image("rtdgi.spatial_filtered").astype(np.float32)
    depth = wb.image("depth")[..., 0]
    assert {"sun_shadow_mask", "accum", "debug_out", "taa.this_frame_out"} <= set(wb.image_names())
    assert np.isfinite(out[depth != 0]).all() and out[depth != 0][:, :3].mean() > 0.01
    m = wb.image("sun_shadow_mask")[..., 0]
    assert set(np.unique(m)) <= {0, 255}                  # 1 spp: lit or shadowed
    # hard sun: the configuration in which upstream skips its shadow denoiser too
    _, wc, report = parity.run_lockstep(oracle_lib, emu_lib, scene, view, 64, 40, 3, enable_lighting=True, hard_sun=True)
    _clean(report)


def _orbit(view, f):
    import math
    v = dict(view); px, py, pz = view["camera_position"]
    v["camera_position"] = (px + 0.25 * math.sin(0.7 * f), py + 0.05 * f, pz - 0.1 * f)
    return v


def test_shadow_denoiser(oracle_lib, emu_lib):
    """ShadowDenoiseRenderer (shadow_denoise.rs): bitpack, temporal (tile classification, moments, history clamp under a moving camera:
    disocclusions and the Catmull-Rom history fetch), three a-trous passes; every image bit for bit, odd extents included"""
    scene, view = scenes.cornell_box()
    for (w, h) in ((96, 60), (77, 45)):
        wa, wb = parity.make_world(oracle_lib, scene, w, h, enable_lighting=True), parity.make_world(emu_lib, scene, w, h, enable_lighting=True)
        for f in range(5):
            v = _orbit(view, f)
            wa.render_frame(**v); wb.render_frame(**v)
            assert not parity.compare_images(wa, wb), (w, h, f)
        names = set(wb.image_names())
        assert {"shadow_denoise.bitpacked", "shadow_denoise.metadata", "shadow_denoise.spatial_input", "shadow_denoise.temp", "shadow_denoise_accum:0", "shadow_denoise_moments:0"} <= names
        raw = wb.image("sun_shadow_mask")[..., 0].astype(np.float32) / 255.0
        den = wb.image("shadow_denoise.spatial_input")[..., 0].astype(np.float32)
        meta = wb.image("shadow_denoise.metadata")[: (h + 7) // 8, :, 0]
        bits = wb.image("shadow_denoise.bitpacked")[..., 0]
        assert ((meta & 1) == 0).any() and ((meta & 1) == 1).any()           # penumbra tiles are filtered, uniform ones are cleared
        geo = wb.image("depth")[..., 0] != 0                                   # sky texels are not shadow receivers: 0 in filtered tiles, 1 in all-lit ones
        assert ((den[geo] > 0.02) & (den[geo] < 0.98)).mean() > 0.01          # the 1-bit mask became a soft one ...
        assert abs(den[geo].mean() - raw[geo].mean()) < 0.05 and np.isfinite(den).all() and den.min() >= 0 and den.max() <= 1.25   # ... with the same amount of light (the Catmull-Rom history fetch may overshoot 1 a little, as upstream)
        # the bit masks are the mask: bit (y%4)*8 + x%8 of tile (x/8, y/4)
        yy, xx = np.mgrid[0:h, 0:w]
        assert np.array_equal(((bits[yy // 4, xx // 8] >> ((yy % 4) * 8 + (xx % 8))) & 1).astype(bool), raw > 0.5)


def _cornell_with_ceiling_light(lib, w, h, **kw):
    """the bundled Cornell box has no emitter: add a small emissive quad under the ceiling, registered as triangle lights (AddMeshOptions::use_lights)"""
    from kajiya_b200.world import World
    scene, view = scenes.cornell_box()
    world = World(lib, w, h, **kw)
    mesh, transforms = _glossy(scene)[0]
    hm = world.add_mesh(mesh)
    for t in transforms: world.add_instance(hm, t)
    P = np.array([[-0.3, 1.9, -0.3], [0.3, 1.9, -0.3], [0.3, 1.9, 0.3], [-0.3, 1.9, 0.3]], np.float32)
    light = dict(positions=P, normals=np.tile(np.array([0, -1, 0], np.float32), (4, 1)), indices=np.array([0, 1, 2, 0, 2, 3], np.uint32), material_ids=np.zeros(4, np.uint32),
                 materials=[dict(base_color=[0, 0, 0, 1], roughness=1.0, metallic=0.0, emissive=[17.0, 12.0, 4.0])])
    hl = world.add_mesh(light, use_lights=True)
    world.add_instance(hl, np.array([[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, 0]], np.float32))
    world.set_blue_noise(scenes.blue_noise()); world.set_spatial_resolve_offsets(scenes.spatial_resolve_offsets())
    return world, view


def test_triangle_light_specular(oracle_lib, emu_lib):
    """LightingRenderer::render_specular (lighting.rs): "sample lights" + "spatial reuse lights" add the emissive triangles' specular into the
    resolved reflections before their temporal filter; whole reflection path around it, every image bit for bit"""
    kw = dict(enable_rtr=True, enable_lighting=True, enable_taa=True)
    wa, view = _cornell_with_ceiling_light(oracle_lib, 88, 56, **kw); wb, _ = _cornell_with_ceiling_light(emu_lib, 88, 56, **kw)
    for f in range(4):
        v = _orbit(view, f)
        wa.render_frame(**v); wb.render_frame(**v)
        assert not parity.compare_images(wa, wb), f
    assert {"lighting.refl0", "lighting.refl1", "lighting.refl2"} <= set(wb.image_names())
    r0 = wb.image("lighting.refl0").astype(np.float32)
    assert (r0[..., 3] == 1).mean() > 0.3 and (r0[..., :3].max(-1) > 0).mean() > 0.1      # valid samples, a good part of them unshadowed
    assert wb.image("rtr.resolved").astype(np.float32).mean() > 0


def test_everything_at_once(oracle_lib, emu_lib):
    """every feature of the frame driver in one configuration — 2 spatial passes with ray-traced reservoir visibility, irradiance cache,
    reflections + triangle-light specular, SSAO guide, soft sun through the shadow denoiser, lit composite, TAA upsampling 1.5x — on the
    imported glTF fixture (textured, emissive-mapped lights) under camera motion: bit for bit, frame after frame"""
    from kajiya_b200 import asset
    from kajiya_b200.world import World
    import os, conftest
    path = os.path.join(conftest.ROOT, "tests", "golden", "gltf", "courtyard.gltf")
    view = dict(camera_position=(0.5, 2.5, 7.0), camera_rotation=(float(np.sin(-0.15)), 0.0, 0.0, float(np.cos(-0.15))), sun_direction=(0.35, 0.8, 0.45))
    kw = dict(spatial_reuse_pass_count=2, use_raytraced_reservoir_visibility=True, enable_ircache=True, enable_rtr=True, enable_ssao=True, enable_lighting=True, enable_taa=True, upscale=(108, 72))
    worlds = []
    for lib in (oracle_lib, emu_lib):
        sc = asset.GltfScene(path)
        w = World(lib, 72, 48, **kw)
        w.add_instance(w.add_mesh_desc(sc.desc, use_lights=True), np.array([[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, 0]], np.float32))
        w.set_blue_noise(scenes.blue_noise()); w.set_spatial_resolve_offsets(scenes.spatial_resolve_offsets())
        sc.close(); worlds.append(w)
    wa, wb = worlds
    for f in range(5):
        v = _orbit(view, f)
        wa.render_frame(**v); wb.render_frame(**v)
        assert not parity.compare_images(wa, wb), f
    names = set(wb.image_names())
    assert {"lighting.refl0", "shadow_denoise.spatial_input", "ssao", "rtr.resolved", "ircache.meta_buf", "taa.this_frame_out", "debug_out"} <= names
    assert wb.image("taa.this_frame_out").shape[:2] == (72, 108) and int(wb.image("ircache.meta_buf").ravel()[3]) > 20
    assert wb.stats()["passes"] >= 50        # render-graph passes of one frame


def test_position_cache_is_invisible(emu_lib):
    """KJB_OPTION_HALF_RES_POSITION_CACHE hoists hit_ws_from_uv_depth out of the D7/D9 neighbour loops: same bits, no extra launch when the producers cover the whole image"""
    scene, view = scenes.cornell_box()
    wa, wb = parity.make_world(emu_lib, scene, 70, 46), parity.make_world(emu_lib, scene, 70, 46)
    wb.set_option(1, 0)
    for f in range(4):
        wa.render_frame(**view); wb.render_frame(**view)
        assert not parity.compare_images(wa, wb), f
    assert wa.stats()["launches"] == wb.stats()["launches"]   # both position sets ride in kernels that run anyway (fused extract, restir temporal)


def test_shadow_denoiser_neighbourhood_against_a_plain_convolution(oracle_lib):
    """Independent pin of the denoiser's bit-mask arithmetic (three 8x4 tiles -> 17 horizontal taps, group-shared vertical pass): for tiles that
    are filtered, moments.w must equal the separable 17x17 FFX kernel applied to the binary mask with zero padding (fp16 storage tolerance)"""
    scene, view = scenes.cornell_box()
    w_, h_ = 90, 58
    w = parity.make_world(oracle_lib, scene, w_, h_, enable_lighting=True)
    w.render_frame(**view)
    mask = (w.image("sun_shadow_mask")[..., 0] > 127).astype(np.float64)
    k = np.exp(-3.0 * np.arange(9) ** 2 / 81.0); k = k / (k[0] + 2 * k[1:].sum())
    kern = np.concatenate([k[:0:-1], k])
    pad = np.pad(mask, 8)
    hor = sum(kern[i] * pad[8:-8, i:i + w_] for i in range(17))
    padv = np.pad(hor, ((8, 8), (0, 0)))
    want = sum(kern[i] * padv[i:i + h_] for i in range(17))
    got = w.image("shadow_denoise_moments:0")[..., 3].astype(np.float64)
    meta = w.image("shadow_denoise.metadata")[: (h_ + 7) // 8, : (w_ + 7) // 8, 0]
    filtered = np.kron((meta & 1) == 0, np.ones((8, 8), bool))[:h_, :w_]
    assert filtered.mean() > 0.05
    assert np.abs(got - want)[filtered].max() < 2e-3, np.abs(got - want)[filtered].max()
    # cleared tiles carry the uniform value instead
    cleared_lit = np.kron(meta == 3, np.ones((8, 8), bool))[:h_, :w_]
    assert (got[cleared_lit] == 1.0).all()


ORDERED_CACHE_SCHEDULE = 2   # KJB_OPTION_ORDERED_CACHE_SCHEDULE (kjb.h): the GPU's default, off in the emulator unless set


def _ordered_cache_invariants(w):
    """the bookkeeping of the ordered schedule: live entries = the allocated count, one entry per cell, every other entry free (none
    leaked), and no live entry at or beyond entry_count.  (The pool is rebuilt from the free entries at the start of each chain.)"""
    meta = w.image("ircache.meta_buf").ravel()
    life = w.image("ircache.life_buf").ravel()
    cell = w.image("ircache.entry_cell_buf").ravel()
    live = np.nonzero(life < 12)[0]
    assert int(meta[3]) == len(live), (int(meta[3]), len(live))
    assert len(set(cell[live].tolist())) == len(live)
    assert len(live) == 0 or int(live.max()) < int(meta[2])
    assert int((life == 0x8000001).sum()) + len(live) == len(life)


def test_ordered_cache_schedule_against_the_oracle(oracle_lib, emu_lib):
    """The GPU's default cache schedule (kjb_ircache.cuh) run by the emulator: claims wait for the next chain and take entries in cell
    order, keep-alives wait too, votes go to the smallest hash.  Under a moving camera (scrolling, deallocation, ageing, recycling) its
    bookkeeping stays consistent every frame; on a still camera it settles where the oracle's schedule does (live entries within 5 %,
    mean L0 irradiance of the live entries and of the GI image within 10 %)."""
    scene, view = scenes.cornell_box()
    kw = dict(enable_ircache=True, spatial_reuse_pass_count=1)
    w = parity.make_world(emu_lib, scene, 80, 48, **kw)
    w.set_option(ORDERED_CACHE_SCHEDULE, 1)
    peak = 0
    for v in _moving_views(view, 16):
        w.render_frame(**v)
        _ordered_cache_invariants(w)
        peak = max(peak, int(w.image("ircache.meta_buf").ravel()[3]))
    assert 0 < int(w.image("ircache.meta_buf").ravel()[3]) < peak         # entries were allocated and recycled

    wa, wb = parity.make_world(oracle_lib, scene, 96, 64, **kw), parity.make_world(emu_lib, scene, 96, 64, **kw)
    wb.set_option(ORDERED_CACHE_SCHEDULE, 1)
    for f in range(12):
        wa.render_frame(**view); wb.render_frame(**view)
    _ordered_cache_invariants(wb)
    def summary(x):
        life = x.image("ircache.life_buf").ravel()
        irr = x.image("ircache.irradiance_buf").reshape(-1, 3, 4)
        return int(x.image("ircache.meta_buf").ravel()[3]), float(irr[life < 12][:, :, 0].mean()), float(x.image("rtdgi.spatial_filtered").astype(np.float64)[..., :3].mean())
    (na, ra, ga), (nb, rb, gb) = summary(wa), summary(wb)
    assert abs(na - nb) <= 0.05 * na + 2, (na, nb)
    assert abs(ra - rb) <= 0.10 * abs(ra), (ra, rb)
    assert abs(ga - gb) <= 0.10 * ga, (ga, gb)


def test_cache_schedule_cannot_change_under_pending_claims(emu_lib):
    """the ordered schedule keeps claims pending until the next chain: switching to another schedule after it ran is refused"""
    import pytest
    from kajiya_b200._abi import KjbError
    scene, view = scenes.cornell_box()
    w = parity.make_world(emu_lib, scene, 48, 32, enable_ircache=True)
    w.set_option(ORDERED_CACHE_SCHEDULE, 1)
    w.render_frame(**view)
    with pytest.raises(KjbError):
        w.set_debug_serial(True)
    with pytest.raises(KjbError):
        w.set_option(ORDERED_CACHE_SCHEDULE, 0)
    w.render_frame(**view)
    _ordered_cache_invariants(w)
