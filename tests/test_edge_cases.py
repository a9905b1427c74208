"""Edge cases of the pass API: empty scene, degenerate extents, error behaviour (same code in the CUDA build — exercised here through
the CPU builds), instanced + moving geometry."""
import ctypes as C
import numpy as np, pytest
import parity
from parity import glossy
from kajiya_b200 import scenes
from kajiya_b200.world import World
from kajiya_b200._abi import Image, KjbError, FMT


def _empty_world(lib, w, h, **kw):
    wd = World(lib, w, h, **kw)
    wd.set_blue_noise(scenes.blue_noise()); wd.set_spatial_resolve_offsets(scenes.spatial_resolve_offsets())
    return wd


def test_empty_scene_is_all_sky(oracle_lib, emu_lib):
    """No meshes at all: every ray misses, every pass takes its depth == 0 branch; the full path must still run and agree."""
    _, view = scenes.cornell_box()
    kw = dict(enable_ircache=True, enable_rtr=True, enable_taa=True)
    wa, wb = _empty_world(oracle_lib, 40, 24, **kw), _empty_world(emu_lib, 40, 24, **kw)
    for f in range(4):
        wa.render_frame(**view); wb.render_frame(**view)
        assert not parity.compare_images(wa, wb), f
    assert (wb.image("depth") == 0).all()
    assert (wb.image("rtdgi.spatial_filtered")[..., :3] == 0).all()
    assert wb.image("ircache.meta_buf").ravel()[3] == 0          # nothing was allocated


@pytest.mark.parametrize("extent", [(1, 1), (2, 2), (3, 5), (17, 2)])
def test_degenerate_extents(oracle_lib, emu_lib, extent):
    """1x1 .. ragged tiny frames: half-res = div_up, blocks mostly out of range, stencils all clamp/zero paths."""
    scene, view = scenes.cornell_box()
    _, _, report = parity.run_lockstep(oracle_lib, emu_lib, scene, view, extent[0], extent[1], 4, enable_rtr=True, enable_taa=True)
    assert not [b for fr in report for b in fr]


def test_pass_argument_errors_are_reported(emu_lib):
    """Every entry point validates formats/extents and reports through the return code + kjb_last_error (no exceptions across the ABI)."""
    d = emu_lib.dll
    ctx = C.c_void_p(); assert d.kjb_create(0, C.byref(ctx)) == 0
    img = Image()
    assert d.kjb_image_alloc(ctx, 8, 8, 1, FMT["RGBA16_FLOAT"], C.byref(img)) == 0
    assert d.kjb_image_alloc(ctx, 0, 8, 1, FMT["RGBA16_FLOAT"], C.byref(Image())) != 0
    assert b"bad format or extent" in d.kjb_last_error(ctx)

    class ReprojArgs(C.Structure):   # kjb_rtdgi_reproject_args
        _fields_ = [("input_tex", Image), ("reprojection_tex", Image), ("output_tex", Image), ("output_tex_size", C.c_float * 4)]
    a = ReprojArgs(); a.input_tex = img; a.output_tex = img            # reprojection_tex left NULL
    d.kjb_pass_rtdgi_reproject.restype = C.c_int; d.kjb_pass_rtdgi_reproject.argtypes = [C.c_void_p, C.c_void_p]
    assert d.kjb_pass_rtdgi_reproject(ctx, C.byref(a)) != 0
    assert b"rtdgi reproject" in d.kjb_last_error(ctx) and b"null" in d.kjb_last_error(ctx)
    wrong = Image(); assert d.kjb_image_alloc(ctx, 8, 8, 1, FMT["R32_FLOAT"], C.byref(wrong)) == 0
    a.reprojection_tex = wrong
    assert d.kjb_pass_rtdgi_reproject(ctx, C.byref(a)) != 0
    assert b"format" in d.kjb_last_error(ctx)
    d.kjb_destroy(ctx)


def test_world_refuses_unsupported_combinations(emu_lib):
    with pytest.raises(KjbError):
        World(emu_lib, 64, 64, enable_lighting=True, tile=(0, 2))     # the lit composite (shadow-denoiser history) does not shard yet (DESIGN §7)
    with pytest.raises(KjbError):
        World(emu_lib, 64, 64, tile=(2, 2))                            # tile_rank must be < tile_count
    World(emu_lib, 64, 64, enable_rtr=True, tile=(0, 2)).close()      # reflections shard since round 2 (second all-gather carries this frame's GI)
    w = World(emu_lib, 32, 32, enable_rtr=True)
    w.set_blue_noise(scenes.blue_noise())
    _, view = scenes.cornell_box()
    with pytest.raises(KjbError):
        w.render_frame(**view)                                         # rtr needs SPATIAL_RESOLVE_OFFSETS from the host


def test_instanced_moving_geometry(oracle_lib, emu_lib):
    """Two instances of one mesh, one of them moving every frame: "rebuild tlas" re-flattens, velocities are non-zero, histories
    reproject — all bit for bit."""
    scene, view = scenes.cornell_box()
    mesh, transforms = scene[0]
    worlds = []
    for lib in (oracle_lib, emu_lib):
        w = World(lib, 72, 44, enable_rtr=True, enable_taa=True)
        h = w.add_mesh(mesh)
        w.add_instance(h, transforms[0])
        w.set_blue_noise(scenes.blue_noise()); w.set_spatial_resolve_offsets(scenes.spatial_resolve_offsets())
        worlds.append((w, h))
    small = np.array([[0.25, 0, 0, 0.1], [0, 0.25, 0, 0.3], [0, 0, 0.25, 0.2]], np.float32)
    ids = [w.add_instance(h, small) for w, h in worlds]
    for f in range(5):
        for (w, h), iid in zip(worlds, ids):
            if hasattr(w, "set_instance_transform"):
                t = small.copy(); t[0, 3] += 0.05 * f
                w.set_instance_transform(iid, t)
            w.render_frame(**view)
        assert not parity.compare_images(worlds[0][0], worlds[1][0]), f
    # "rebuild tlas" every frame as upstream: the first frame builds the structure, every later transform-only change is a device refit
    ts = worlds[1][0].tlas_stats()
    assert ts["rebuilds"] == 1 and ts["refits"] == 4, ts
    # the moving instance has object motion in its velocity (last frame's transform), the static one only camera motion (none here)
    vel = worlds[1][0].image("velocity").astype(np.float32)
    assert np.abs(vel[..., 0]).max() > 0.01
    assert (np.abs(vel[..., :3]).sum(-1) == 0).mean() > 0.5


def test_every_pass_entry_rejects_a_zeroed_argument_block(emu_lib):
    """all `kjb_pass_*` entries of include/kjb.h called with null images / buffers: an error code and a message naming the pass and the
    resource, never a crash (the closures upstream return Err and the graph panics with the pass name, graph.rs:989-993)"""
    import ctypes as C, re, os, conftest
    d = emu_lib.dll
    ctx = C.c_void_p(); assert d.kjb_create(-1, C.byref(ctx)) == 0
    names = sorted(set(re.findall(r"\b(kjb_pass_[a-z0-9_]+)\s*\(", open(os.path.join(conftest.ROOT, "include", "kjb.h")).read())))
    assert len(names) >= 56
    zero = (C.c_uint8 * 8192)()
    for n in names:
        f = getattr(d, n); f.restype = C.c_int; f.argtypes = [C.c_void_p, C.c_void_p]
        assert f(ctx, C.cast(zero, C.c_void_p)) != 0, n
        msg = d.kjb_last_error(ctx) or b""
        assert len(msg) > 8 and b":" in msg, (n, msg)
    d.kjb_destroy(ctx)


def test_remove_instance_and_emissive_multiplier(oracle_lib, emu_lib):
    """WorldRenderer::remove_instance is a swap_remove (the last instance takes the freed slot); InstanceDynamicParameters::emissive_multiplier
    scales emissive hits and the instance's triangle lights.  Frames before and after the edits: bit for bit on oracle and emulator."""
    import parity
    scene, view = scenes.cornell_box()
    mesh, transforms = scene[0]
    P = np.array([[-0.3, 1.9, -0.3], [0.3, 1.9, -0.3], [0.3, 1.9, 0.3], [-0.3, 1.9, 0.3]], np.float32)
    light = dict(positions=P, normals=np.tile(np.array([0, -1, 0], np.float32), (4, 1)), indices=np.array([0, 1, 2, 0, 2, 3], np.uint32), material_ids=np.zeros(4, np.uint32),
                 materials=[dict(base_color=[0, 0, 0, 1], roughness=1.0, metallic=0.0, emissive=[6.0, 5.0, 3.0])])
    ident = np.array([[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, 0]], np.float32)
    worlds = []
    for lib in (oracle_lib, emu_lib):
        w = World(lib, 64, 40)
        hm = w.add_mesh(mesh); hl = w.add_mesh(light, use_lights=True)
        a = w.add_instance(hm, transforms[0])
        b = w.add_instance(hm, np.array([[2, 0, 0, 4.5], [0, 2, 0, -1], [0, 0, 2, 0]], np.float32))   # a second box to the right
        c = w.add_instance(hl, ident)
        assert (a, b, c) == (0, 1, 2)
        w.set_blue_noise(scenes.blue_noise()); worlds.append((w, a, b, c))
    def frame():
        for w, *_ in worlds: w.render_frame(**view)
        assert not parity.compare_images(worlds[0][0], worlds[1][0])
    frame(); frame()
    lit = worlds[1][0].image("rtdgi.spatial_filtered").astype(np.float32).mean()
    for w, a, b, c in worlds: w.set_instance_emissive_multiplier(c, 0.0)
    for _ in range(6): frame()
    assert worlds[1][0].image("rtdgi.spatial_filtered").astype(np.float32).mean() < lit          # the light went dark
    for w, a, b, c in worlds: w.remove_instance(a)                                                # the light (last) moves into slot 0
    frame(); frame()
    depth = worlds[1][0].image("depth")[..., 0]
    ref = World(emu_lib, 64, 40); hm = ref.add_mesh(mesh); hl = ref.add_mesh(light, use_lights=True)
    ref.add_instance(hl, ident); ref.add_instance(hm, np.array([[2, 0, 0, 4.5], [0, 2, 0, -1], [0, 0, 2, 0]], np.float32))   # the order swap_remove leaves
    ref.set_blue_noise(scenes.blue_noise())
    ref.render_frame(**view); ref.render_frame(**view); ref.render_frame(**view)
    # same jitter sequence position? frame indices differ, so compare coverage rather than bits: the first box is gone, the second and the light stay
    assert abs((depth > 0).mean() - (ref.image("depth")[..., 0] > 0).mean()) < 0.02
    for w, a, b, c in worlds:
        with pytest.raises(KjbError):
            w.remove_instance(a)                                                                  # "no such instance"
        w.set_instance_transform(b, ident[None][0] * 1.0)                                         # handles of the survivors stay valid
    frame()


def test_sun_size_multiplier_at_run_time(oracle_lib, emu_lib):
    """WorldRenderer::sun_size_multiplier: a larger disk softens the shadows (denoiser on), 0 is the point sun (denoiser off, world_render_passes.rs:130)"""
    import parity
    scene, view = scenes.cornell_box()
    wa, wb = parity.make_world(oracle_lib, scene, 72, 44, enable_lighting=True), parity.make_world(emu_lib, scene, 72, 44, enable_lighting=True)
    def frames(n):
        for _ in range(n):
            wa.render_frame(**view); wb.render_frame(**view)
            assert not parity.compare_images(wa, wb)
    frames(2)
    raw1 = wb.image("sun_shadow_mask")[..., 0].astype(np.float32).copy(); launches_soft = wb.stats()["launches"]
    for w in (wa, wb): w.set_sun_size_multiplier(8.0)
    frames(3)
    geo = wb.image("depth")[..., 0] != 0
    # a disk 8x wider: more texels differ between two 1-spp masks of consecutive frames (wider penumbrae)
    m_a = wb.image("sun_shadow_mask")[..., 0].astype(np.float32).copy(); frames(1); m_b = wb.image("sun_shadow_mask")[..., 0].astype(np.float32)
    assert (m_a[geo] != m_b[geo]).mean() > 0.005
    for w in (wa, wb): w.set_sun_size_multiplier(0.0)
    frames(2)
    assert wb.stats()["launches"] == launches_soft - 5                   # bitpack + temporal + 3 spatial are gone
    with pytest.raises(KjbError):
        wb.set_sun_size_multiplier(-1.0)


def test_world_renderer_knobs(oracle_lib, emu_lib):
    """sun_color_multiplier / sky_ambient (re-bake the sky cubes), RenderOverrides (closest-hit shader), debug_shading_mode (lit composite):
    each change takes effect and stays bit-exact between oracle and emulator"""
    import parity
    scene, view = scenes.cornell_box()
    kw = dict(enable_lighting=True, enable_rtr=True)
    wa, wb = parity.make_world(oracle_lib, glossy(scene), 64, 40, **kw), parity.make_world(emu_lib, glossy(scene), 64, 40, **kw)
    def frames(n):
        for _ in range(n):
            wa.render_frame(**view); wb.render_frame(**view)
            assert not parity.compare_images(wa, wb)
        return wb.image("debug_out")[..., :3].astype(np.float32).copy(), wb.image("sky_cube").astype(np.float32).copy()
    base, sky0 = frames(3)
    for w in (wa, wb): w.set_sun_color_multiplier((0.2, 0.2, 1.5))
    tinted, sky1 = frames(3)
    assert not np.array_equal(sky0, sky1) and tinted[..., 2].mean() / max(tinted[..., 0].mean(), 1e-6) > base[..., 2].mean() / max(base[..., 0].mean(), 1e-6) * 1.5
    for w in (wa, wb): w.set_sun_color_multiplier((1, 1, 1)); w.set_sky_ambient((0.5, 0.5, 0.5))
    amb, sky2 = frames(3)
    assert sky2.mean() > sky0.mean()
    for w in (wa, wb): w.set_sky_ambient((0, 0, 0)); w.set_render_overrides(8, 0.25)      # NO_METAL + quarter roughness
    frames(3)
    for w in (wa, wb): w.set_render_overrides(0, 1.0); w.set_debug_shading_mode(2)           # diffuse GI only
    gi_only, _ = frames(2)
    for w in (wa, wb): w.set_debug_shading_mode(3)                                            # reflections only
    refl_only, _ = frames(2)
    assert not np.array_equal(gi_only, refl_only)
    for bad in (lambda: wb.set_debug_shading_mode(1), lambda: wb.set_debug_shading_mode(5), lambda: wb.set_render_overrides(16, 1.0)):
        with pytest.raises(KjbError):
            bad()


def test_reference_accumulation_reset(oracle_lib, emu_lib):
    """reset_reference_accumulation: the path tracer's running mean (accum.w = sample count) restarts from a cleared image"""
    import parity
    scene, view = scenes.cornell_box()
    wa, wb = parity.make_world(oracle_lib, scene, 40, 28), parity.make_world(emu_lib, scene, 40, 28)
    for _ in range(3):
        wa.render_reference(**view); wb.render_reference(**view)
    assert float(wb.image("refpt.accum")[..., 3].max()) == 3.0
    for w in (wa, wb): w.reset_reference_accumulation()
    moved = dict(view, camera_position=(0.5, 1.2, 6.0))
    wa.render_reference(**moved); wb.render_reference(**moved)
    a, b = wa.image("refpt.accum"), wb.image("refpt.accum")
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32)) and float(b[..., 3].max()) == 1.0


SCAN_SIZES = [1, 7, 8, 9, 1023, 8191, 8192, 8193, 40000, 65535, 65536]


def _scan_case(lib, n, seed=0, misalign=False):
    """kjb_pass_inclusive_prefix_scan_u32 on n seeded values (wrapping u32 sums) -> (got, want)"""
    d = lib.dll
    class Buf(C.Structure):
        _fields_ = [("data", C.c_void_p), ("size_bytes", C.c_uint64)]
    class ScanArgs(C.Structure):
        _fields_ = [("inout_buf", Buf), ("element_count", C.c_uint32)]
    for f in ("kjb_buffer_alloc", "kjb_buffer_upload", "kjb_buffer_download", "kjb_buffer_free", "kjb_pass_inclusive_prefix_scan_u32"):
        getattr(d, f).restype = C.c_int
    d.kjb_buffer_alloc.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p]
    d.kjb_buffer_upload.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64]
    d.kjb_buffer_download.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64]
    d.kjb_buffer_free.argtypes = [C.c_void_p, C.c_void_p]
    d.kjb_pass_inclusive_prefix_scan_u32.argtypes = [C.c_void_p, C.c_void_p]
    ctx = C.c_void_p(); assert d.kjb_create(0, C.byref(ctx)) == 0
    rng = np.random.default_rng(seed + n)
    vals = rng.integers(0, 2 ** 32 if n < 100 else 2 ** 18, size=n, dtype=np.uint64).astype(np.uint32)
    buf = Buf(); assert d.kjb_buffer_alloc(ctx, 4 * n + 16, C.byref(buf)) == 0
    view = Buf(buf.data + (4 if misalign else 0), 4 * n)     # a 4-byte-aligned sub-range exercises the scalar path of the CUDA kernel
    assert d.kjb_buffer_upload(ctx, C.byref(view), 0, vals.ctypes.data, 4 * n) == 0
    a = ScanArgs(view, n)
    assert d.kjb_pass_inclusive_prefix_scan_u32(ctx, C.byref(a)) == 0, d.kjb_last_error(ctx)
    assert d.kjb_sync(ctx) == 0
    got = np.zeros(n, np.uint32); assert d.kjb_buffer_download(ctx, C.byref(view), 0, got.ctypes.data, 4 * n) == 0
    assert d.kjb_buffer_free(ctx, C.byref(buf)) == 0
    d.kjb_destroy(ctx)
    return got, np.cumsum(vals.astype(np.uint64)).astype(np.uint32)


@pytest.mark.parametrize("n", SCAN_SIZES)
def test_prefix_scan_ragged_sizes(oracle_lib, emu_lib, n):
    """"_prefix scan" (prefix_scan.rs:10-39) at ragged element counts, against numpy's cumulative sum (mod 2^32)"""
    for lib in (oracle_lib, emu_lib):
        got, want = _scan_case(lib, n)
        assert np.array_equal(got, want), lib.backend
    got, want = _scan_case(emu_lib, n, misalign=True)
    assert np.array_equal(got, want)


@pytest.mark.gpu
@pytest.mark.parametrize("n", SCAN_SIZES)
def test_gpu_prefix_scan_ragged_sizes(cuda_lib, n):
    for mis in (False, True):
        got, want = _scan_case(cuda_lib, n, misalign=mis)
        assert np.array_equal(got, want), (n, mis)


class _Buf(C.Structure):
    _fields_ = [("data", C.c_void_p), ("size_bytes", C.c_uint64)]


class _CacheBindings(C.Structure):   # kjb_ircache_bindings (kjb.h): the reference's binding order
    _fields_ = [(n, _Buf) for n in ("meta_buf", "pool_buf", "reposition_proposal_buf", "reposition_proposal_count_buf", "grid_meta_buf", "entry_cell_buf",
                                    "spatial_buf", "irradiance_buf", "life_buf")]


def _cache_bindings(w):
    """kjb_ircache_bindings of a world's cache from the buffers the frame driver keeps by name"""
    Buf, Bindings = _Buf, _CacheBindings
    b = Bindings()
    for field, _ in Bindings._fields_:
        name = "ircache." + field
        if field == "grid_meta_buf" and w._cache_parity:
            name = "ircache.grid_meta_buf2"
        img = w.image_handle(name)
        setattr(b, field, Buf(img.data, img.width * img.height * w.lib.dll.kjb_format_texel_bytes(img.format)))
    return Bindings, Buf, b


def test_cache_request_exchange_between_two_replicas(emu_lib):
    """kjb_pass_ircache_export_requests / kjb_pass_ircache_merge_requests (the multi-GPU cache exchange, kjb.h): cache A has seen one half of the screen's
    rays, cache B the other half (two views).  After A's records are merged into B, every cell a screen ray of A keeps alive is occupied in B with a life no
    older than A's; the number of live entries grows by exactly the cells B did not have; merging the same block again changes nothing but vote counts."""
    scene, view = scenes.cornell_box()
    kw = dict(enable_ircache=True, spatial_reuse_pass_count=1)
    wa, wb = _empty_world(emu_lib, 96, 64, **kw), _empty_world(emu_lib, 96, 64, **kw)
    for w in (wa, wb):
        scenes.populate(w, scene)
    vb = dict(view, camera_position=(1.2, 1.4, 4.0))
    frames = 3
    for _ in range(frames):
        wa.render_frame(**view); wb.render_frame(**vb)
    d = emu_lib.dll
    for w in (wa, wb):
        w._cache_parity = frames % 2 == 0     # ircache_parity flips every frame after the first: which of the two grid_meta buffers is current
    BA, Buf, ba = _cache_bindings(wa)
    _, _, bb = _cache_bindings(wb)

    class ShareArgs(C.Structure):
        _fields_ = [("ircache", BA), ("block", Buf), ("max_records", C.c_uint32), ("seed", C.c_uint32)]
    for f in ("kjb_pass_ircache_export_requests", "kjb_pass_ircache_merge_requests", "kjb_buffer_alloc"):
        getattr(d, f).restype = C.c_int
    d.kjb_pass_ircache_export_requests.argtypes = [C.c_void_p, C.c_void_p]; d.kjb_pass_ircache_merge_requests.argtypes = [C.c_void_p, C.c_void_p]
    d.kjb_buffer_alloc.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p]
    R = 4096
    block = Buf(); assert d.kjb_buffer_alloc(wa.ctx, 16 + R * 32, C.byref(block)) == 0
    a = ShareArgs(ba, block, R, 0)
    assert d.kjb_pass_ircache_export_requests(wa.ctx, C.byref(a)) == 0, d.kjb_last_error(wa.ctx)
    wa.sync()
    rec = np.ctypeslib.as_array((C.c_uint32 * (4 + R * 8)).from_address(block.data)).copy()      # emulator: device memory is host memory
    n = int(rec[0]); assert 0 < n <= R
    cells, lives = rec[4:4 + n * 8].reshape(n, 8)[:, 0], rec[4:4 + n * 8].reshape(n, 8)[:, 1]
    assert len(set(cells.tolist())) == n and (lives < 8).all()                                    # one record per cell; ranks 0 and 1 only

    def state(w, b):
        gm = np.ctypeslib.as_array((C.c_uint32 * (b.grid_meta_buf.size_bytes // 4)).from_address(b.grid_meta_buf.data)).reshape(-1, 2)
        life = np.ctypeslib.as_array((C.c_uint32 * (b.life_buf.size_bytes // 4)).from_address(b.life_buf.data))
        meta = np.ctypeslib.as_array((C.c_uint32 * 8).from_address(b.meta_buf.data))
        return gm, life, meta
    gm_b, life_b, meta_b = state(wb, bb)
    occupied_before = (gm_b[cells, 1] & 1) != 0
    alloc_before = int(meta_b[3])
    m = ShareArgs(bb, block, R, 7)
    assert d.kjb_pass_ircache_merge_requests(wb.ctx, C.byref(m)) == 0, d.kjb_last_error(wb.ctx)
    wb.sync()
    assert ((gm_b[cells, 1] & 1) != 0).all()                                                      # every requested cell now lives in B
    assert int(meta_b[3]) == alloc_before + int((~occupied_before).sum())                         # allocations == the cells B lacked
    assert (life_b[gm_b[cells, 0]] <= lives).all()                                                # kept alive at least as well as in A
    alloc_after = int(meta_b[3]); life_after = life_b.copy()
    assert d.kjb_pass_ircache_merge_requests(wb.ctx, C.byref(m)) == 0
    wb.sync()
    assert int(meta_b[3]) == alloc_after and np.array_equal(life_b, life_after)                   # idempotent
    wb.render_frame(**vb); wb.render_frame(**vb)                                                  # the merged cache keeps working
    assert np.isfinite(wb.image("rtdgi.spatial_filtered").astype(np.float32)).all()
