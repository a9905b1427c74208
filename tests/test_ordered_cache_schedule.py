"""The irradiance cache's ordered schedule (KJB_OPTION_ORDERED_CACHE_SCHEDULE, kjb_ircache.cuh), the GPU's default and the schedule bench.py
times, tested as the deterministic schedule it claims to be: its frames do not change when the emulator runs blocks and threads in another
order, its entry assignment follows the rule it states (the n-th claimed cell in cell order takes the n-th free entry), it stays consistent
when the pool runs out and when replicas exchange requests, and the GPU renders the same bits as the emulator.  Every comparison is exact."""
import ctypes as C
import hashlib
import numpy as np
import pytest
import parity
from kajiya_b200 import scenes
from kajiya_b200._abi import KjbError
from parity import glossy
from test_emu_parity import _moving_views, _ordered_cache_invariants
from test_edge_cases import _cache_bindings

ORDERED_CACHE_SCHEDULE = 2            # KJB_OPTION_ORDERED_CACHE_SCHEDULE (kjb.h)
MAX_ENTRIES, CASCADE_CELLS = 1024 * 64, 32 ** 3
OCCUPIED, JUST_ALLOCATED = 1, 2
LIFE_RECYCLED = 0x8000001
FULL_PATH = dict(enable_ircache=True, enable_rtr=True, enable_taa=True, spatial_reuse_pass_count=2)
CACHE_BUFFERS = ("meta_buf", "grid_meta_buf", "grid_meta_buf2", "entry_cell_buf", "life_buf", "pool_buf", "spatial_buf", "irradiance_buf", "aux_buf",
                 "entry_indirection_buf", "reposition_proposal_buf", "reposition_proposal_count_buf")
ORDERS = ((0, 0), (1, 0), (2, 1), (2, 0x9E3779B9))   # (mode, seed) of kjb_emu_set_launch_order: forward, reverse, two permutations


@pytest.fixture
def launch_order(emu_lib):
    """sets the emulator's launch order (tests/emu/cuda_shim.cpp); forward again afterwards, whatever happens"""
    f = emu_lib.dll.kjb_emu_set_launch_order
    f.argtypes, f.restype = [C.c_int, C.c_uint32], None
    f(0, 0)
    try:
        yield lambda mode, seed=0: f(mode, seed)
    finally:
        f(0, 0)


def _digests(w):
    """raw bytes of every image and buffer: -0 / +0 and NaN payloads count as differences here"""
    return {n: hashlib.blake2b(w.image(n).tobytes(), digest_size=16).digest() for n in w.image_names()}


def _first_difference(runs):
    ref = runs[ORDERS[0]]
    for order, frames in runs.items():
        for f, (a, b) in enumerate(zip(ref, frames)):
            bad = sorted(n for n in a if a[n] != b.get(n))
            if bad or a.keys() != b.keys():
                return order, f, bad
    return None


def _render_in_orders(lib, set_order, scene, width, height, views, option, orders=ORDERS, **kw):
    runs = {}
    for mode, seed in orders:
        set_order(mode, seed)
        w = parity.make_world(lib, scene, width, height, **kw)
        w.set_option(ORDERED_CACHE_SCHEDULE, option)
        runs[(mode, seed)] = frames = []
        for v in views:
            w.render_frame(**v)
            frames.append(_digests(w))
        w.close()
    set_order(0)
    return runs


def _current_grid(frames_rendered):
    """the grid_meta buffer the cache's passes use after `frames_rendered` frames (the two swap at every chain after the first)"""
    return "ircache.grid_meta_buf2" if frames_rendered % 2 == 0 else "ircache.grid_meta_buf"


def _host_u32(w, name):
    """a cache buffer in place (emulator and oracle: device memory is host memory)"""
    h = w.image_handle(name)
    n = h.width * h.height * w.lib.dll.kjb_format_texel_bytes(h.format) // 4
    return np.ctypeslib.as_array((C.c_uint32 * n).from_address(h.data))


def _coords(cells):
    cells = np.asarray(cells, np.int64)
    return np.stack([cells & 31, (cells >> 5) & 31, (cells >> 10) & 31], -1), cells >> 15


def _pending_claims_and_free(w, frames_rendered):
    gm = w.image(_current_grid(frames_rendered)).reshape(-1, 2)
    life = w.image("ircache.life_buf").ravel()
    return np.nonzero((gm[:, 1] & 3) == 3)[0], np.nonzero(life == LIFE_RECYCLED)[0]


def _check_assignment(w, frames_rendered, claims, free, life_before, still):
    """numpy restatement of k_ircache_scroll_cascades' chain start (k_ircache_det_*): the n-th claimed cell in ascending cell order takes
    the n-th free entry in ascending entry order; on a moving camera the cell has moved with its cascade since (or scrolled out)"""
    life = w.image("ircache.life_buf").ravel()
    cell = w.image("ircache.entry_cell_buf").ravel()
    gm = w.image(_current_grid(frames_rendered)).reshape(-1, 2)
    assert len(claims) <= len(free), (len(claims), len(free))
    e = free[:len(claims)]
    newly_live = np.nonzero((life_before == LIFE_RECYCLED) & (life < 12))[0]
    if still:
        assert np.array_equal(newly_live, np.sort(e)), (len(newly_live), len(e))
        assert np.array_equal(cell[e], claims)
        assert np.array_equal(gm[claims, 0], e) and (gm[claims, 1] & OCCUPIED).all()
        return
    assert np.isin(newly_live, e).all()
    kept = life[e] < 12
    (q0, c0), (q1, c1) = _coords(claims), _coords(cell[e])
    for cascade in np.unique(c0):
        sel = c0 == cascade
        k = sel & kept
        if not k.any():
            continue
        assert (c1[k] == cascade).all()
        shift = q1[k] - q0[k]
        assert (shift == shift[0]).all(), (cascade, np.unique(shift, axis=0))        # one scroll per cascade
        gone = q0[sel & ~kept] + shift[0]
        assert ((gone < 0) | (gone >= 32)).any(-1).all(), cascade                     # recycled only because its cell scrolled out
        assert np.array_equal(gm[cell[e[k]], 0], e[k]) and (gm[cell[e[k]], 1] & OCCUPIED).all()


# ------------------------------------------------------------------------------------------------ CPU (the launch emulator)
def test_ordered_schedule_is_independent_of_launch_order(emu_lib, launch_order):
    """full path (rtdgi with 2 spatial passes + cache + reflections + taa) on a glossy Cornell box under a moving, turning camera (cascades scroll,
    entries are deallocated, age out and are recycled): forward, reverse and two permuted launch orders give the same raw bytes in every image
    and cache buffer after every frame"""
    scene, view = scenes.cornell_box()
    views = list(_moving_views(view, 16))
    runs = _render_in_orders(emu_lib, launch_order, glossy(scene), 80, 48, views, 1, **FULL_PATH)
    assert _first_difference(runs) is None, _first_difference(runs)
    names = set(runs[ORDERS[0]][-1])
    assert {"ircache." + b for b in CACHE_BUFFERS} <= names and {"rtr.resolved", "taa.this_frame_out"} <= names


def test_ordered_schedule_is_independent_of_launch_order_atrium(emu_lib, launch_order):
    scene, view = scenes.atrium(target_tris=12000)
    runs = _render_in_orders(emu_lib, launch_order, scene, 160, 90, [view] * 4, 1, **FULL_PATH)
    assert _first_difference(runs) is None, _first_difference(runs)


def test_reference_atomics_depend_on_launch_order(emu_lib, launch_order):
    """control for the two tests above: with the reference's atomics (which thread claims first decides the entry) reversing the launch order
    changes the cache buffers within the first frames, so the knob does reach the cache kernels"""
    scene, view = scenes.cornell_box()
    runs = _render_in_orders(emu_lib, launch_order, glossy(scene), 80, 48, list(_moving_views(view, 3)), 0, orders=ORDERS[:2], **FULL_PATH)
    diff = _first_difference(runs)
    assert diff is not None and any(n in diff[2] for n in ("ircache.entry_cell_buf", "ircache.grid_meta_buf", "ircache.grid_meta_buf2")), diff


@pytest.mark.parametrize("moving", [False, True])
def test_ordered_entry_assignment_rule(emu_lib, launch_order, moving):
    """pending claims (cells flagged OCCUPIED | JUST_ALLOCATED) at the end of a frame get their entries at the start of the next: the n-th
    claimed cell in ascending cell order takes the n-th free entry in ascending entry order; the bookkeeping invariants hold every frame"""
    scene, view = scenes.cornell_box()
    launch_order(2, 7)
    w = parity.make_world(emu_lib, glossy(scene), 80, 48, **FULL_PATH)
    w.set_option(ORDERED_CACHE_SCHEDULE, 1)
    views = list(_moving_views(view, 12)) if moving else [view] * 8
    checked = 0
    w.render_frame(**views[0])
    for f, v in enumerate(views[1:], start=1):
        claims, free = _pending_claims_and_free(w, f)
        life_before = w.image("ircache.life_buf").ravel().copy()
        w.render_frame(**v)
        _check_assignment(w, f + 1, claims, free, life_before, still=not moving)
        _ordered_cache_invariants(w)
        checked += len(claims)
    assert checked > 100


def _fill_cache_leaving(w, frames_rendered, keep, ordered):
    """make every free entry but `keep` live, in cells of cascades 10-11 that no ray of the scene reaches: live (life 0), pointing at their cell,
    the cell occupied and pointing back.  Returns the entries left free, in the order the cache hands them out."""
    gm = _host_u32(w, _current_grid(frames_rendered)).reshape(-1, 2)
    life, cell, meta, pool = (_host_u32(w, "ircache." + n) for n in ("life_buf", "entry_cell_buf", "meta_buf", "pool_buf"))
    assert not gm[10 * CASCADE_CELLS:].any()
    free = np.nonzero(life == LIFE_RECYCLED)[0]
    if ordered:   # the chain start rebuilds the pool from the free entries, lowest first
        kept, fill = free[:keep], free[keep:]
    else:         # the reference's atomics pop pool[alloc_count], pool[alloc_count + 1], ...
        order = pool[int(meta[3]):].copy()
        assert np.array_equal(np.sort(order), free)
        kept, fill = order[len(order) - keep:], order[:len(order) - keep]
    targets = 10 * CASCADE_CELLS + np.arange(len(fill), dtype=np.uint32)
    life[fill] = 0; cell[fill] = targets
    gm[targets, 0] = fill; gm[targets, 1] = OCCUPIED
    meta[2] = MAX_ENTRIES; meta[3] = MAX_ENTRIES - keep
    return kept


def test_ordered_pool_exhaustion_assigns_the_first_free_entries(emu_lib, launch_order):
    """k_ircache_det_assign when the claims outnumber the free entries: the first k claimed cells in cell order get the k free entries, the
    claims beyond have OCCUPIED | JUST_ALLOCATED cleared, and the bookkeeping stays consistent"""
    scene, view = scenes.cornell_box()
    launch_order(2, 3)
    w = parity.make_world(emu_lib, scene, 64, 40, enable_ircache=True, spatial_reuse_pass_count=1)
    w.set_option(ORDERED_CACHE_SCHEDULE, 1)
    for _ in range(2):
        w.render_frame(**view)
    w.sync()
    claims, _ = _pending_claims_and_free(w, 2)
    assert len(claims) >= 8, len(claims)
    k = len(claims) // 2
    _fill_cache_leaving(w, 2, k, ordered=True)
    free = np.nonzero(w.image("ircache.life_buf").ravel() == LIFE_RECYCLED)[0]
    assert len(free) == k
    w.stop_after("scroll cascades")             # the chain start, before any pass of the frame can claim again
    w.render_frame(**view)
    w.stop_after(None)
    life, cell = w.image("ircache.life_buf").ravel(), w.image("ircache.entry_cell_buf").ravel()
    gm = w.image(_current_grid(3)).reshape(-1, 2)
    assert np.array_equal(cell[free], claims[:k]) and (life[free] < 12).all()
    assert np.array_equal(gm[claims[:k], 0], free) and ((gm[claims[:k], 1] & 3) == 3).all()
    assert not (gm[claims[k:], 1] & (OCCUPIED | JUST_ALLOCATED)).any()
    assert not (life == LIFE_RECYCLED).any()
    _ordered_cache_invariants(w)


def test_reference_pool_exhaustion_matches_the_oracle(oracle_lib, emu_lib):
    """the reference atomics' undo path (ircache_lookup, alloc_idx >= 1024 * 64): the oracle and the emulator, poked into the same almost full
    cache, stay bit-identical through the frames that run the pool dry"""
    scene, view = scenes.cornell_box()
    kw = dict(enable_ircache=True, spatial_reuse_pass_count=1)
    wa, wb = parity.make_world(oracle_lib, scene, 64, 40, **kw), parity.make_world(emu_lib, scene, 64, 40, **kw)
    control = parity.make_world(emu_lib, scene, 64, 40, **kw)
    for _ in range(2):
        for w in (wa, wb, control):
            w.render_frame(**view)
        assert not parity.compare_images(wa, wb)
    before = int(control.image("ircache.meta_buf").ravel()[3])
    control.render_frame(**view)
    new = int(control.image("ircache.meta_buf").ravel()[3]) - before
    keep = 2
    assert new > keep, new                                          # the next frame claims more cells than the pool has left
    wa.sync(); wb.sync()
    kept = [_fill_cache_leaving(w, 2, keep, ordered=False) for w in (wa, wb)]
    assert np.array_equal(kept[0], kept[1])
    for f in range(2):
        wa.render_frame(**view); wb.render_frame(**view)
        bad = parity.compare_images(wa, wb)
        assert not bad, (f, bad[:5])
        assert int(wb.image("ircache.meta_buf").ravel()[3]) == MAX_ENTRIES    # full: the claims beyond were undone
    gm = wb.image(_current_grid(4)).reshape(-1, 2)
    life, cell = wb.image("ircache.life_buf").ravel(), wb.image("ircache.entry_cell_buf").ravel()
    assert (life < 12).all() and len(np.unique(cell)) == MAX_ENTRIES
    assert int((gm[:, 1] & OCCUPIED).astype(bool).sum()) == MAX_ENTRIES        # no cell left claimed without an entry


def _exchange_scenario(emu_lib):
    """cache A has seen one view, cache B another; A's requests are merged into B twice (ordered schedule on both), then B renders a frame.
    Returns what the assertions need and the raw state of B after the merge and after the frame."""
    scene, view = scenes.cornell_box()
    kw = dict(enable_ircache=True, spatial_reuse_pass_count=1)
    wa, wb = parity.make_world(emu_lib, scene, 96, 64, **kw), parity.make_world(emu_lib, scene, 96, 64, **kw)
    for w in (wa, wb):
        w.set_option(ORDERED_CACHE_SCHEDULE, 1)
    vb = dict(view, camera_position=(1.2, 1.4, 4.0))
    frames = 3
    for _ in range(frames):
        wa.render_frame(**view); wb.render_frame(**vb)
    d = emu_lib.dll
    for w in (wa, wb):
        w._cache_parity = frames % 2 == 0
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
    assert d.kjb_pass_ircache_export_requests(wa.ctx, C.byref(ShareArgs(ba, block, R, 0))) == 0, d.kjb_last_error(wa.ctx)
    wa.sync()
    rec = np.ctypeslib.as_array((C.c_uint32 * (4 + R * 8)).from_address(block.data)).copy()
    n = int(rec[0]); assert 0 < n <= R
    records = rec[4:4 + n * 8].reshape(n, 8)
    records = records[np.argsort(records[:, 0])]                     # slots are taken with atom_add: compare the records by cell
    grid = _current_grid(frames)
    out = dict(records=records, life_b=wb.image("ircache.life_buf").ravel().copy(), gm_b=wb.image(grid).reshape(-1, 2).copy(),
               alloc_b=int(wb.image("ircache.meta_buf").ravel()[3]))
    m = ShareArgs(bb, block, R, 7)
    assert d.kjb_pass_ircache_merge_requests(wb.ctx, C.byref(m)) == 0, d.kjb_last_error(wb.ctx)
    wb.sync()
    out["merged"] = {n: wb.image("ircache." + n).copy() for n in ("meta_buf", "life_buf", "entry_cell_buf", "grid_meta_buf", "grid_meta_buf2", "pool_buf")}
    assert d.kjb_pass_ircache_merge_requests(wb.ctx, C.byref(m)) == 0
    wb.sync()
    out["merged_twice"] = {n: wb.image("ircache." + n).copy() for n in out["merged"]}
    out["claims"], out["free"] = _pending_claims_and_free(wb, frames)
    out["digest_merged"] = _digests(wb)
    wb.render_frame(**vb)
    out["after_frame"] = {n: wb.image("ircache." + n).copy() for n in ("life_buf", "entry_cell_buf")}
    out["digest_after"] = _digests(wb)
    out["grid"], out["frames"] = grid, frames
    _ordered_cache_invariants(wb)
    wa.close(); wb.close()
    return out


def test_cache_request_exchange_on_the_ordered_schedule(emu_lib, launch_order):
    """kjb_pass_ircache_merge_requests with the ordered schedule on both replicas: the cells B lacked become claims (OCCUPIED | JUST_ALLOCATED,
    no allocation until B's next chain) and get their entries there in cell order; cells B held keep a life no older than A's; a second merge
    changes nothing but vote counts; and B's merged state is the same raw bytes under forward, reverse and permuted launch orders"""
    runs = {}
    for order in ORDERS:
        launch_order(*order)
        runs[order] = _exchange_scenario(emu_lib)
    launch_order(0)
    s = runs[ORDERS[0]]
    cells, lives = s["records"][:, 0], s["records"][:, 1]
    held = (s["gm_b"][cells, 1] & 3) == OCCUPIED
    assert (~held).sum() > 10 and held.sum() > 10, (held.sum(), (~held).sum())
    gm = s["merged"][s["grid"].split(".")[1]].reshape(-1, 2)
    assert ((gm[cells[~held], 1] & 3) == 3).all()                                   # claims ...
    assert int(s["merged"]["meta_buf"].ravel()[3]) == s["alloc_b"]                   # ... not allocations
    assert np.array_equal(gm[cells[held], 0], s["gm_b"][cells[held], 0])
    life_m = s["merged"]["life_buf"].ravel()
    assert (life_m[gm[cells[held], 0]] <= lives[held]).all()
    for n in ("meta_buf", "life_buf", "entry_cell_buf", "grid_meta_buf", "grid_meta_buf2", "pool_buf"):
        assert np.array_equal(s["merged"][n], s["merged_twice"][n]), n               # idempotent but for the vote counts
    assert np.isin(cells[~held], s["claims"]).all()
    # B's next frame: the pending claims, its own and the merged ones, take the free entries in cell order (still camera)
    after = s["after_frame"]
    e = s["free"][:len(s["claims"])]
    assert np.array_equal(after["entry_cell_buf"].ravel()[e], s["claims"]) and (after["life_buf"].ravel()[e] < 12).all()
    for order, r in runs.items():
        assert np.array_equal(r["records"], s["records"]), order
        assert r["digest_merged"] == s["digest_merged"], (order, sorted(k for k in s["digest_merged"] if s["digest_merged"][k] != r["digest_merged"].get(k)))
        assert r["digest_after"] == s["digest_after"], (order, sorted(k for k in s["digest_after"] if s["digest_after"][k] != r["digest_after"].get(k)))


# ------------------------------------------------------------------------------------------------ GPU against the emulator
def _gpu_against_emulator(cuda_lib, emu_lib, scene, width, height, views, **kw):
    """the GPU on its default schedule (not set: asserted to be the ordered one), the emulator on the ordered schedule; every image and cache
    buffer bit for bit after every frame"""
    wg, we = parity.make_world(cuda_lib, scene, width, height, **kw), parity.make_world(emu_lib, scene, width, height, **kw)
    we.set_option(ORDERED_CACHE_SCHEDULE, 1)
    for f, v in enumerate(views):
        wg.render_frame(**v); we.render_frame(**v)
        if f == 0:
            with pytest.raises(KjbError):          # refused once the ordered schedule holds pending claims: it is the GPU's default
                wg.set_debug_serial(True)
        bad = parity.compare_images(wg, we)
        assert not bad, (f, bad[:8])
    names = set(wg.image_names())
    assert {"ircache." + b for b in CACHE_BUFFERS} <= names
    assert int(wg.image("ircache.meta_buf").ravel()[3]) > 50
    return wg, we


@pytest.mark.gpu
def test_gpu_ordered_schedule_matches_the_emulator_cornell(cuda_lib, emu_lib):
    scene, view = scenes.cornell_box()
    _gpu_against_emulator(cuda_lib, emu_lib, glossy(scene), 160, 90, list(_moving_views(view, 16)), **FULL_PATH)


@pytest.mark.gpu
def test_gpu_ordered_schedule_matches_the_emulator_atrium(cuda_lib, emu_lib):
    scene, view = scenes.atrium()
    _gpu_against_emulator(cuda_lib, emu_lib, scene, 480, 270, [view] * 6, **FULL_PATH)


@pytest.mark.gpu
def test_gpu_headline_frame_matches_the_emulator_1080p(cuda_lib, emu_lib):
    """bench.py's headline configuration as it times it: the atrium at 1920x1080, rtdgi with 2 spatial passes + cache + reflections + taa, the
    GPU's default submission (CUDA graphs and the async cache chain from the fifth frame) — every image and cache buffer bit for bit"""
    scene, view = scenes.atrium()
    wg, _ = _gpu_against_emulator(cuda_lib, emu_lib, scene, 1920, 1080, [view] * 6, **FULL_PATH)
    assert wg.graph_stats()["launches"] > 0


@pytest.mark.gpu
def test_cuda_graph_frames_with_the_cache_match_directly_launched_frames(cuda_lib):
    """the cache's passes recorded into the frame's CUDA graph (kernel-node parameters updated in place every frame): every image and cache
    buffer bit for bit against launching the kernels one by one, full path with the cache, camera in motion"""
    scene, view = scenes.cornell_box()
    kw = dict(enable_rtr=True, enable_ircache=True, enable_taa=True)
    wa, wb = parity.make_world(cuda_lib, glossy(scene), 320, 180, **kw), parity.make_world(cuda_lib, glossy(scene), 320, 180, **kw)
    for w in (wa, wb):
        w.set_async_compute(False)
    wb.set_cuda_graph(False)
    cp = np.array(view["camera_position"], np.float32)
    for f in range(12):
        v = dict(view); v["camera_position"] = tuple(cp + np.array([0.02 * f, 0.0, -0.03 * f], np.float32))
        wa.render_frame(**v); wb.render_frame(**v)
        bad = parity.compare_images(wa, wb)
        assert not bad, (f, bad[:8])
    ga, gb = wa.graph_stats(), wb.graph_stats()
    assert ga["launches"] == 8 and ga["instantiations"] <= 2 and gb["launches"] == 0, (ga, gb)
    assert int(wa.image("ircache.meta_buf").ravel()[3]) > 50
