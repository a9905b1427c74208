"""Tile-sharded frames with the irradiance cache on, bit for bit like one GPU.

On the ordered schedule (KJB_OPTION_ORDERED_CACHE_SCHEDULE = 1) the ranks' cache replicas exchange their pending requests exactly
(kjb_pass_ircache_export_pending / _merge_pending, kjb.h), so every replica stays the single-GPU cache.  After every frame, on every rank:
every cache buffer equals the untiled world's, the pending state (claims, keep-alives, votes; read back through the export) equals it,
and the rank's rows of every temporal image and of the result equal it.  The one exception is reposition_proposal_count_buf, a
max over ranks instead of a sum: only where it is non-zero must match.  CPU: the kernel emulator with gloo ranks.  GPU: several rank
processes on one H100 over the staged callback transport."""
import ctypes as C, os, sys
import numpy as np, pytest
import torch.distributed as dist, torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
from parity import glossy   # noqa: E402
from test_tile_upscaled import _compare_bands, _free_port, _gloo_allgather, _names, _view   # noqa: E402

ORDERED_CACHE_SCHEDULE = 2     # KJB_OPTION_ORDERED_CACHE_SCHEDULE (kjb.h)
MAX_ENTRIES, GRID_CELLS = 1 << 16, 32 * 32 * 32 * 12
BLOCK_BYTES = 256 + MAX_ENTRIES * 48   # KJB_IRCACHE_PENDING_BLOCK_BYTES
COUNT_BUF = "ircache.reposition_proposal_count_buf"


def _pending_api(lib):
    from test_edge_cases import _Buf, _CacheBindings

    class PendingArgs(C.Structure):   # kjb_ircache_pending_args
        _fields_ = [("ircache", _CacheBindings), ("blocks", _Buf), ("block_count", C.c_uint32)]
    d = lib.dll
    for f in ("kjb_pass_ircache_export_pending", "kjb_pass_ircache_merge_pending"):
        getattr(d, f).restype = C.c_int; getattr(d, f).argtypes = [C.c_void_p, C.c_void_p]
    d.kjb_buffer_alloc.restype = C.c_int; d.kjb_buffer_alloc.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p]
    return PendingArgs, _Buf


def _bindings(w, frames_rendered):
    from test_edge_cases import _cache_bindings
    w._cache_parity = frames_rendered % 2 == 0   # the grid_meta buffer of the last frame (the two swap at every chain after the first)
    return _cache_bindings(w)[2]


def _export(w, frames_rendered, block=None):
    """the world's pending state as kjb_pass_ircache_export_pending writes it: (header, entry part, claim part) as numpy arrays"""
    PendingArgs, Buf = _pending_api(w.lib)
    if block is None:
        block = Buf(); assert w.lib.dll.kjb_buffer_alloc(w.ctx, BLOCK_BYTES, C.byref(block)) == 0
    a = PendingArgs(_bindings(w, frames_rendered), block, 1)
    assert w.lib.dll.kjb_pass_ircache_export_pending(w.ctx, C.byref(a)) == 0, w.lib.dll.kjb_last_error(w.ctx)
    w.sync()
    raw = np.frombuffer(w.device_read(block.data, BLOCK_BYTES), np.uint32)
    E = MAX_ENTRIES
    proposal, claim_vertex = raw[64:64 + 4 * E].reshape(E, 4), raw[64 + 4 * E:64 + 8 * E].reshape(E, 4)
    life_pending, votes, cell, rank = (raw[64 + 8 * E + k * E:64 + 8 * E + (k + 1) * E] for k in range(4))
    return raw[:64].copy(), dict(proposal=proposal, life_pending=life_pending, votes=votes), dict(cell=cell, rank=rank, vertex=claim_vertex)


def _compare_cache(tiled, full, frames_rendered):
    """names of the cache buffers and pending parts that differ (the count buffer: only where it is non-zero)"""
    bad = []
    for n in full.image_names():
        if not n.startswith("ircache."):
            continue
        a, b = tiled.image(n), full.image(n)
        if n == COUNT_BUF:
            a, b = a != 0, b != 0
        if not np.array_equal(a.view(np.uint8) if a.dtype != bool else a, b.view(np.uint8) if b.dtype != bool else b):
            bad.append(n)
    (ha, ea, ca), (hb, eb, cb) = _export(tiled, frames_rendered), _export(full, frames_rendered)
    if not np.array_equal(ha, hb):
        bad.append(("pending header", ha[:2].tolist(), hb[:2].tolist()))
    for k in ("proposal", "life_pending"):
        if not np.array_equal(ea[k], eb[k]):
            bad.append(("pending " + k, int((ea[k] != eb[k]).reshape(MAX_ENTRIES, -1).any(-1).sum())))
    if not np.array_equal(ea["votes"] != 0, eb["votes"] != 0):
        bad.append("pending votes (non-zero)")
    n = int(hb[0])
    for k in ("cell", "rank", "vertex"):
        if not np.array_equal(ca[k][:n], cb[k][:n]):
            bad.append(("pending claim " + k, n))
    return bad, n


def _worker(rank, world_size, port, cfg, ret):
    sys.path.insert(0, ROOT); sys.path.insert(0, HERE)
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    os.environ["KJB_EMU_THREADS"] = "2"
    dist.init_process_group("gloo", rank=rank, world_size=world_size)
    from kajiya_b200._abi import KjbLib
    from kajiya_b200 import scenes
    import parity
    lib = KjbLib(os.path.join(HERE, "emu", "_build", "libkjb_emu.so"))
    if cfg.get("order"):
        f = lib.dll.kjb_emu_set_launch_order; f.argtypes, f.restype = [C.c_int, C.c_uint32], None
        f(*cfg["order"])
    W, H, up, rtr, taa = cfg["W"], cfg["H"], cfg.get("up"), cfg.get("rtr", False), cfg.get("taa", False)
    OH = up[1] if up else H
    scene, view = scenes.cornell_box()
    if rtr:
        scene = glossy(scene)
    kw = dict(enable_ircache=True, enable_taa=taa, enable_rtr=rtr, spatial_reuse_pass_count=cfg.get("spatial", 1), upscale=up)
    tiled = parity.make_world(lib, scene, W, H, tile=(rank, world_size), **kw)
    calls = [0]
    tiled.comm_set_callback(_gloo_allgather(world_size, calls), rank, world_size)
    full = parity.make_world(lib, scene, W, H, **kw)
    schedule = cfg.get("schedule", 1)
    for w in (tiled, full):
        w.set_option(ORDERED_CACHE_SCHEDULE, schedule)
    names = [n for n in _names(full, rtr) if taa or not n.startswith("taa")]
    frames, out = cfg.get("frames", 4), []
    for f in range(frames):
        v = _view(view, f, cfg.get("move", False))
        full.render_frame(**v); tiled.render_frame(**v)
        bad = _compare_bands(tiled, full, H, OH, rank, world_size, [n for n in names if n in full.image_names()])
        if schedule == 1:
            cache_bad, claims = _compare_cache(tiled, full, f + 1)
        else:
            cache_bad, claims = [n for n in full.image_names() if n.startswith("ircache.") and n != COUNT_BUF
                                 and not np.array_equal(tiled.image(n).view(np.uint8), full.image(n).view(np.uint8))], 0
        out.append((bad + cache_bad, claims, int(full.image("ircache.meta_buf").ravel()[3])))
        if f == cfg.get("exhaust_after", -1):   # every free entry but a few made live, on every replica alike (test_ordered_cache_schedule)
            from test_ordered_cache_schedule import _fill_cache_leaving
            for w in (tiled, full):
                w.sync(); _fill_cache_leaving(w, f + 1, cfg["keep"], ordered=True)
    probe = None
    if cfg.get("probe"):   # one more frame, stopped after the last cache user: this rank's own requests, before any exchange
        for w in (tiled, full):
            w.stop_after("reflection validate" if rtr else "rtdgi trace")
            w.render_frame(**_view(view, frames, cfg.get("move", False)))
        (ht, et, ct), (hf, ef, cf) = _export(tiled, frames + 1), _export(full, frames + 1)
        probe = (ct["cell"][:ht[0]].copy(), ct["rank"][:ht[0]].copy(), et["life_pending"].copy(), et["proposal"].any(-1),
                 cf["cell"][:hf[0]].copy(), cf["rank"][:hf[0]].copy(), ef["life_pending"].copy(), ef["proposal"].any(-1))
    ret[rank] = (out, calls[0] - (1 if probe is not None and rtr else 0), probe)   # the probe frame's GI gather
    dist.destroy_process_group()


def _run(world_size, cfg):
    ret = mp.Manager().dict()
    mp.spawn(_worker, args=(world_size, _free_port(), cfg, ret), nprocs=world_size, join=True)
    return [ret[r] for r in range(world_size)]


def _assert_exact(results, cfg):
    per_frame = 2 + bool(cfg.get("rtr"))   # history borders + cache exchange (+ this frame's GI for the reflection rays)
    claims = 0
    for rank, (frames, calls, _) in enumerate(results):
        assert calls == per_frame * len(frames), f"rank {rank}: {calls} all-gathers in {len(frames)} frames"
        for f, (bad, n, live) in enumerate(frames):
            assert not bad, f"rank {rank}, frame {f}: differs from the single-GPU frame: {bad}"
            claims += n
        assert frames[-1][2] > 50, frames[-1][2]    # the cache is really in use
    assert claims > 0
    if "exhaust_after" in cfg:                      # the chain after the fill had more claims than free entries
        assert results[0][0][cfg["exhaust_after"]][1] > cfg["keep"], results[0][0][cfg["exhaust_after"]][1]
    if cfg.get("probe"):
        # The halo rows: each rank's own requests before the exchange are requests the single frame makes too (a claimed cell, a keep-alive
        # no stronger, a vote only where the single frame votes), and together the ranks make all of them — no halo row invents one.
        probes = [p for _, _, p in results]
        cells_f, rank_f, life_f, vote_f = probes[0][4:]
        for r, (cells, ranks, life, vote, *_rest) in enumerate(probes):
            assert np.isin(cells, cells_f).all(), r
            assert (ranks <= rank_f[np.searchsorted(cells_f, cells)]).all() and (life <= life_f).all() and not (vote & ~vote_f).any(), r
        assert np.array_equal(np.unique(np.concatenate([p[0] for p in probes])), cells_f)
        assert np.array_equal(np.maximum.reduce([p[2] for p in probes]), life_f) and np.array_equal(np.logical_or.reduce([p[3] for p in probes]), vote_f)
        assert len(cells_f) > 0 and life_f.any()


# 2 and 4 ranks at 384 rows: bands of 96 / 48 half-res rows against halos of 40-60; 8 ranks: bands of 18, narrower than the halos
CASES = {
    "2_ranks_moving": (2, dict(W=48, H=384, move=True)),
    "4_ranks_moving": (4, dict(W=48, H=384, move=True)),
    "2_ranks_full_path": (2, dict(W=48, H=384, rtr=True, taa=True, spatial=2, move=True, probe=True)),
    "8_narrow_bands": (8, dict(W=32, H=288, taa=True, frames=3, probe=True)),
    "2_ranks_odd_height_upsampled": (2, dict(W=48, H=321, taa=True, up=(72, 482))),
    "2_ranks_pool_exhausted": (2, dict(W=48, H=384, exhaust_after=1, keep=6, frames=4)),
    "2_ranks_reversed_launch_order": (2, dict(W=48, H=384, move=True, order=(1, 0), frames=3)),
    "2_ranks_permuted_launch_order": (2, dict(W=48, H=384, move=True, order=(2, 0x9E3779B9), frames=3)),
}


@pytest.mark.parametrize("case", list(CASES))
def test_tiled_cache_frames_are_bit_identical(case, emu_lib):
    world_size, cfg = CASES[case]
    _assert_exact(_run(world_size, cfg), cfg)


def test_statistical_exchange_is_not_bit_identical(emu_lib):
    """control: the same tiled run on the reference's atomics takes the statistical exchange (kjb_pass_ircache_export_requests), and its
    replicas drift from the single cache"""
    results = _run(2, dict(W=48, H=384, move=True, schedule=0))
    assert any(bad for frames, _, _ in results for bad, _, _ in frames)


# ------------------------------------------------------------------------------------------------ the passes alone (CPU)
def _world(emu_lib, schedule, frames=1, **kw):
    import parity
    from kajiya_b200 import scenes
    scene, view = scenes.cornell_box()
    w = parity.make_world(emu_lib, scene, 64, 40, enable_ircache=True, spatial_reuse_pass_count=1, **kw)
    w.set_option(ORDERED_CACHE_SCHEDULE, schedule)
    for _ in range(frames):
        w.render_frame(**view)
    w.sync()
    return w, view


def test_pending_passes_refuse_the_reference_atomics_and_short_blocks(emu_lib):
    """schedule 0, a block one byte short, no block, zero blocks, two blocks to export: each an error with a message, nothing written"""
    PendingArgs, Buf = _pending_api(emu_lib)
    d = emu_lib.dll
    w0, _ = _world(emu_lib, 0)
    block = Buf(); assert d.kjb_buffer_alloc(w0.ctx, 2 * BLOCK_BYTES, C.byref(block)) == 0
    C.memset(block.data, 0xAB, 2 * BLOCK_BYTES)
    for f in (d.kjb_pass_ircache_export_pending, d.kjb_pass_ircache_merge_pending):
        assert f(w0.ctx, C.byref(PendingArgs(_bindings(w0, 1), block, 1))) != 0
        assert b"ordered cache schedule" in d.kjb_last_error(w0.ctx)
    w1, _ = _world(emu_lib, 1)
    b = _bindings(w1, 1)
    short = Buf(block.data, BLOCK_BYTES - 1)
    for f in (d.kjb_pass_ircache_export_pending, d.kjb_pass_ircache_merge_pending):
        for args in (PendingArgs(b, short, 1), PendingArgs(b, Buf(0, 0), 1), PendingArgs(b, block, 0), PendingArgs(b, Buf(block.data, BLOCK_BYTES), 2)):
            assert f(w1.ctx, C.byref(args)) != 0
            assert b"block" in d.kjb_last_error(w1.ctx)
    assert d.kjb_pass_ircache_export_pending(w1.ctx, C.byref(PendingArgs(b, block, 2))) != 0   # export writes one block
    assert (np.frombuffer((C.c_uint8 * (2 * BLOCK_BYTES)).from_address(block.data), np.uint8) == 0xAB).all()
    w0.close(); w1.close()


def test_claims_beyond_max_entries_are_dropped_exactly(emu_lib):
    """more claims than the cache has entries: A holds 70000 extra claims (merged in through the statistical pass), exports its first
    MAX_ENTRIES in cell order and B merges them.  B's pending claims are then A's first MAX_ENTRIES exactly; after the next chain start both
    caches are the same bits (the claims beyond were dropped on A and never reached B)"""
    PendingArgs, Buf = _pending_api(emu_lib)
    d = emu_lib.dll
    wa, view = _world(emu_lib, 1, frames=1)
    wb, _ = _world(emu_lib, 1, frames=1)

    class ShareArgs(C.Structure):
        from test_edge_cases import _Buf as B, _CacheBindings as CB
        _fields_ = [("ircache", CB), ("block", B), ("max_records", C.c_uint32), ("seed", C.c_uint32)]
    d.kjb_pass_ircache_merge_requests.restype = C.c_int; d.kjb_pass_ircache_merge_requests.argtypes = [C.c_void_p, C.c_void_p]
    extra = 70000
    rec = np.zeros((extra + 1) * 8, np.uint32)   # one 16-byte header + 32-byte records {cell, life, votes, 0, vertex}
    rec[0] = extra
    r = rec[4:4 + extra * 8].reshape(extra, 8)
    empty = np.nonzero(wa.image("ircache.grid_meta_buf").reshape(-1, 2)[:, 1] == 0)[0]
    r[:, 0] = empty[-extra:]                                     # the outer cascades, where no ray of the scene goes
    r[:, 1] = 4                                                  # rank 1
    r[:, 4:8] = np.float32(1.0).view(np.uint32)
    req = Buf(); assert d.kjb_buffer_alloc(wa.ctx, rec.nbytes, C.byref(req)) == 0
    C.memmove(req.data, rec.ctypes.data, rec.nbytes)
    assert d.kjb_pass_ircache_merge_requests(wa.ctx, C.byref(ShareArgs(_bindings(wa, 1), req, extra, 0))) == 0, d.kjb_last_error(wa.ctx)
    wa.sync()
    ha, ea, ca = _export(wa, 1)
    assert ha[0] == MAX_ENTRIES and ha[1] > extra, ha[:2]
    assert (np.diff(ca["cell"].astype(np.int64)) > 0).all()      # ascending cell order
    block = Buf(); assert d.kjb_buffer_alloc(wb.ctx, BLOCK_BYTES, C.byref(block)) == 0
    _export(wa, 1, block)
    assert d.kjb_pass_ircache_merge_pending(wb.ctx, C.byref(PendingArgs(_bindings(wb, 1), block, 1))) == 0, d.kjb_last_error(wb.ctx)
    wb.sync()
    hb, eb, cb = _export(wb, 1)
    assert hb[0] == MAX_ENTRIES and hb[1] == MAX_ENTRIES
    for k in ("cell", "rank", "vertex"):
        assert np.array_equal(ca[k], cb[k]), k
    for w in (wa, wb):
        w.stop_after("scroll cascades")
        w.render_frame(**view)
    bad = [n for n in wa.image_names() if n.startswith("ircache.") and n != COUNT_BUF and not np.array_equal(wa.image(n).view(np.uint8), wb.image(n).view(np.uint8))]
    assert not bad, bad
    wa.close(); wb.close()


def test_merge_is_idempotent_and_independent_of_block_order(emu_lib):
    """merging [A, B] or [B, A, A] into a third replica gives the same bits"""
    import parity
    from kajiya_b200 import scenes
    PendingArgs, Buf = _pending_api(emu_lib)
    d = emu_lib.dll
    scene, view = scenes.cornell_box()
    ws = []
    for cam in ((0.0, 1.0, 5.0), (1.2, 1.4, 4.0), (0.0, 1.0, 5.0), (0.0, 1.0, 5.0)):
        w = parity.make_world(emu_lib, scene, 64, 40, enable_ircache=True, spatial_reuse_pass_count=1)
        w.set_option(ORDERED_CACHE_SCHEDULE, 1)
        w.render_frame(**view)                          # identical first frame: identical replicas
        w.render_frame(**dict(view, camera_position=cam))
        w.sync(); ws.append(w)
    blocks = Buf(); assert d.kjb_buffer_alloc(ws[0].ctx, 3 * BLOCK_BYTES, C.byref(blocks)) == 0
    one = [Buf(blocks.data + k * BLOCK_BYTES, BLOCK_BYTES) for k in range(3)]
    _export(ws[0], 2, one[0]); _export(ws[1], 2, one[1])
    assert d.kjb_pass_ircache_merge_pending(ws[2].ctx, C.byref(PendingArgs(_bindings(ws[2], 2), Buf(blocks.data, 2 * BLOCK_BYTES), 2))) == 0
    _export(ws[1], 2, one[0]); _export(ws[0], 2, one[1]); _export(ws[0], 2, one[2])
    assert d.kjb_pass_ircache_merge_pending(ws[3].ctx, C.byref(PendingArgs(_bindings(ws[3], 2), blocks, 3))) == 0
    for w in ws:
        w.sync()
    bad, _ = _compare_cache(ws[3], ws[2], 2)
    assert not bad, bad
    assert not np.array_equal(ws[2].image("ircache.grid_meta_buf2"), ws[0].image("ircache.grid_meta_buf2"))   # B's claims did arrive
    for w in ws:
        w.close()


# ------------------------------------------------------------------------------------------------ GPU
def _gpu_worker(rank, world_size, port, ret):
    sys.path.insert(0, ROOT); sys.path.insert(0, HERE)
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    os.environ.pop("TORCHELASTIC_USE_AGENT_STORE", None)
    import torch
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=world_size)
    import kajiya_b200
    from kajiya_b200 import scenes
    import parity
    lib = kajiya_b200.lib()
    scene, view = scenes.atrium()
    W, H = 480, 270
    kw = dict(enable_ircache=True, enable_taa=True, enable_rtr=True, spatial_reuse_pass_count=2)
    tiled = parity.make_world(lib, scene, W, H, device=0, tile=(rank, world_size), **kw)
    calls = [0]
    tiled.comm_set_callback(_gloo_allgather(world_size, calls, staged_world=tiled), rank, world_size)
    full = parity.make_world(lib, scene, W, H, device=0, **kw)
    for w in (tiled, full):   # the GPU's default schedule, CUDA graphs and async compute: asserted, not set
        assert lib.dll.kjb_get_option is not None
        v = C.c_uint32(); lib.dll.kjb_get_option.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p]
        assert lib.dll.kjb_get_option(w.ctx, ORDERED_CACHE_SCHEDULE, C.byref(v)) == 0 and v.value == 1
    out = []
    names = _names(full, True)
    for f in range(6):
        full.render_frame(**view); tiled.render_frame(**view)
        bad = _compare_bands(tiled, full, H, H, rank, world_size, names)
        cache_bad, claims = _compare_cache(tiled, full, f + 1)
        out.append((bad + cache_bad, claims, int(full.image("ircache.meta_buf").ravel()[3])))
    ret[rank] = (out, calls[0], full.graph_stats()["launches"])
    dist.destroy_process_group()


@pytest.mark.gpu
@pytest.mark.parametrize("world_size", [2, 3])
def test_gpu_tiled_cache_frames_are_bit_identical(world_size):
    """2 / 3 rank processes share one H100 over the staged callback: the atrium at 480x270, full path with the cache, CUDA graphs and async
    compute from the fifth frame, 6 frames — every image band and cache buffer of every rank after every frame equals the single-GPU world"""
    ret = mp.Manager().dict()
    mp.spawn(_gpu_worker, args=(world_size, _free_port(), ret), nprocs=world_size, join=True)
    for rank in range(world_size):
        frames, calls, graph_launches = ret[rank]
        assert calls == 3 * 6, calls
        assert graph_launches > 0
        for f, (bad, n, live) in enumerate(frames):
            assert not bad, f"rank {rank}, frame {f}: {bad}"
        assert frames[-1][2] > 50
