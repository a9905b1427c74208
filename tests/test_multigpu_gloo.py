"""Tile-sharded frames (SURVEY §8e) on CPU: world_size 2 and 3 over gloo.  Every rank renders its band of the frame with the
kernel emulator, exchanges tile borders through ONE all-gather per frame (kjb_allgather -> gloo callback) and must reproduce,
bit for bit, the rows of a single-process full-frame render."""
import ctypes as C, os, socket, sys
import numpy as np, pytest
import torch, torch.distributed as dist, torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

W, H, FRAMES = 64, 640, 5      # tall and narrow: bands of 160/107 half-res rows vs halos of 64-76 rows: every pass runs on a PARTIAL row range


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _worker(rank, world_size, port, enable_taa, H, ret, enable_rtr=False, host_inputs=False):
    sys.path.insert(0, ROOT); sys.path.insert(0, HERE)
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    os.environ["KJB_EMU_THREADS"] = "2"
    dist.init_process_group("gloo", rank=rank, world_size=world_size)
    from kajiya_b200._abi import KjbLib
    from kajiya_b200 import scenes
    import parity
    lib = KjbLib(os.path.join(HERE, "emu", "_build", "libkjb_emu.so"))
    scene, view = scenes.cornell_box()
    view = dict(view, camera_position=(0.0, 1.0, 5.0))
    kw = dict(enable_taa=enable_taa, spatial_reuse_pass_count=2, enable_ssao=(world_size == 2), enable_rtr=enable_rtr)   # the 2-rank case also runs the SSAO guide (whole image on every rank)
    if enable_rtr:   # glossy walls so that the reflection passes really trace (roughness <= 0.6)
        import copy
        scene = copy.deepcopy(scene)
        for i, m in enumerate(scene[0][0]["materials"]):
            m["roughness"] = [0.05, 0.2, 0.35, 0.5, 0.8][i % 5]; m["metallic"] = [1.0, 0.0, 0.5][i % 3]
    tiled = parity.make_world(lib, scene, W, H, tile=(rank, world_size), **kw)
    calls = [0]

    def allgather(send, recv, n):
        s = torch.frombuffer((C.c_uint8 * n).from_address(send), dtype=torch.uint8)
        r = torch.frombuffer((C.c_uint8 * (n * world_size)).from_address(recv), dtype=torch.uint8)
        dist.all_gather_into_tensor(r, s)
        calls[0] += 1
        return 0

    tiled.comm_set_callback(allgather, rank, world_size)
    full = parity.make_world(lib, scene, W, H, **kw)
    hh = (H + 1) // 2
    band_result = None
    for _ in range(FRAMES):
        full.render_frame(**view)
        if host_inputs:   # the G-buffer arrives from the host: the rank uploads ITS band, the bands travel through an extra all-gather, the result comes back band-wise
            inputs = [full.image(n).copy() for n in ("gbuffer", "depth", "geometric_normal", "velocity")]
            band_result = np.zeros((H, W, 4), np.float16)
            tiled.render_frame(host_inputs=tuple(a.ctypes.data for a in inputs), host_result=band_result.ctypes.data, **view)
        else:
            tiled.render_frame(**view)
    y0, y1 = hh * rank // world_size, hh * (rank + 1) // world_size
    bad = []
    names = ["rtdgi.spatial_filtered", "rtdgi.temporal_filtered", "rtdgi.irradiance"] + [n for n in full.image_names() if n.endswith(":0") or n.endswith(":1")]
    if enable_taa:
        names += ["taa.this_frame_out"]
    if enable_rtr:
        names += ["rtr.resolved"]
    for n in names:
        a, b = tiled.image(n), full.image(n)
        s = a.shape[0] // hh            # 1 for half-res images, 2 for full-res
        ra, rb = a[y0 * s:y1 * s].view(np.uint8), b[y0 * s:y1 * s].view(np.uint8)
        if not np.array_equal(ra, rb):
            bad.append((n, int((ra != rb).any(-1).sum())))
    if host_inputs:
        y0f, y1f = 2 * (hh * rank // world_size), 2 * (hh * (rank + 1) // world_size)
        want = full.image("taa.this_frame_out" if enable_taa else "rtdgi.spatial_filtered")
        if not np.array_equal(band_result[y0f:y1f].view(np.uint16), want[y0f:y1f].view(np.uint16)):
            bad.append(("host_result band", -1))
    ret[rank] = (bad, calls[0])
    dist.destroy_process_group()


# (4 ranks, 288 rows): bands of 36 half-res rows — narrower than the halo and than the exchanged border, as on 8 GPUs at 1080p:
# ranks need rows from beyond their direct neighbours and both border strips of a band coincide.
@pytest.mark.parametrize("world_size,enable_taa,height", [(2, False, H), (3, True, H), (4, False, 288)])
def test_tile_sharded_frames_match_single_process(world_size, enable_taa, height, emu_lib):
    ret = mp.Manager().dict()
    mp.spawn(_worker, args=(world_size, _free_port(), enable_taa, height, ret), nprocs=world_size, join=True)
    for rank in range(world_size):
        bad, calls = ret[rank]
        assert calls == FRAMES, "exactly one all-gather per frame"
        assert not bad, f"rank {rank}: band differs from the single-process frame: {bad}"


def _worker_ircache(rank, world_size, port, ret, full_path=False):
    """tiles + irradiance cache: every rank owns a replica of the cache, so only statistical agreement with the single-process frame is promised"""
    sys.path.insert(0, ROOT); sys.path.insert(0, HERE)
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port); os.environ["KJB_EMU_THREADS"] = "2"
    dist.init_process_group("gloo", rank=rank, world_size=world_size)
    from kajiya_b200._abi import KjbLib
    from kajiya_b200 import scenes
    import parity
    lib = KjbLib(os.path.join(HERE, "emu", "_build", "libkjb_emu.so"))
    scene, view = scenes.cornell_box()
    Wi, Hi, frames = 48, 768, 8      # bands of 192 half-res rows against halos of 52: each replica misses the rays of ~35 % of the frame
    kw = dict(enable_ircache=True, spatial_reuse_pass_count=1)
    if full_path:   # the bench's headline feature set: reflections (mid-frame GI gather, in place) + TAA + the cache exchange, all in one tile-sharded frame
        kw.update(enable_rtr=True, enable_taa=True, spatial_reuse_pass_count=2)
    tiled = parity.make_world(lib, scene, Wi, Hi, tile=(rank, world_size), **kw)

    def allgather(send, recv, n):
        s = torch.frombuffer((C.c_uint8 * n).from_address(send), dtype=torch.uint8)
        r = torch.frombuffer((C.c_uint8 * (n * world_size)).from_address(recv), dtype=torch.uint8)
        dist.all_gather_into_tensor(r, s)
        return 0

    tiled.comm_set_callback(allgather, rank, world_size)
    full = parity.make_world(lib, scene, Wi, Hi, **kw)
    for _ in range(frames):
        tiled.render_frame(**view); full.render_frame(**view)
    y0, y1 = Hi * rank // world_size, Hi * (rank + 1) // world_size
    name = "taa.this_frame_out" if full_path else "rtdgi.spatial_filtered"
    a = tiled.image(name)[y0:y1, :, :3].astype(np.float64); b = full.image(name)[y0:y1, :, :3].astype(np.float64)
    live = int(tiled.image("ircache.meta_buf").ravel()[3]), int(full.image("ircache.meta_buf").ravel()[3])
    ret[rank] = (bool(np.isfinite(a).all()), float(a.mean()), float(b.mean()), float(np.sqrt(((a - b) ** 2).mean())), live)
    dist.destroy_process_group()


@pytest.mark.parametrize("world_size", [2, 4])
def test_tile_sharded_frames_with_replicated_irradiance_cache(world_size, emu_lib):
    """Every rank keeps a replica of the cache and the replicas exchange their rays' requests each frame (kjb_pass_ircache_export_requests / _merge_requests):
    the band's mean GI within 10 % of the single-process frame's, RMS difference below 25 % of the mean (48 px wide frame: the noise of the band mean is
    several percent), and — the point of the exchange — every replica holds the single cache's number of live entries to within 5 % (without the exchange a
    replica only sees its band's rays: 65-85 %)."""
    ret = mp.Manager().dict()
    mp.spawn(_worker_ircache, args=(world_size, _free_port(), ret), nprocs=world_size, join=True)
    for rank in range(world_size):
        finite, ma, mb, rms, (la, lb) = ret[rank]
        print(f"rank {rank}: band mean {ma:.4f} vs {mb:.4f}, rms {rms:.4f}, live entries {la} vs {lb}")
        assert finite and mb > 0
        assert abs(ma - mb) <= (0.10 if world_size == 2 else 0.15) * mb, (rank, ma, mb)   # narrower bands: fewer texels in the mean
        assert rms <= 0.25 * mb, (rank, rms, mb)
        assert 0.95 * lb <= la <= 1.05 * lb, (rank, la, lb)


def test_tile_sharded_reflections_match_single_process(emu_lib):
    """rtdgi + reflections + taa on 2 ranks: the reflection passes run on the band plus their halos (resolve footprint, cleanup offsets, history
    search radius), this frame's GI travels in a second all-gather (reflection rays read it anywhere on screen) and every rtr history image
    joins the end-of-frame border exchange — each rank's band must still equal the single-process frame bit for bit."""
    ret = mp.Manager().dict()
    mp.spawn(_worker, args=(2, _free_port(), True, H, ret, True), nprocs=2, join=True)
    for rank in range(2):
        bad, calls = ret[rank]
        assert calls == 2 * FRAMES, "two all-gathers per frame: this frame's GI for the reflection rays, then the history borders"
        assert not bad, f"rank {rank}: band differs from the single-process frame: {bad}"


def test_tile_sharded_frames_with_host_inputs(emu_lib):
    """host G-buffers in, result out, 2 ranks: each rank uploads only its band of the inputs, an all-gather distributes the bands (NVLink on a multi-GPU box),
    the frame is rendered tile-sharded and each rank hands back its band of the result — bit-identical to the single-process frame"""
    ret = mp.Manager().dict()
    mp.spawn(_worker, args=(2, _free_port(), False, H, ret, False, True), nprocs=2, join=True)
    for rank in range(2):
        bad, calls = ret[rank]
        assert calls == 2 * FRAMES, "input bands + history borders"
        assert not bad, f"rank {rank}: {bad}"


def test_tile_sharded_reflections_on_eight_narrow_bands(emu_lib):
    """8 ranks x 288 rows: bands of 18 half-res rows against reflection halos of 70+ — every rank needs rows from several ranks away, both border strips of a
    band coincide, the GI all-gather feeds rays that land in any band.  rtdgi + reflections + taa, bit for bit (the geometry of 8 GPUs at 1080p / 1440p, where
    the bench's own parity check can only be statistical because the irradiance cache is on)."""
    ret = mp.Manager().dict()
    mp.spawn(_worker, args=(8, _free_port(), True, 288, ret, True), nprocs=8, join=True)
    for rank in range(8):
        bad, calls = ret[rank]
        assert calls == 2 * FRAMES
        assert not bad, f"rank {rank}: band differs from the single-process frame: {bad}"


def test_tile_sharded_full_path_with_cache_exchange(emu_lib):
    """The headline feature set on 2 ranks — rtdgi (2 spatial passes) + irradiance cache + reflections + TAA: four exchanges per frame (input-free: GI bands in
    place, history borders, cache requests).  Statistical like every cache-on comparison: finite, band mean of the TAA output within 10 %, RMS below 25 % of
    the mean, every replica within 5 % of the single cache's live entries."""
    ret = mp.Manager().dict()
    mp.spawn(_worker_ircache, args=(2, _free_port(), ret, True), nprocs=2, join=True)
    for rank in range(2):
        finite, ma, mb, rms, (la, lb) = ret[rank]
        print(f"rank {rank}: band mean {ma:.4f} vs {mb:.4f}, rms {rms:.4f}, live entries {la} vs {lb}")
        assert finite and mb > 0
        assert abs(ma - mb) <= 0.10 * mb and rms <= 0.25 * mb, (rank, ma, mb, rms)
        assert 0.95 * lb <= la <= 1.05 * lb, (rank, la, lb)
