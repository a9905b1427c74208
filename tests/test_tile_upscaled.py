"""Tile-sharded frames with temporal upsampling (TAA output larger than the render extent) and odd render heights.

A rank owns half-res rows [b0, b1) of the render grid, full-res rows [2·b0, 2·b1) clipped to H, and the result rows that
kjb_world_result_rows reports: floor(OH·min(2b, H)/H) at each band boundary.  Every rank's rows of every temporal image, on the
grid the image lives on, must equal the same rows of a single-process render bit for bit.  CPU: the kernel emulator with gloo
ranks.  GPU: several rank processes on one H100 over the callback transport with host-staged gloo, and NCCL where there are
two GPUs or more."""
import ctypes as C, os, socket, sys
import numpy as np, pytest
import torch, torch.distributed as dist, torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
FRAMES = 5


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _view(view, frame, move):
    # `move`: the camera rises by 0.002 per frame at 5 units from the box, about a quarter of a render row per frame at H = 640, inside the
    # motion bound of the exchanged borders (one render row per frame, DESIGN §7)
    return dict(view, camera_position=(0.0, 1.0 + (0.002 * frame if move else 0.0), 5.0))


def _band_rows(h, rank, n):
    """(half-res rows, full-res rows) of rank's band: the balanced split of the half-res rows, full-res rows clipped to h"""
    hh = (h + 1) // 2
    b0, b1 = hh * rank // n, hh * (rank + 1) // n
    return (b0, b1), (min(2 * b0, h), min(2 * b1, h))


def _compare_bands(tiled, full, h, oh, rank, n, names):
    """names of images whose owned rows differ, with the count of differing texels"""
    hh = (h + 1) // 2
    (b0, b1), (f0, f1) = _band_rows(h, rank, n)
    o0, o1 = tiled.result_rows()
    bad = []
    for name in names:
        a, b = tiled.image(name), full.image(name)
        rows = a.shape[0]
        if name.split(":")[0] in ("taa", "taa.velocity", "taa.smooth_var", "taa.this_frame_out"):
            assert rows == oh, name
            y0, y1 = o0, o1                          # the output grid
        elif rows == h:
            y0, y1 = f0, f1
        elif rows == hh:
            y0, y1 = b0, b1
        else:
            continue
        ra, rb = a[y0:y1].view(np.uint8), b[y0:y1].view(np.uint8)
        if y1 <= y0 or not np.array_equal(ra, rb):
            bad.append((name, int((ra != rb).any(-1).sum()) if y1 > y0 else -1))
    return bad


def _names(full, enable_rtr):
    names = ["rtdgi.spatial_filtered", "rtdgi.temporal_filtered", "rtdgi.irradiance", "taa.this_frame_out"]
    names += [n for n in full.image_names() if n.endswith(":0") or n.endswith(":1")]
    if enable_rtr:
        names += ["rtr.resolved"]
    return names


def _gloo_allgather(world_size, calls, staged_world=None):
    """all-gather callback over gloo; `staged_world`: the callback receives device pointers (CUDA build) and stages them through the host"""
    def allgather(send, recv, n):
        if staged_world is None:
            s = torch.frombuffer((C.c_uint8 * n).from_address(send), dtype=torch.uint8)
            r = torch.frombuffer((C.c_uint8 * (n * world_size)).from_address(recv), dtype=torch.uint8)
            dist.all_gather_into_tensor(r, s)
        else:
            s = torch.from_numpy(staged_world.device_read(send, n))
            r = torch.empty(n * world_size, dtype=torch.uint8)
            dist.all_gather_into_tensor(r, s)
            staged_world.device_write(recv, r.numpy())
        calls[0] += 1
        return 0
    return allgather


def _worker(rank, world_size, port, cfg, ret):
    sys.path.insert(0, ROOT); sys.path.insert(0, HERE)
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    os.environ["KJB_EMU_THREADS"] = "2"
    dist.init_process_group("gloo", rank=rank, world_size=world_size)
    from kajiya_b200._abi import KjbLib
    from kajiya_b200 import scenes
    import parity
    lib = KjbLib(os.path.join(HERE, "emu", "_build", "libkjb_emu.so"))
    W, H, up, rtr = cfg["W"], cfg["H"], cfg.get("up"), cfg.get("rtr", False)
    OH = up[1] if up else H
    scene, view = scenes.cornell_box()
    if rtr:
        scene = parity.glossy(scene)
    kw = dict(enable_taa=True, spatial_reuse_pass_count=2, enable_rtr=rtr, upscale=up)
    tiled = parity.make_world(lib, scene, W, H, tile=(rank, world_size), **kw)
    calls = [0]
    tiled.comm_set_callback(_gloo_allgather(world_size, calls), rank, world_size)
    full = parity.make_world(lib, scene, W, H, **kw)
    assert full.result_rows() == (0, OH)
    host, streaming = cfg.get("host_inputs", False), cfg.get("streaming", False)
    keep, results = [], []
    for f in range(FRAMES):
        v = _view(view, f, cfg.get("move", False))
        full.render_frame(**v)
        if host:   # the G-buffer from the host, the result back to the host: each rank's rows of it
            inputs = [full.image(n).copy() for n in ("gbuffer", "depth", "geometric_normal", "velocity")]
            result = np.zeros((OH, up[0] if up else W, 4), np.float16)
            keep.append(inputs); results.append(result)
            tiled.render_frame(host_inputs=tuple(a.ctypes.data for a in inputs), host_result=result.ctypes.data, streaming=streaming, **v)
        else:
            tiled.render_frame(**v)
    if streaming:
        tiled.wait()
    bad = _compare_bands(tiled, full, H, OH, rank, world_size, _names(full, rtr))
    if host:
        o0, o1 = tiled.result_rows()
        want = full.image("taa.this_frame_out")
        if not np.array_equal(results[-1][o0:o1].view(np.uint16), want[o0:o1].view(np.uint16)):
            bad.append(("host_result rows", -1))
        if results[-1][:o0].any() or results[-1][o1:].any():
            bad.append(("host_result wrote outside the owned rows", -1))
    ret[rank] = (bad, calls[0], tiled.result_rows())
    dist.destroy_process_group()


def _run(world_size, cfg):
    ret = mp.Manager().dict()
    mp.spawn(_worker, args=(world_size, _free_port(), cfg, ret), nprocs=world_size, join=True)
    oh = cfg["up"][1] if cfg.get("up") else cfg["H"]
    per_frame = 1 + bool(cfg.get("rtr")) + bool(cfg.get("host_inputs"))   # history borders (+ this frame's GI for the reflection rays) (+ the input bands)
    rows = []
    for rank in range(world_size):
        bad, calls, result_rows = ret[rank]
        assert calls == per_frame * FRAMES, f"rank {rank}: {calls} all-gathers in {FRAMES} frames"
        assert not bad, f"rank {rank}: band differs from the single-process frame: {bad}"
        rows.append(result_rows)
    assert rows[0][0] == 0 and rows[-1][1] == oh and all(rows[i][1] == rows[i + 1][0] for i in range(world_size - 1)), rows


# W x H -> upscale: 1.5x, 2x, and 2.5 output rows per half-res row (64x288 -> 80x360 and 64x640 -> 80x800); 4 and 8 ranks at 288 rows give bands
# of 36 / 18 half-res rows, narrower than the halos: ranks need rows from beyond their direct neighbours and both border strips of a band coincide.
CASES = {
    "2_ranks_1.5x_reflections": (2, dict(W=64, H=640, up=(96, 960), rtr=True)),
    "3_ranks_2x": (3, dict(W=64, H=640, up=(128, 1280))),
    "4_ranks_2.5_rows_per_half_row": (4, dict(W=64, H=288, up=(80, 360))),
    "8_ranks_2x_reflections": (8, dict(W=64, H=288, up=(128, 576), rtr=True)),
    "2_ranks_800_of_640": (2, dict(W=64, H=640, up=(80, 800))),
    "2_ranks_odd_height_upsampled": (2, dict(W=64, H=321, up=(96, 482))),
    "3_ranks_odd_height": (3, dict(W=64, H=321)),
}


@pytest.mark.parametrize("case", list(CASES))
def test_upscaled_tiles_match_single_process(case, emu_lib):
    world_size, cfg = CASES[case]
    _run(world_size, cfg)


@pytest.mark.parametrize("up", [(80, 800), None], ids=["upsampled", "native"])
def test_upscaled_tiles_under_a_moving_camera(up, emu_lib):
    """the camera rises by about a quarter of a render row per frame: history is read away from where it was written, within the motion bound"""
    _run(2, dict(W=64, H=640, up=up, move=True))


@pytest.mark.parametrize("streaming", [False, True], ids=["blocking", "streaming"])
def test_upscaled_tiles_with_host_inputs_and_result(streaming, emu_lib):
    """host G-buffer in, each rank uploads its full-res rows; host_result out, each rank writes exactly its result rows"""
    _run(2, dict(W=64, H=640, up=(80, 800), host_inputs=True, streaming=streaming))


def _worker_ircache(rank, world_size, port, ret):
    sys.path.insert(0, ROOT); sys.path.insert(0, HERE)
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port); os.environ["KJB_EMU_THREADS"] = "2"
    dist.init_process_group("gloo", rank=rank, world_size=world_size)
    from kajiya_b200._abi import KjbLib
    from kajiya_b200 import scenes
    import parity
    lib = KjbLib(os.path.join(HERE, "emu", "_build", "libkjb_emu.so"))
    scene, view = scenes.cornell_box()
    Wi, Hi, frames = 48, 768, 8
    kw = dict(enable_ircache=True, enable_taa=True, spatial_reuse_pass_count=1, upscale=(72, 1152))
    tiled = parity.make_world(lib, scene, Wi, Hi, tile=(rank, world_size), **kw)
    tiled.comm_set_callback(_gloo_allgather(world_size, [0]), rank, world_size)
    full = parity.make_world(lib, scene, Wi, Hi, **kw)
    for _ in range(frames):
        tiled.render_frame(**view); full.render_frame(**view)
    y0, y1 = tiled.result_rows()
    a = tiled.image("taa.this_frame_out")[y0:y1, :, :3].astype(np.float64); b = full.image("taa.this_frame_out")[y0:y1, :, :3].astype(np.float64)
    live = int(tiled.image("ircache.meta_buf").ravel()[3]), int(full.image("ircache.meta_buf").ravel()[3])
    ret[rank] = (bool(np.isfinite(a).all()), float(a.mean()), float(b.mean()), float(np.sqrt(((a - b) ** 2).mean())), live)
    dist.destroy_process_group()


def test_upscaled_tiles_with_replicated_irradiance_cache(emu_lib):
    """cache on, 2 ranks, 1.5x upsampling: statistical, with the thresholds of the native-resolution cache test (band mean within 10 %, RMS below
    25 % of the mean, every replica within 5 % of the single cache's live entries)"""
    ret = mp.Manager().dict()
    mp.spawn(_worker_ircache, args=(2, _free_port(), ret), nprocs=2, join=True)
    for rank in range(2):
        finite, ma, mb, rms, (la, lb) = ret[rank]
        print(f"rank {rank}: band mean {ma:.4f} vs {mb:.4f}, rms {rms:.4f}, live entries {la} vs {lb}")
        assert finite and mb > 0
        assert abs(ma - mb) <= 0.10 * mb and rms <= 0.25 * mb, (rank, ma, mb, rms)
        assert 0.95 * lb <= la <= 1.05 * lb, (rank, la, lb)


def test_result_rows_partition_the_output(emu_lib):
    """kjb_world_result_rows over a sweep of render heights (odd ones too), output heights (integer and non-integer ratios) and rank counts:
    the ranks' rows tile [0, OH) without gap or overlap, and without upsampling they are the full-res rows of the band"""
    from kajiya_b200.world import World
    for h in (1, 2, 7, 64, 321, 640, 1080, 1441):
        for oh in sorted({h, h + 1, (3 * h + 1) // 2, 2 * h, (5 * h) // 4, 3 * h}):
            for n in (1, 2, 3, 4, 5, 8):
                if n > (h + 1) // 2:
                    continue
                rows = []
                for r in range(n):
                    w = World(emu_lib, 8, h, enable_taa=True, upscale=(8, oh), tile=(r, n))
                    rows.append(w.result_rows()); w.close()
                assert rows[0][0] == 0 and rows[-1][1] == oh, (h, oh, n, rows)
                assert all(rows[i][1] == rows[i + 1][0] and rows[i][0] <= rows[i][1] for i in range(n - 1)), (h, oh, n, rows)
                if oh == h:
                    assert rows == [_band_rows(h, r, n)[1] for r in range(n)], (h, n, rows)
    w = World(emu_lib, 8, 9, enable_taa=True, upscale=(8, 20)); assert w.result_rows() == (0, 20); w.close()
    w = World(emu_lib, 8, 9, upscale=(8, 20), tile=(1, 2)); assert w.result_rows() == _band_rows(9, 1, 2)[1]; w.close()   # no TAA: the render-res result


# ---------------------------------------------------------------------------------------------------------------- GPU
def _gpu_worker(rank, world_size, port, transport, W, H, up, ret):
    sys.path.insert(0, ROOT); sys.path.insert(0, HERE)
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    os.environ.pop("TORCHELASTIC_USE_AGENT_STORE", None)
    device = rank if transport == "nccl" else 0
    torch.cuda.set_device(device)
    if transport == "nccl":
        dist.init_process_group("nccl", rank=rank, world_size=world_size, device_id=torch.device("cuda", device))
    else:
        dist.init_process_group("gloo", rank=rank, world_size=world_size)
    import kajiya_b200
    from kajiya_b200 import scenes
    import parity
    lib = kajiya_b200.lib()
    scene, view = scenes.cornell_box()
    scene = parity.glossy(scene)
    kw = dict(enable_taa=True, enable_rtr=True, spatial_reuse_pass_count=2, upscale=up)
    tiled = parity.make_world(lib, scene, W, H, device=device, tile=(rank, world_size), **kw)
    calls = [0]
    if transport == "nccl":
        uid = [None]
        if rank == 0:
            buf = C.create_string_buffer(128); assert lib.dll.kjb_comm_nccl_unique_id(buf) == 0; uid[0] = buf.raw
        dist.broadcast_object_list(uid, src=0)
        tiled.comm_init_nccl(uid[0], rank, world_size)
    else:
        tiled.comm_set_callback(_gloo_allgather(world_size, calls, staged_world=tiled), rank, world_size)
    full = parity.make_world(lib, scene, W, H, device=device, **kw)
    for f in range(6):
        v = _view(view, f, False)
        tiled.render_frame(**v); full.render_frame(**v)
    ret[rank] = (_compare_bands(tiled, full, H, up[1], rank, world_size, _names(full, True)), calls[0])
    dist.destroy_process_group()


def _gpu_run(world_size, transport, W, H, up):
    ret = mp.Manager().dict()
    mp.spawn(_gpu_worker, args=(world_size, _free_port(), transport, W, H, up, ret), nprocs=world_size, join=True)
    for rank in range(world_size):
        bad, calls = ret[rank]
        assert not bad, f"rank {rank}: band differs from the single-GPU frame: {bad}"
        if transport == "gloo":
            assert calls == 2 * 6, "GI bands + history borders, once per frame each"


@pytest.mark.gpu
@pytest.mark.parametrize("world_size", [2, 3])
def test_gpu_upscaled_tiles_on_one_gpu_over_staged_callback(world_size):
    """2 / 3 rank processes share one H100: 640x360 -> 960x540, TAA + reflections; the callback transport stages every in-place gather"""
    _gpu_run(world_size, "gloo", 640, 360, (960, 540))


@pytest.mark.gpu
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")
def test_gpu_upscaled_tiles_over_nccl():
    _gpu_run(min(torch.cuda.device_count(), 8), "nccl", 1280, 720, (1920, 1080))
