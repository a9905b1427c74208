"""Strong scaling of the tile-sharded upsampled frame: BASELINE configs[4]'s "full GI + temporal upsample" — the 2 M-triangle ruins rendered at
2560x1440 and upsampled to 3840x2160 by the TAA, with rtdgi (2 spatial passes) + irradiance cache + reflections + TAA — sharded over N ranks.

    torchrun --nproc_per_node 8 tools/tile_scaling.py [--frames 32] [--warmup 8]

Every N = 1, 2, 4, ... up to the launched rank count is timed in turn (ranks [0, N) render, the others wait; each group gets its own NCCL
communicator).  Prints one JSON line per N on rank 0: ms/frame (device timer events around K frames on every rank, after a barrier; the frame's G-buffer
replayed from HBM as bench.py does), the GPU name and its power limit, and for N > 1 each rank's parity: its result rows against the same rows
of an untiled render on the same GPU (statistical: every rank keeps a replica of the irradiance cache, DESIGN §7).  bench.py's configs[4] adds
SSAO and the lit composite, which do not shard."""
import argparse, ctypes as C, json, os, subprocess, sys
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
W, H, UP = 2560, 1440, (3840, 2160)
FLAGS = dict(enable_ircache=True, enable_rtr=True, enable_taa=True, spatial_reuse_pass_count=2, upscale=UP)


def gpu_name_and_power_limit(index):
    try:
        out = subprocess.run(["nvidia-smi", f"--id={index}", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        name, limit = [x.strip() for x in out.strip().split(",")][:2]
        return name, limit
    except Exception:
        import torch
        return torch.cuda.get_device_name(index), "unknown"


def make_world(lib, scene, device, tile):
    from kajiya_b200 import scenes
    from kajiya_b200.world import World
    w = World(lib, W, H, device=device, tile=tile, **FLAGS)
    scenes.populate(w, scene)
    return w


def run_n(n, rank, local_rank, lib, scene, view, args, torch, dist):
    """time N = n on ranks [0, n); returns (ms/frame on rank 0, [parity dict per rank]) on rank 0"""
    group = dist.new_group(list(range(n)))
    result = None
    if rank < n:
        w = make_world(lib, scene, local_rank, (rank, n) if n > 1 else None)
        if n > 1:
            uid = [None]
            if rank == 0:
                buf = C.create_string_buffer(128); assert lib.dll.kjb_comm_nccl_unique_id(buf) == 0; uid[0] = buf.raw
            dist.broadcast_object_list(uid, src=0, group=group)
            w.comm_init_nccl(uid[0], rank, n)
        w.render_frame(capture_slot=1, **view)
        for _ in range(args.warmup):
            w.render_frame(replay_slot=1, **view)
        w.sync(); dist.barrier(group=group)
        w.timer_record(0)
        for _ in range(args.frames):
            w.render_frame(replay_slot=1, **view)
        w.timer_record(1); w.sync()
        ms = w.timer_elapsed_ms(0, 1) / args.frames
        parity = None
        if n > 1:   # the same frame sequence untiled on this GPU: this rank's result rows against the same rows
            w.close()
            w = make_world(lib, scene, local_rank, (rank, n))
            full = make_world(lib, scene, local_rank, None)
            uid2 = [None]
            if rank == 0:
                buf = C.create_string_buffer(128); assert lib.dll.kjb_comm_nccl_unique_id(buf) == 0; uid2[0] = buf.raw
            dist.broadcast_object_list(uid2, src=0, group=group)
            w.comm_init_nccl(uid2[0], rank, n)
            for _ in range(args.parity_frames):
                w.render_frame(**view); full.render_frame(**view)
            y0, y1 = w.result_rows()
            a = w.image("taa.this_frame_out")[y0:y1, :, :3]; b = full.image("taa.this_frame_out")[y0:y1, :, :3]
            fa, fb = a.astype(np.float64), b.astype(np.float64)
            parity = dict(rank=rank, rows=[y0, y1], bit_identical_fraction=float((a.view(np.uint16) == b.view(np.uint16)).all(-1).mean()),
                          mean=[float(fa.mean()), float(fb.mean())], rms_over_mean=float(np.sqrt(((fa - fb) ** 2).mean()) / max(fb.mean(), 1e-12)))
            full.close()
        w.close()
        gathered = [None] * n
        dist.all_gather_object(gathered, (ms, parity), group=group)
        result = gathered
    dist.barrier()
    return result


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=32)
    ap.add_argument("--warmup", type=int, default=8)
    ap.add_argument("--parity-frames", type=int, default=8)
    args = ap.parse_args()
    import torch, torch.distributed as dist
    rank, world_size, local_rank = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local_rank)
    if "MASTER_ADDR" not in os.environ:
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT="29533")
    dist.init_process_group("nccl", rank=rank, world_size=world_size, device_id=torch.device("cuda", local_rank))
    import kajiya_b200
    from kajiya_b200 import scenes
    lib = kajiya_b200.lib()
    scene, view = scenes.ruins()
    name, limit = gpu_name_and_power_limit(local_rank)
    n = 1
    while n <= world_size:
        res = run_n(n, rank, local_rank, lib, scene, view, args, torch, dist)
        if rank == 0:
            print(json.dumps(dict(ranks=n, ms_per_frame=round(res[0][0], 3), per_rank_ms=[round(r[0], 3) for r in res], gpu=name, power_limit=limit,
                                  resolution=[W, H], output_resolution=list(UP), features="rtdgi(2 spatial)+ircache+rtr+taa",
                                  parity=[r[1] for r in res if r[1]] or "untiled")), flush=True)
        n *= 2
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
