"""One process per GPU: the host-side plumbing of the N > 1 runs (bench.py, the sharded large-window solve).

Windows are independent optimisation problems, so the data path of the headline workload has NO collective: every rank
owns its own batch of windows (weak scaling) and torch.distributed is used for the barrier around the timed region, the
max-over-ranks of the device times and the window count only.  `shard_window` is the partition used when ONE large
window (BASELINE config 5) is split by landmark blocks: every rank keeps all keyframes and a contiguous, observation-
balanced range of landmarks; what has to be exchanged then is the reduced pose system (see DESIGN.md section 6).

Everything here works on CPU tensors with the gloo backend as well (tests/test_parallel_gloo.py, world_size 2).
"""
import os

import numpy as np


def rank_info():
    """(rank, local_rank, world_size) from the torchrun environment; (0, 0, 1) when launched plainly"""
    return (int(os.environ.get("RANK", "0")), int(os.environ.get("LOCAL_RANK", "0")),
            int(os.environ.get("WORLD_SIZE", "1")))


def init(backend, device=None):
    """join the process group when WORLD_SIZE > 1 (MASTER_ADDR / MASTER_PORT from the environment)"""
    import torch.distributed as dist
    _, _, world = rank_info()
    if world > 1 and not dist.is_initialized():
        kw = {"device_id": device} if (device is not None and backend == "nccl") else {}
        dist.init_process_group(backend, **kw)
    return world > 1


def finalize():
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized():
        dist.destroy_process_group()


def barrier(cuda=False):
    import torch
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized():
        dist.barrier()
    if cuda:
        torch.cuda.synchronize()


def max_over_ranks(values, device="cpu"):
    """element-wise maximum of a list of floats over all ranks (device times: the slowest rank defines the step)"""
    import torch
    import torch.distributed as dist
    t = torch.tensor(list(values), dtype=torch.float64, device=device)
    if dist.is_available() and dist.is_initialized():
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return [float(x) for x in t.cpu()]


def sum_over_ranks(values, device="cpu"):
    import torch
    import torch.distributed as dist
    t = torch.tensor(list(values), dtype=torch.float64, device=device)
    if dist.is_available() and dist.is_initialized():
        dist.all_reduce(t, op=dist.ReduceOp.SUM)
    return [float(x) for x in t.cpu()]


def window_seeds(n_distinct, rank):
    """seeds of the synthetic windows of one rank: disjoint between ranks, reproducible"""
    return [0xBA5E0000 + 1000 * rank + i for i in range(n_distinct)]


def windows_for_rank(n_distinct, rank, config=2):
    from limo_b200 import synth
    return [synth.make_window(config, seed=s) for s in window_seeds(n_distinct, rank)]


def landmark_ranges(lm_obs_ptr, world):
    """contiguous landmark ranges [j0, j1) per rank with (nearly) equal observation counts"""
    ptr = np.asarray(lm_obs_ptr, dtype=np.int64)
    n_lm, n_obs = len(ptr) - 1, int(ptr[-1])
    cuts = [0]
    for r in range(1, world):
        cuts.append(int(np.searchsorted(ptr, n_obs * r / world, side="left")))
    cuts.append(n_lm)
    cuts = np.maximum.accumulate(np.clip(cuts, 0, n_lm))
    return [(int(cuts[r]), int(cuts[r + 1])) for r in range(world)]


def shard_window(win, rank, world):
    """the part of `win` owned by `rank`: all keyframes / cameras / priors, landmarks [j0, j1) with their observations
    and ground-plane residuals.  Returns (sub_window, j0, j1)."""
    from limo_b200.capi_types import Window
    j0, j1 = landmark_ranges(win.lm_obs_ptr, world)[rank]
    o0, o1 = int(win.lm_obs_ptr[j0]), int(win.lm_obs_ptr[j1])
    gp = {}
    if win.n_gp:
        keep = (win.gp_lm >= j0) & (win.gp_lm < j1)
        gp = dict(gp_lm=win.gp_lm[keep] - j0, gp_kf=win.gp_kf[keep], gp_weight=win.gp_weight[keep])
    sub = Window(
        win.kf_pose, win.kf_fixed, win.cam_intr, win.cam_pose, win.lm_pos[j0:j1], win.lm_weight[j0:j1],
        win.lm_obs_ptr[j0:j1 + 1] - o0, win.obs_kf[o0:o1], win.obs_u[o0:o1], win.obs_v[o0:o1], win.obs_d[o0:o1],
        obs_cam=None if win.obs_cam is None else win.obs_cam[o0:o1], kf_plane=win.kf_plane,
        scale_kf0=win.scale_kf0, scale_kf1=win.scale_kf1, scale_weight=win.scale_weight, scale_value=win.scale_value,
        plane_reg_weight=win.plane_reg_weight, plane_dist_fixed=win.plane_dist_fixed,
        landmarks_fixed=win.landmarks_fixed, speed_kf=win.speed_kf, speed_weight=win.speed_weight,
        speed_dt=win.speed_dt, speed_v_before=win.speed_v_before, speed_T_origin_before=win.speed_T_origin_before, **gp)
    return sub, j0, j1


def solve_sharded_local(win, world, opt=None, handles=None, iterations_capacity=256, repeats=1):
    """solve `win` sharded over `world` ranks of THIS process on one GPU (capi.ShardComm.local): rank r's shard is solved by its
    own handle from its own thread, as each rank is its own process with NCCL.  The exchanged sums are those of a `world`-GPU
    run; the time is not (the ranks share one device).  Returns [(result, j0, j1)] per rank; `repeats` > 1 solves again
    (every solve of a batch starts from the uploaded state) and also returns the wall time of each solve in seconds."""
    import threading
    import time
    from limo_b200 import capi
    own = handles is None
    handles = [capi.Handle(0) for _ in range(world)] if own else list(handles)
    parts = [shard_window(win, r, world) for r in range(world)]
    comms = capi.ShardComm.local(handles)
    batches = [handles[r].batch([parts[r][0]]) for r in range(world)]
    out, errors, times = [None] * world, [None] * world, [[] for _ in range(world)]

    def run(r):
        try:
            batches[r].set_shard(comms[r], parts[r][1], win.n_lm)
            for _ in range(repeats):
                t0 = time.perf_counter()
                batches[r].solve(opt or capi.default_options())
                times[r].append(time.perf_counter() - t0)
            out[r] = batches[r].download(iterations_capacity)[0]
        except Exception as e:  # noqa: BLE001 -- re-raised below, after every thread has ended
            errors[r] = e

    threads = [threading.Thread(target=run, args=(r,)) for r in range(world)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    for b in batches:
        b.close()
    for c in comms:
        c.close()
    if own:
        for h in handles:
            h.close()
    for e in errors:
        if e is not None:
            raise e
    res = [(out[r], parts[r][1], parts[r][2]) for r in range(world)]
    return (res, [max(ts) for ts in zip(*times)]) if repeats > 1 else res


def merge_shards(results, n_lm):
    """(kf_pose, kf_plane, lm_pos, lm_rejected) of the whole window from the ranks' results (poses / planes of rank 0)"""
    lm_pos = np.zeros((n_lm, 3))
    rej = np.zeros(n_lm, dtype=np.uint8)
    for r, j0, j1 in results:
        lm_pos[j0:j1] = r.lm_pos[:j1 - j0]
        rej[j0:j1] = r.lm_rejected[:j1 - j0]
    return results[0][0].kf_pose, results[0][0].kf_plane, lm_pos, rej
