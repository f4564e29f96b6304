"""Time one 60-keyframe ground-plane window (synth config 3) solved three ways: plain, sharded at world 1 over NCCL, and -- under
torchrun with N GPUs -- sharded at world N.  Reports per-solve time (median / p90), iterations, parity against the plain solve,
and the card's name and power limit read in the same run.

    python scripts/shard_ground_bench.py [--steps K] [--n-kf 60] [--loopback W]
    torchrun --nproc_per_node N scripts/shard_ground_bench.py          # world N, one GPU per rank

--loopback W also runs the window over the in-process exchange at world W on ONE GPU.  That run checks the cross-rank sums
(parity); its ranks share one device, so its time is not a multi-GPU time and is reported as `loopback_ms_not_a_speedup`.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from limo_b200 import capi, parallel, synth  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except Exception:  # noqa: BLE001
        return "unknown"


def stats(ts):
    ms = np.array(ts) * 1e3
    return {"median_ms": float(np.median(ms)), "p90_ms": float(np.percentile(ms, 90)), "n": len(ts)}


def parity(kf_pose, final_cost, ref):
    return {"max_translation_diff_m": float(np.linalg.norm(kf_pose[:, 4:] - ref.kf_pose[:, 4:], axis=1).max()),
            "final_cost_rel_diff": float(abs(final_cost - ref.solves[-1].final_cost) / abs(ref.solves[-1].final_cost))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--n-kf", type=int, default=60)
    ap.add_argument("--loopback", type=int, default=0)
    args = ap.parse_args()
    rank, local_rank, world = parallel.rank_info()
    import torch
    torch.cuda.set_device(local_rank)
    parallel.init("nccl", torch.device("cuda", local_rank))
    win = synth.make_window(3, n_kf=args.n_kf)
    h = capi.Handle(local_rank)
    opt = capi.default_options()
    out = {"workload": "config 3 ground-plane window: %d KF / %d LM / %d obs / %d ground points" % (win.n_kf, win.n_lm, win.n_obs, win.n_gp),
           "card": card(), "world": world}

    def timed(fn):
        for _ in range(args.warmup):
            fn()
        ts = []
        for _ in range(args.steps):
            parallel.barrier()
            t0 = time.perf_counter()
            fn()
            ts.append(time.perf_counter() - t0)
        return ts

    plain = {}

    def solve_plain():
        plain["r"] = h.solve_window(win, opt)

    # every rank solves the whole window on its own GPU: timed() meets the other ranks at a barrier per step, so all ranks must
    # make the same calls before the NCCL id is broadcast (rank 0's numbers are reported)
    plain_ts = timed(solve_plain)
    if rank == 0:
        out["plain"] = stats(plain_ts)
        out["plain"]["iterations"] = [s.num_iterations for s in plain["r"].solves]

    # sharded over NCCL at the launch's world size (1 without torchrun)
    sub, j0, j1 = parallel.shard_window(win, rank, world)
    idt = torch.zeros(capi.SHARD_ID_BYTES, dtype=torch.uint8, device="cuda")
    if rank == 0:
        idt.copy_(torch.frombuffer(bytearray(capi.shard_unique_id()), dtype=torch.uint8))
    if world > 1:
        import torch.distributed as dist
        dist.broadcast(idt, 0)
    comm = capi.ShardComm(h, rank, world, bytes(idt.cpu().numpy().tobytes()))
    batch = h.batch([sub])
    batch.set_shard(comm, j0, win.n_lm)
    ts = timed(lambda: batch.solve(opt))
    rs = batch.download(256)[0]
    rec = dict(stats(parallel.max_over_ranks(ts, device="cuda")), iterations=[s.num_iterations for s in rs.solves])
    if rank == 0:
        rec.update(parity(rs.kf_pose, rs.solves[-1].final_cost, plain["r"]))
        if world == 1:
            rec["bit_identical_to_plain"] = bool(np.array_equal(rs.kf_pose, plain["r"].kf_pose) and
                                                 np.array_equal(rs.kf_plane, plain["r"].kf_plane))
        else:
            rec["speedup_vs_plain"] = out["plain"]["median_ms"] / rec["median_ms"]
    out["sharded_nccl_world%d" % world] = rec
    batch.close()
    comm.close()

    if rank == 0 and args.loopback > 1:
        res, lts = parallel.solve_sharded_local(win, args.loopback, opt, repeats=args.warmup + args.steps)
        kf_pose, _, _, rej = parallel.merge_shards(res, win.n_lm)
        lrec = {"loopback_ms_not_a_speedup": stats(lts[args.warmup:]), "iterations": [s.num_iterations for s in res[0][0].solves],
                "rejections_equal": bool(np.array_equal(rej, plain["r"].lm_rejected[:win.n_lm]))}
        lrec.update(parity(kf_pose, res[0][0].solves[-1].final_cost, plain["r"]))
        out["loopback_world%d" % args.loopback] = lrec
    if rank == 0:
        print(json.dumps(out))
    h.close()
    parallel.finalize()


if __name__ == "__main__":
    main()
