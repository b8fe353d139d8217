#!/usr/bin/env python
"""A sliding landmark-sharded window: the per-frame cycle of a VIO session on a cfg-5 shaped window (20 keyframes,
4 cameras) dealt to `world` ranks.  Each step optimizes, marginalises the oldest frame (pose, speed/bias, its IMU term
and the landmarks whose track ends within the first three frames), removes them, re-fixes the first pose and adds the
next frame with its IMU term, its new landmarks and its observations, routed by slot owner (okvis_b200.sharding).

`Slide` drives the ranks one process holds: all of them (okb_shard_connect_local, tests and tools/bench_shard_marg.py),
one of them (this file run by torchrun, mailboxes over cudaIpc), or an unsharded window (world 1).  Run as a torchrun
rank, it slides --steps steps and rank 0 writes every step's summaries, priors and merged estimates to --out:

    torchrun --nproc-per-node 2 tools/shard_slide_worker.py --landmarks 2000 --steps 2 --out slide.npz
"""
import argparse
import dataclasses
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from okvis_b200 import abi, sharding, synthetic  # noqa: E402

P, SB = abi.BLOCK_POSE, abi.BLOCK_SPEED_BIAS
PRIOR_KEYS = ("n", "block_kind", "block_idx", "x0", "J", "e0", "H", "b0", "status")


def slide_problem(n_landmarks=2000, extra=3, K=20, seed=0):
    """(the generated window of K + extra frames, its first K frames).  Landmarks first seen after frame K-1 are empty
    slots in the first window; they are created when their frame arrives."""
    cfg = dataclasses.replace(synthetic.CONFIGS[5], n_frames=K + extra, n_landmarks=n_landmarks)
    full = synthetic.make_window(5, seed, cfg=cfg)
    first = np.full(len(full.landmarks), K + extra)
    np.minimum.at(first, full.obs["lm_idx"], full.obs["pose_idx"])
    lm = full.landmarks.copy()
    lm[first >= K] = 0.0
    w0 = dataclasses.replace(full, poses=np.ascontiguousarray(full.poses[:K]), speed_bias=np.ascontiguousarray(full.speed_bias[:K]),
                             landmarks=lm, obs=np.ascontiguousarray(full.obs[full.obs["pose_idx"] < K]),
                             imu_terms=np.ascontiguousarray(full.imu_terms[:K - 1]), name=full.name + "/first%d" % K)
    return full, w0, first


class Slide:
    """members: [(rank, Context)] this process drives, all on window slot 0; world 1 = an unsharded window."""

    def __init__(self, members, world, full, w0, first_seen, features=None):
        self.members, self.world, self.full, self.first_seen = members, world, full, first_seen
        self.K, self.L = len(w0.poses), len(w0.landmarks)
        self.w = w0                  # host mirror of the current window (global landmark slots; estimates not tracked)
        self.step = 0
        self.local = {}
        for r, c in members:
            sw, idx = sharding.shard_window(w0, r, world)
            self.local[r] = idx
            c.reserve(0, self.K, len(sw.landmarks), int(np.isin(full.obs["lm_idx"], idx).sum()), len(full.imu_samples) + 4096, 160)
            if features:                 # (feature slots, cameras, keypoints, descriptor bytes) of a replicated store
                c.reserve_features(0, *features)
            c.upload(0, sw)

    def optimize(self, iters):
        for _, c in self.members:        # pending edits of every rank applied before any rank's solver spins
            c.commit(0, 1)
        for _, c in self.members:        # every rank must be in flight together: launches first
            c.optimize_async(0, 1, max_iterations=iters)
        return [c.optimize_finish(0, 1)[0] for _, c in self.members]

    def parts(self):
        return [(self.local[r], c.download(0, dims=(self.K, self.K, len(self.local[r])))) for r, c in self.members]

    def job(self, est, select=None):
        """(make_marg_job keyword lists with global landmark slots, landmarks to remove) of this step: frame 0 and its
        speed/bias marginalised with IMU term 0 (and the speed/bias prior on the first step), poses 0..2 connected.
        select(window at `est`, candidates) picks the landmarks to linearise; the rest are removed without."""
        w = self.w
        L = len(w.landmarks)
        first, last = np.full(L, 1 << 30), np.full(L, -1)
        np.minimum.at(first, w.obs["lm_idx"], w.obs["pose_idx"])
        np.maximum.at(last, w.obs["lm_idx"], w.obs["pose_idx"])
        cand = np.nonzero((first == 0) & (last <= 2))[0].astype(np.uint32)
        we = dataclasses.replace(w, poses=est["poses"], speed_bias=est["speed_bias"], landmarks=est["landmarks"])
        lms = cand if select is None else np.asarray(select(we, cand), np.uint32)
        prev = [-1] * 5 if self.step == 0 else [0, 1, 2, -1, -1]
        kw = dict(block_kind=[P, SB, P, SB, P], block_idx=[0, 0, 1, 1, 2], block_prev=prev, block_marginalize=[1, 1, 0, 0, 0],
                  imu_terms=[0], sb_priors=[0] if len(w.sb_priors) else [], landmarks=lms)
        return kw, cand

    def marginalize(self, kw):
        for r, c in self.members:
            c.marginalize(0, sharding.shard_marg_job(r, self.world, **kw))

    def priors(self):
        return [c.download_marg(0) for _, c in self.members]

    def edit(self, op, *args):
        for r, c in self.members:
            a = sharding.route_edit(op, r, self.world, *args)
            if a is not None:
                getattr(c, op)(0, *a)

    def advance(self, cand, first_pose):
        """The bookkeeping half of the step, then the next frame of the generated window."""
        new, obs, pp = self.edits(cand, first_pose)
        self.follow(cand, new, obs, pp)

    def edits(self, cand, first_pose):
        """The resident edits of advance(); returns what follow() needs."""
        self.edit("remove_landmarks", cand)
        self.edit("remove_frame", 0, 0)
        pp = np.zeros(1, abi.pose_prior_dtype)
        pp["pose_idx"], pp["meas"] = 0, first_pose
        pp["sqrt_info"] = np.diag([1e7, 1e7, 1e7, 0, 0, 1e7]).reshape(-1)
        self.edit("set_priors", pp, np.zeros(0, abi.sb_prior_dtype))
        k = self.K + self.step                # frame of the generated window that arrives; it becomes position K-1
        shift = self.step + 1
        f = self.full
        t = f.imu_terms[k - 1].copy()
        lo, n = int(t["sample_offset"]), int(t["sample_count"])
        t["sample_offset"] = 0
        for key in ("pose0", "sb0", "pose1", "sb1"):
            t[key] -= shift
        self.edit("add_frame", f.poses[k], f.speed_bias[k], t, f.imu_samples[lo:lo + n])
        new = np.nonzero(self.first_seen == k)[0].astype(np.uint32)
        if len(new):
            self.edit("set_landmarks", new, f.landmarks[new])
        obs = f.obs[f.obs["pose_idx"] == k].copy()
        obs["pose_idx"] -= shift
        self.edit("add_observations", obs)
        return new, obs, pp

    def follow(self, cand, new, obs, pp):
        """The host mirror after edits()."""
        f = self.full
        w = self.w
        keep = (w.obs["pose_idx"] != 0) & ~np.isin(w.obs["lm_idx"], cand)
        o = w.obs[keep].copy()
        o["pose_idx"] -= 1
        lm = w.landmarks.copy()
        lm[cand] = 0.0
        lm[new] = f.landmarks[new]
        self.w = dataclasses.replace(w, obs=np.ascontiguousarray(np.concatenate([o, obs])), landmarks=lm,
                                     sb_priors=np.zeros(0, abi.sb_prior_dtype), pose_priors=pp)
        self.step += 1


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--landmarks", type=int, default=2000)
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--iterations", type=int, default=6)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import torch
    import torch.distributed as dist
    from okvis_b200 import capi
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import marg_reference as mr
    rank, world, local_rank = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local_rank)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
    full, w0, first_seen = slide_problem(a.landmarks, extra=a.steps)
    ctx = capi.Context(local_rank, 1)
    sharding.connect_shards(ctx, dist, torch.device("cuda", local_rank), rank, world, len(w0.poses))
    s = Slide([(rank, ctx)], world, full, w0, first_seen)
    dist.barrier()
    out = {}
    for step in range(a.steps):
        summ = s.optimize(a.iterations)[0]
        parts = [None] * world
        dist.all_gather_object(parts, s.parts()[0])          # every rank forms the same global job
        est = sharding.merge_shard_results(s.L, parts)
        kw, cand = s.job(est, select=mr.well_conditioned)
        s.marginalize(kw)
        prior = s.priors()[0]
        res = [None] * world
        dist.all_gather_object(res, dict(summary=summ, prior=prior, stats=ctx.shard_stats(0)))
        if rank == 0:
            out["summaries_%d" % step] = np.array([x["summary"] for x in res], dtype=object)
            out["faults_%d" % step] = np.array([x["stats"]["fault"] for x in res])
            for r, x in enumerate(res):
                for k in PRIOR_KEYS:
                    out["prior_%d_%d_%s" % (step, r, k)] = np.asarray(x["prior"][k])
            out["poses_%d" % step], out["sb_%d" % step] = est["poses"], est["speed_bias"]
            out["landmarks_%d" % step] = kw["landmarks"]
        s.advance(cand, est["poses"][1])
    if rank == 0 and a.out:
        np.savez(a.out, **out)
    ctx.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
