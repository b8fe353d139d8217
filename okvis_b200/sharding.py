"""Multi-GPU plumbing for the hot path.  Keyframe windows are independent (no shared state between
okvis::Estimator instances, SURVEY.md 8e), so the path shards by window with NO data-path collective:
window w runs on rank w mod world.  torch.distributed is used only to (a) agree on the partition and
(b) reduce the measurement (max time over ranks, sums of counters) -- works with nccl and gloo alike.
"""
import numpy as np


def shard_indices(n_items, world, rank):
    """Round-robin ownership: item i belongs to rank i % world (SURVEY.md 8e: window w -> GPU w mod n)."""
    return list(range(rank, n_items, world))


def reduce_measurement(dist, device, elapsed_ms, counters):
    """Returns (max elapsed over ranks, counters summed over ranks).  `dist` may be None (single rank)."""
    import torch
    t = torch.tensor(list(elapsed_ms), dtype=torch.float64, device=device)
    c = torch.tensor([float(x) for x in counters], dtype=torch.float64, device=device)
    if dist is not None and dist.is_initialized() and dist.get_world_size() > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        dist.all_reduce(c, op=dist.ReduceOp.SUM)
    return [float(x) for x in t], [float(x) for x in c]


def gather_summaries(dist, summaries):
    """All ranks' per-window summaries, ordered by global window index (rank-major round robin undone)."""
    if dist is None or not dist.is_initialized() or dist.get_world_size() == 1:
        return list(summaries)
    world = dist.get_world_size()
    out = [None] * world
    dist.all_gather_object(out, list(summaries))
    n = sum(len(x) for x in out)
    merged = [None] * n
    for r, part in enumerate(out):
        for j, s in enumerate(part):
            merged[r + j * world] = s
    return merged


def shard_window(window, rank, world):
    """Landmark-block shard of ONE window (SURVEY.md 8e row 2, BASELINE.json configs[4]): rank r keeps the
    landmarks with lm_idx % world == r and their observations; poses, speed/bias, extrinsics, IMU terms and priors
    are replicated.  Returns (shard window, global landmark indices of the shard's landmarks)."""
    import dataclasses
    L = len(window.landmarks)
    mine = np.arange(rank, L, world)
    local = np.full(L, -1, np.int64)
    local[mine] = np.arange(len(mine))
    keep = local[window.obs["lm_idx"]] >= 0
    obs = window.obs[keep].copy()
    obs["lm_idx"] = local[obs["lm_idx"]].astype(np.uint32)
    w = dataclasses.replace(window, landmarks=np.ascontiguousarray(window.landmarks[mine]), obs=np.ascontiguousarray(obs),
                            name="%s/shard%d of %d" % (window.name, rank, world))
    return w, mine


def owned_slots(idx, rank, world):
    """(positions in `idx` of the global landmark slots rank `rank` holds, their local slots).  The rule shard_window
    deals by: global slot g lives on rank g % world at local slot g // world.  Slots are chosen by the caller and stable,
    so the rule holds while the window slides."""
    idx = np.asarray(idx, np.int64).reshape(-1)
    pos = np.nonzero(idx % world == rank)[0]
    return pos, (idx[pos] // world).astype(np.uint32)


def global_slots(local, rank, world):
    """Inverse of owned_slots: the global slots of rank `rank`'s local slots."""
    return np.asarray(local, np.int64) * world + rank


def shard_marg_job(rank, world, block_kind, block_idx, block_prev, block_marginalize, imu_terms=(), sb_priors=(), landmarks=()):
    """Rank `rank`'s okb_marg_job for a landmark-sharded window: the same dense part on every rank (blocks, IMU terms,
    speed/bias priors), and of the global `landmarks` only those the rank holds, as local slots.  A rank that holds none
    gets n_landmarks = 0 and must still call okb_window_marginalize*."""
    from . import abi
    _, local = owned_slots(landmarks, rank, world)
    return abi.make_marg_job(block_kind, block_idx, block_prev, block_marginalize, imu_terms=imu_terms, sb_priors=sb_priors,
                             landmarks=local)


# Resident edits of a sliding landmark-sharded window: landmark edits go to the slot's owner, the dense edits (frames,
# states, priors, speed/bias removal) to every rank unchanged.  The feature store is replicated and names global
# landmark slots, so its edits also go to every rank unchanged; a landmark's initialised flag is landmark state and goes
# to its owner.  Any other op is refused: its arguments may hold landmark slots that would be read as local ones.
LANDMARK_EDITS = ("set_landmarks", "remove_landmarks", "add_observations", "remove_observations", "set_landmark_initialized")
DENSE_EDITS = ("add_frame", "remove_frame", "set_states", "set_priors", "remove_speed_bias")
STORE_EDITS = ("reserve_features", "set_features", "set_feature_landmarks", "clear_features")


def route_edit(op, rank, world, *args):
    """Arguments of Context.<op>(win, *args) for rank `rank`, or None when the rank has nothing to do.  `args` are the
    unsharded window's (global landmark slots)."""
    if op in DENSE_EDITS or op in STORE_EDITS:
        return args
    if op == "remove_observations":
        (keys,) = args
        k = np.asarray(keys, np.int64).reshape(-1, 3)          # (pose_idx, lm_idx, cam_idx)
        pos, local = owned_slots(k[:, 1], rank, world)
        if not len(pos):
            return None
        mine = k[pos].copy()
        mine[:, 1] = local
        return (mine,)
    if op == "set_landmarks":
        idx, xyzw = args
        pos, local = owned_slots(idx, rank, world)
        return (local, np.ascontiguousarray(np.asarray(xyzw, np.float64).reshape(-1, 4)[pos])) if len(pos) else None
    if op == "remove_landmarks":
        (idx,) = args
        _, local = owned_slots(idx, rank, world)
        return (local,) if len(local) else None
    if op == "set_landmark_initialized":
        idx, flags = args
        pos, local = owned_slots(idx, rank, world)
        return (local, np.asarray(flags).reshape(-1)[pos]) if len(pos) else None
    if op == "add_observations":
        (obs,) = args
        pos, local = owned_slots(obs["lm_idx"], rank, world)
        if not len(pos):
            return None
        mine = obs[pos].copy()
        mine["lm_idx"] = local
        return (mine,)
    raise ValueError("route_edit: %r is not a resident edit of a sharded window" % (op,))


def merge_shard_results(n_landmarks, parts):
    """parts: list over ranks of (global landmark indices, download dict).  Dense blocks are identical on all ranks."""
    out = dict(poses=parts[0][1]["poses"], speed_bias=parts[0][1]["speed_bias"],
               landmarks=np.zeros((n_landmarks, 4)), quality=np.zeros(n_landmarks))
    for idx, d in parts:
        out["landmarks"][idx] = d["landmarks"]
        if d.get("quality") is not None:
            out["quality"][idx] = d["quality"]
    return out


def connect_shards(ctx, dist, device, rank, world, max_frames, max_landmarks=0):
    """Multi-process mailbox set-up of a landmark-sharded context: export this rank's cudaIpc handle, all-gather the
    handles with torch.distributed (64 bytes per rank; plumbing only), map the peers.  max_landmarks > 0: the global
    landmark slots of the frontend's landmark replica."""
    import torch
    handle = torch.from_numpy(ctx.shard_export(rank, world, max_frames, max_landmarks)).to(device)
    gathered = [torch.zeros_like(handle) for _ in range(world)]
    dist.all_gather(gathered, handle)
    ctx.shard_connect(np.stack([g.cpu().numpy() for g in gathered]))
