"""Multi-GPU plumbing: one process per GPU (torchrun), candidates dealt to the ranks, ONE all-gather
of the per-candidate score blocks -- the counterpart of ``RDD.collect()`` (reference
base_search.py:89).  The data path has no other collective: tasks are independent (reference
base_search.py:56-62 runs one Spark partition per task) and the dataset is replicated on every
GPU exactly as the reference replicates it with ``sc.broadcast`` (base_search.py:63-65).
"""
import numpy as np


def _td():
    try:
        import torch.distributed as td
    except Exception:  # pragma: no cover
        return None
    return td if td.is_available() and td.is_initialized() else None


def rank_world():
    td = _td()
    return (td.get_rank(), td.get_world_size()) if td else (0, 1)


def local_devices():
    """GPUs one plain ``fit()`` drives when torch.distributed is NOT initialised: every visible sm_90 device by default
    (B200GS_DEVICES = "all" | a count | a comma-separated list of indices; "1" keeps the search on one GPU)."""
    import os
    from .engine import device_count
    spec = os.environ.get("B200GS_DEVICES", "all").strip().lower()
    if int(os.environ.get("WORLD_SIZE", "1")) > 1:      # a torchrun rank whose process group is not up: its own GPU only
        return [int(os.environ.get("LOCAL_RANK", "0"))]
    n = device_count()
    if n <= 0:
        return [0]                                      # Engine(0) then fails loudly: there is no CPU fallback
    if spec in ("", "all"):
        return list(range(n))
    if "," in spec:
        return [int(x) for x in spec.split(",") if x.strip() != ""]
    return list(range(max(1, min(n, int(spec)))))


def assign_candidates(n_cand, world, costs=None):
    """Candidate indices of every rank (list of ascending lists).  Without costs: strided, c -> c mod world.  With a
    predicted cost per candidate: sorted by cost and dealt in snake order (0..W-1, W-1..0, ...), so that every rank
    gets the same share of the expensive candidates -- the makespan of a search is set by its longest fits.
    Deterministic and identical on every rank; each rank holds ceil or floor of n_cand / world candidates."""
    if costs is None or world == 1:
        return [list(range(r, n_cand, world)) for r in range(world)]
    costs = np.asarray(costs, dtype=np.float64)
    if costs.shape != (n_cand,) or not np.all(np.isfinite(costs)):
        return [list(range(r, n_cand, world)) for r in range(world)]
    order = np.argsort(-costs, kind="stable")
    parts = [[] for _ in range(world)]
    for pos, c in enumerate(order):
        lap, k = divmod(pos, world)
        parts[k if lap % 2 == 0 else world - 1 - k].append(int(c))
    return [sorted(p) for p in parts]


def assign_groups(n_cand, world, costs, keys, max_imbalance=1.08):
    """Experimental (B200GS_DEAL=groups): deal whole affinity groups (for SVC: all candidates sharing one gamma, which
    share one kernel matrix and one decision-value pass) instead of single candidates.  Groups are sorted by total
    predicted cost and dealt in snake order; if there are fewer than 2*world groups or the predicted loads differ by
    more than ``max_imbalance`` the cost-balanced candidate dealing is used instead."""
    costs = np.asarray(costs, dtype=np.float64)
    groups = {}
    for c, k in enumerate(keys):
        groups.setdefault(k, []).append(c)
    if len(groups) < 2 * world:
        return assign_candidates(n_cand, world, costs)
    order = sorted(groups, key=lambda k: (-costs[groups[k]].sum(), str(k)))
    parts = [[] for _ in range(world)]
    for pos, k in enumerate(order):
        lap, r = divmod(pos, world)
        parts[r if lap % 2 == 0 else world - 1 - r].extend(groups[k])
    load = [costs[p].sum() for p in parts]
    if min(load) <= 0 or max(load) > max_imbalance * min(load):
        return assign_candidates(n_cand, world, costs)
    return [sorted(p) for p in parts]


def assign_affinity(n_cand, world, costs, keys, group_cost):
    """Cost dealing that keeps affinity groups together (for SVC: candidates sharing a gamma share one kernel matrix and one
    float64 decision-value pass per GPU -- `group_cost` in the units of `costs`).  Two tiers:
      1. the 2*world most expensive candidates (the fits that set the makespan) are dealt one by one in snake order, exactly
         as assign_candidates does: every rank gets the same share of the critical path;
      2. the others travel in half-groups (the candidates of one group, split in two by cost): longest half-group first onto
         the rank whose load after taking it -- plus group_cost if the rank does not hold that group yet -- is smallest.
    Deterministic and identical on every rank; ranks may end with different candidate counts (the gather pads)."""
    costs = np.asarray(costs, dtype=np.float64)
    order = np.argsort(-costs, kind="stable")
    n_heavy = min(n_cand, 2 * world)
    parts = [[] for _ in range(world)]
    load = np.zeros(world)
    have = [set() for _ in range(world)]
    for pos, c in enumerate(order[:n_heavy]):
        lap, k = divmod(pos, world)
        r = k if lap % 2 == 0 else world - 1 - k
        c = int(c)
        load[r] += costs[c] + (0.0 if keys[c] in have[r] else group_cost)
        parts[r].append(c); have[r].add(keys[c])
    groups = {}
    for c in order[n_heavy:]:
        groups.setdefault(keys[int(c)], []).append(int(c))                 # descending cost inside a group
    units = []
    for k, members in groups.items():
        half = -(-len(members) // 2)
        for piece in (members[:half], members[half:]):
            if piece:
                units.append((float(costs[piece].sum()), str(k), k, piece))
    units.sort(key=lambda u: (-u[0], u[1]))
    for ucost, _, k, piece in units:
        t = [load[r] + ucost + (0.0 if k in have[r] else group_cost) for r in range(world)]
        r = int(np.argmin(t))
        load[r] = t[r]; parts[r].extend(piece); have[r].add(k)
    return [sorted(p) for p in parts]


def assign_for_plan(plan, n_cand, world):
    """The dealing used by the search driver and by bench.py: by predicted cost (default) or, with B200GS_DEAL=groups,
    by affinity group where that still balances."""
    import os
    if world == 1:
        return assign_candidates(n_cand, 1)
    costs = plan.costs() if hasattr(plan, "costs") else None
    mode = os.environ.get("B200GS_DEAL", "cost")
    if costs is not None and mode in ("groups", "affinity"):
        keys = plan.affinity() if hasattr(plan, "affinity") else None
        if keys is not None and mode == "groups":
            return assign_groups(n_cand, world, costs, keys)
        if keys is not None:
            return assign_affinity(n_cand, world, costs, keys, getattr(plan, "group_cost", 0.0))
    return assign_candidates(n_cand, world, costs)


def merge_candidates(locs, parts, n_cand, n_splits):
    """Host-side merge of per-device score blocks (in-process multi-GPU path): same result layout as allgather_candidates."""
    keys = ["test", "train", "fit_time", "score_time"]
    out = {}
    for k in keys:
        if all(l is None or l.get(k) is None for l in locs):
            out[k] = None
            continue
        full = np.full((n_cand, n_splits), np.nan)
        for l, idx in zip(locs, parts):
            if l is not None and len(idx):
                full[idx] = l[k]
        out[k] = full
    return out


def merge_profiles(profs):
    """Device profiles of concurrent per-GPU calls: times are the slowest device's, counters add up."""
    out = {}
    for p in profs:
        for k, v in p.items():
            if k.startswith("ms_"):
                out[k] = max(out.get(k, 0.0), v)
            else:
                out[k] = out.get(k, 0) + v
    return out


def broadcast_plan(obj):
    """The reference enumerates candidates and CV splits ONCE, on the driver (base_search.py:34-61), and ships them to the
    executors.  With one process per GPU every rank would otherwise draw its own: RandomizedSearchCV(random_state=None)
    or a shuffling splitter reseeded per process (base_search.py:39-41) give each rank different candidates / folds,
    and the all-gather would then merge score blocks of different parameter sets.  Rank 0's objects win."""
    td = _td()
    if td is None or td.get_world_size() == 1:
        return obj
    box = [obj if td.get_rank() == 0 else None]
    if td.get_backend() == "nccl":
        import torch
        import os
        td.broadcast_object_list(box, src=0, device=torch.device("cuda", int(os.environ.get("LOCAL_RANK", "0"))))
    else:
        td.broadcast_object_list(box, src=0)
    return box[0]


def allgather_candidates(local, my, n_cand, n_splits, world, parts=None, device=None):
    """local: dict of [len(my), n_splits] arrays (test, train|None, fit_time, score_time) for the
    candidates ``my`` of this rank.  Returns the same dict for all n_cand candidates, identical on
    every rank and independent of the number of ranks.  ``parts`` = assign_candidates(...) (default: strided)."""
    keys = ["test", "train", "fit_time", "score_time"]
    if world == 1:
        return {k: local.get(k) for k in keys}
    import torch
    td = _td()
    if parts is None:
        parts = assign_candidates(n_cand, world)
    per = max(len(p) for p in parts)                         # pad to equal counts
    buf = np.full((per, n_splits, len(keys)), np.nan)
    for j, k in enumerate(keys):
        if local.get(k) is not None and len(my):
            buf[:len(my), :, j] = local[k]
    # the gather buffer lives on the engine's GPU (LOCAL_RANK), not on whatever torch's current device happens to be
    if td.get_backend() == "nccl":
        dev = torch.device("cuda", torch.cuda.current_device() if device is None else int(device))
    else:
        dev = torch.device("cpu")
    t = torch.from_numpy(buf).to(dev)
    gathered = torch.empty((world * per,) + tuple(t.shape[1:]), dtype=t.dtype, device=dev)
    td.all_gather_into_tensor(gathered, t.contiguous())
    g = gathered.cpu().numpy().reshape((world, per) + tuple(t.shape[1:]))
    out = {}
    for j, k in enumerate(keys):
        if local.get(k) is None and k == "train":
            out[k] = None
            continue
        full = np.empty((n_cand, n_splits))
        for r in range(world):
            idx = parts[r]
            full[idx] = g[r, :len(idx), :, j]
        out[k] = full
    return out
