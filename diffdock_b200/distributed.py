"""Multi-GPU driver (SURVEY.md section 8(e)): poses / complexes are independent units, so each rank samples a contiguous
block with no collective inside the step loop; ONE all_gather of the final ligand coordinates at the end
(NCCL over NVLink on GPUs; gloo in the CPU tests), preceded for packed sampling by one small status exchange.  The
reference samples the N poses of a complex in one process (inference.py:236-262: N deep copies ->
utils/sampling.py:sampling); its only data parallelism is PyG DataParallel over complexes (utils/utils.py:279), so this
module has no reference counterpart to mirror."""
from __future__ import annotations

from typing import Callable, List, Sequence

import torch
import torch.distributed as dist


def _default_device(group):
    """Where a gather runs by default: the current CUDA device under NCCL, the CPU otherwise."""
    nccl = dist.is_initialized() and dist.get_backend(group) == 'nccl'
    return torch.device('cuda', torch.cuda.current_device()) if nccl else torch.device('cpu')


def shard_bounds(n_items: int, rank: int, world: int):
    """Contiguous, size-balanced block [lo, hi) of ``n_items`` for ``rank`` (first ``n_items % world`` ranks get one more)."""
    base, extra = divmod(n_items, world)
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


def all_gather_positions(local: torch.Tensor, n_total: int, group=None) -> torch.Tensor:
    """local [n_local, n_atoms, 3] on every rank -> [n_total, n_atoms, 3] on every rank (shards may differ by one pose)."""
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    n_max = (n_total + world - 1) // world
    pad = torch.zeros((n_max,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
    pad[:local.shape[0]] = local
    bufs = [torch.empty_like(pad) for _ in range(world)]
    dist.all_gather(bufs, pad, group=group)
    out = []
    for r in range(world):
        lo, hi = shard_bounds(n_total, r, world)
        out.append(bufs[r][:hi - lo])
    return torch.cat(out, 0)


def sample_sharded(data_list: Sequence, sampler: Callable[[List], List], group=None, device=None,
                   dtype=torch.float32) -> torch.Tensor:
    """Runs ``sampler(local_block)`` (e.g. a partial of diffdock_b200.sampling.sampling) on this rank's block of poses of
    one complex and returns the final coordinates of ALL poses, [len(data_list), n_atoms, 3], on every rank.
    ``device`` / ``dtype`` fix where the gathered tensor lives on EVERY rank (default: the current CUDA device under NCCL,
    the CPU otherwise): a rank whose block is empty (fewer poses than ranks) must still enter the collective with a
    buffer on the same kind of device and of the same dtype as its peers."""
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    if device is None:
        device = _default_device(group)
    lo, hi = shard_bounds(len(data_list), rank, world)
    block = list(data_list[lo:hi])
    done = sampler(block) if block else []
    n_atoms = data_list[0]['ligand'].pos.shape[0]
    if done:
        local = torch.stack([d['ligand'].pos for d in done]).to(device=device, dtype=dtype)
    else:
        local = torch.zeros((0, n_atoms, 3), device=device, dtype=dtype)
    if world == 1:
        return local
    return all_gather_positions(local, len(data_list), group)


# ---------------------------------------------------------------------------------------------------------------------
# Level-1 partitioning of SURVEY.md section 8(e): whole complexes over GPUs (inference.py:224 walks them one after another)
def assign_balanced(costs: Sequence[float], world: int) -> List[List[int]]:
    """Longest-processing-time-first assignment of items with the given costs (N_r * N_l * poses per complex) to ``world``
    ranks; deterministic (ties broken by index), every rank gets its items in ascending index order."""
    order = sorted(range(len(costs)), key=lambda i: (-float(costs[i]), i))
    load = [0.0] * world
    out: List[List[int]] = [[] for _ in range(world)]
    for i in order:
        r = min(range(world), key=lambda q: (load[q], q))
        out[r].append(i)
        load[r] += float(costs[i])
    return [sorted(v) for v in out]


def gather_ragged(local: Sequence[torch.Tensor], owner: Sequence[int], shapes: Sequence[Sequence[int]], group=None,
                  device=None, dtype=torch.float32) -> List[torch.Tensor]:
    """``local[j]`` = result of the j-th item this rank owns (items in ascending index order); ``owner[i]`` / ``shapes[i]`` are
    known on every rank.  ONE all_gather of a packed, padded buffer; returns all items, in index order, on every rank."""
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    if device is None:
        device = _default_device(group)
    numel = [int(torch.Size(sh).numel()) for sh in shapes]
    per_rank = [sum(numel[i] for i in range(len(owner)) if owner[i] == r) for r in range(world)]
    mine = [i for i in range(len(owner)) if owner[i] == rank]
    assert len(mine) == len(local), (len(mine), len(local))
    flat = torch.zeros(max(max(per_rank), 1), device=device, dtype=dtype)
    off = 0
    for i, t in zip(mine, local):
        assert tuple(t.shape) == tuple(shapes[i]), (tuple(t.shape), tuple(shapes[i]))
        flat[off:off + numel[i]] = t.reshape(-1).to(device=device, dtype=dtype)
        off += numel[i]
    if world == 1:
        bufs = [flat]
    else:
        bufs = [torch.empty_like(flat) for _ in range(world)]
        dist.all_gather(bufs, flat, group=group)
    offs = [0] * world
    out = []
    for i in range(len(owner)):
        r = owner[i]
        out.append(bufs[r][offs[r]:offs[r] + numel[i]].reshape(tuple(shapes[i])))
        offs[r] += numel[i]
    return out


def sample_complexes_sharded(n_complexes: int, costs: Sequence[float], shapes: Sequence[Sequence[int]],
                             sample_one: Callable[[int], torch.Tensor], group=None, device=None) -> List[torch.Tensor]:
    """Config-5-style job: ``n_complexes`` independent complexes, each sampled as ONE batch of all its poses by
    ``sample_one(i) -> [n_poses, n_atoms, 3]`` on the rank that owns it (so the batch a pose is scored in - which the default
    centre convolution depends on, models/cg_model.py:374 - never depends on the number of GPUs), then one collective
    returning every complex's final coordinates on every rank.  With ``rng='philox'`` noise keyed by (complex, pose) the
    gathered result is the same for any world size up to the fp32 summation order of the scatter atomics."""
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    parts = assign_balanced(costs, world)
    local = [sample_one(i) for i in parts[rank]]
    return gather_ragged(local, _owners(parts, n_complexes), shapes, group=group, device=device)


def _owners(parts: Sequence[Sequence[int]], n_items: int) -> List[int]:
    """``owner[i]``: the rank whose part holds item i."""
    owner = [0] * n_items
    for r, items in enumerate(parts):
        for i in items:
            owner[i] = r
    return owner


def exchange_rows(row: Sequence[int], group=None, device=None) -> torch.Tensor:
    """Every rank's ``row`` (the same length on every rank) as int64 [world, len(row)] on the CPU, by one all_gather on
    ``device`` (default: the current CUDA device under NCCL, the CPU otherwise).  Every rank of ``group`` must call it."""
    world = dist.get_world_size(group)
    t = torch.tensor([int(v) for v in row], dtype=torch.int64, device=device or _default_device(group))
    bufs = [torch.empty_like(t) for _ in range(world)]
    dist.all_gather(bufs, t, group=group)
    return torch.stack(bufs).cpu()


def _confidence_kind(results) -> tuple:
    """(ndim, columns) shared by the confidences of ``results`` [(pos [P, ...], confidence)]: (0, 0) for None, (1, 1) for
    [P], (2, C) for [P, C] - so [P] and [P, 1] stay apart."""
    kinds = set()
    for pos, conf in results:
        if conf is None:
            kinds.add((0, 0))
        elif conf.dim() in (1, 2) and conf.shape[0] == pos.shape[0]:
            kinds.add((conf.dim(), 1 if conf.dim() == 1 else int(conf.shape[1])))
        else:
            raise ValueError(f"a confidence of shape {tuple(conf.shape)} for {pos.shape[0]} poses")
    if len(kinds) != 1:
        raise ValueError(f"complexes of one call with different confidence shapes: {sorted(kinds)}")
    return kinds.pop()


def _sample_owned(ks, shapes, load, sample_args, seed, options):
    """One rank's share: ``load(k)`` for every complex k of ``ks`` (ascending), then ONE ``sampling.sample_packed`` over them
    with their global indices as ``complex_ids``.  Returns ([(pos [n_poses, n_atoms, 3], confidence or None)] in the order of
    ``ks``, whether confidence graphs were given)."""
    from . import sampling
    if not ks:
        return [], False
    poses, graphs = [], []
    for k in ks:
        p, c = load(k)
        atoms = sorted({int(d['ligand'].num_nodes) for d in p})
        if len(p) != shapes[k][0] or atoms != [shapes[k][1]]:
            raise ValueError(f"complex {k}: load gave {len(p)} poses of {atoms} ligand atoms, shapes[{k}] = "
                             f"{tuple(shapes[k])}")
        poses.append(p)
        graphs.append(c)
    given = [c is not None for c in graphs]
    if any(given) and not all(given):
        raise ValueError("load must return confidence graphs for every complex or for none")
    out = sampling.sample_packed(poses, *sample_args, seed=seed, complex_ids=list(ks),
                                 confidence_data=graphs if all(given) else None, **options)
    return [(torch.stack([d['ligand'].pos for d in dl]), conf) for dl, conf in out], all(given)


def sample_packed_sharded(n_complexes: int, costs: Sequence[float], shapes: Sequence[Sequence[int]],
                          load: Callable[[int], tuple], model, inference_steps, tr_schedule, rot_schedule, tor_schedule,
                          device, t_to_sigma, model_args, *, seed, group=None, gather_device=None,
                          **sample_packed_options) -> List[tuple]:
    """``sampling.sample_packed`` over the ranks of ``group``: whole complexes per rank, packed within each rank, ONE
    gather of every complex's final poses and confidences.

    ``costs[k]``: what ``assign_balanced`` balances on (N_r * N_l * poses; ``sampling.pack_cost`` gives the same number for a
    loaded complex).  ``shapes[k] = (n_poses, n_atoms)`` sizes the gather.  ``load(k) -> (poses, confidence_graphs or
    None)`` is called once per call, only on the rank that owns complex k; it returns confidence graphs for every complex or
    for none.  ``sample_packed_options``: the keywords of ``sample_packed`` (``confidence_model``, ``confidence_model_args``,
    ``max_pairs``, ``cuda_graph``, ``no_random``, ``ode``, ``no_final_step_noise``, ``temp_*``), passed through unchanged.

    Each rank owns ``assign_balanced(costs, world)[rank]`` (computed alike on every rank, no communication) and makes ONE
    ``sample_packed`` call over its complexes in ascending order with ``complex_ids`` = their global indices, so every pose
    draws the Philox noise keyed ``(k << 32) | pose`` that it draws on one GPU, and the confidence graphs go in as
    ``confidence_data``.  A complex's result therefore does not depend on the number of ranks, up to the summation order of
    the scatter atomics (``sample_packed``'s own guarantee against one ``sampling()`` call per complex).

    Two collectives, entered by every rank, also by one that owns nothing: an int64 [world, 4] exchange of each rank's
    status (ok / failed, with the exception caught), whether it had confidence graphs and its confidence shape, then
    ``gather_ragged`` of each complex as n_poses x (3 n_atoms + C) fp32 rows (C = 0 without a confidence model).  If any rank
    failed - ``load`` or ``sample_packed`` raised, e.g. a refusal of ``sample_packed`` that only the owning rank meets - or
    the ranks disagree on confidence graphs or shape, every rank raises ``RuntimeError`` naming the failed ranks, with its
    own exception as the cause, and no rank enters the gather.  The gather runs on ``gather_device``, default the current
    CUDA device under NCCL and the CPU otherwise.  Without a process group, or with one rank, the call is one
    ``sample_packed`` over all complexes and no collective (results moved to ``gather_device`` when given).

    Returns ``[(pos [n_poses, n_atoms, 3], confidence or None)]`` per complex, in complex order, on every rank: the
    confidences are ``sample_packed``'s (``nan_to_num(..., nan=-1000)``), of shape [n_poses] or [n_poses, C] as it gave them."""
    if len(costs) != n_complexes or len(shapes) != n_complexes:
        raise ValueError("one cost and one shape per complex")
    sample_args = (model, inference_steps, tr_schedule, rot_schedule, tor_schedule, device, t_to_sigma, model_args)
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    if world == 1:
        out, _ = _sample_owned(list(range(n_complexes)), shapes, load, sample_args, seed, sample_packed_options)
        if gather_device is not None:
            out = [(p.to(gather_device), c if c is None else c.to(gather_device)) for p, c in out]
        return out
    if n_complexes == 0:
        return []
    rank = dist.get_rank(group)
    parts = assign_balanced(costs, world)
    row, err, local = [0, -1, -1, 0], None, []          # failed, confidence graphs given, confidence ndim, columns
    try:
        local, given = _sample_owned(parts[rank], shapes, load, sample_args, seed, sample_packed_options)
        if local:
            row = [0, int(given), *_confidence_kind(local)]
    except Exception as e:                               # reported to every rank below, then raised here
        row, err = [1, -1, -1, 0], e
    gdev = gather_device if gather_device is not None else _default_device(group)
    rows = exchange_rows(row, group, gdev)
    failed = [r for r in range(world) if int(rows[r, 0])]
    if failed:
        msg = f"sample_packed_sharded: rank(s) {failed} failed"
        if err is not None:
            msg += f"; rank {rank}: {type(err).__name__}: {err}"
        raise RuntimeError(msg) from err
    kinds = {tuple(rows[r, 1:].tolist()) for r in range(world) if parts[r]}
    if len(kinds) != 1:
        raise RuntimeError(f"sample_packed_sharded: the ranks disagree on (confidence graphs given, confidence ndim, "
                           f"columns): {rows[:, 1:].tolist()}")
    _, ndim, cols = kinds.pop()
    C = cols if ndim else 0
    flat = gather_ragged([torch.cat([p.reshape(p.shape[0], -1)] + ([c.reshape(p.shape[0], -1)] if C else []), 1)
                          for p, c in local], _owners(parts, n_complexes),
                         [(P, 3 * a + C) for P, a in shapes], group=group, device=gdev)
    out = []
    for f, (P, a) in zip(flat, shapes):
        conf = None if ndim == 0 else f[:, 3 * a] if ndim == 1 else f[:, 3 * a:]
        out.append((f[:, :3 * a].reshape(P, a, 3), conf))
    return out
