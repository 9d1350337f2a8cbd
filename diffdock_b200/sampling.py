"""Reverse-diffusion sampler: drop-in for ``utils/sampling.py:sampling`` (same arguments and return value).

Per step the reference runs ~40 small PyTorch ops, a Python loop over rotatable bonds with host-sync asserts and a
batched cuSOLVER SVD (utils/sampling.py:133-191, utils/diffusion_utils.py:60-78, utils/torsion.py:75-90,
utils/geometry.py:246-276).  Here a step is: ``set_time`` (device fills) -> score model -> ONE pose-update kernel
(``ddb200_pose_update``) that forms the three perturbations from host-computed SDE coefficients, moves the ligand
rigidly, applies the torsion updates sequentially and Kabsch-aligns - no host synchronisation inside the loop apart
from the neighbour-list sizes in the score model.
"""
from __future__ import annotations

import copy
import math
import os

import numpy as np
import torch

from . import ops
from .diffusion_utils import set_time
from .hetero import HeteroGraph, collate, collate_packed, collate_shared_receptor


def randomize_position(data_list, no_torsion, no_random, tr_sigma_max, pocket_knowledge=False, pocket_cutoff=7,
                       initial_noise_std_proportion=-1.0, choose_residue=False):
    """Prior sample of every pose, in place: drop-in for ``utils/sampling.py:16-58`` (called by inference.py:237 right before
    ``sampling``).  Same arguments, same random streams in the same order - numpy's global generator for the torsion angles
    (all poses first, :33-40) and, through scipy's ``Rotation.random``, for the rotations; Python's ``random`` / torch's
    global generator for the translation (:45-57) - so a seeded run reproduces the reference's poses bit for bit.
    Host arithmetic like the reference's (a few hundred flops per pose); what changes is that the poses may be the
    light-weight ``inputs.pose_copies`` of a device-resident complex: receptor statistics are then taken on the device once
    and only three floats come back."""
    import random as _random
    from scipy.spatial.transform import Rotation as R
    rec0 = data_list[0]['receptor']
    lig_dev = data_list[0]['ligand'].pos.device
    center_pocket = rec0.pos.mean(dim=0).to(lig_dev)
    if pocket_knowledge:
        cpx = data_list[0]
        ref_lig = torch.from_numpy(cpx['ligand'].orig_pos[0]).float() - cpx.original_center.cpu()
        d = torch.cdist(rec0.pos.cpu(), ref_lig)
        label = torch.any(d < pocket_cutoff, dim=1)
        if torch.any(label):
            center_pocket = rec0.pos.cpu()[label].mean(dim=0)
        else:
            print("No pocket residue below minimum distance ", pocket_cutoff, "taking closest at", torch.min(d))
            center_pocket = rec0.pos.cpu()[torch.argmin(torch.min(d, dim=1)[0])]
    if not no_torsion:
        for g in data_list:
            lig = g['ligand']
            mask = lig.mask_rotate[0] if isinstance(lig.mask_rotate, list) else lig.mask_rotate
            updates = np.random.uniform(low=-np.pi, high=np.pi, size=int(lig.edge_mask.sum()))
            bonds = g['ligand', 'ligand'].edge_index.T[lig.edge_mask].cpu().numpy()
            pos = lig.pos.cpu().numpy().copy()
            for k, (u, v) in enumerate(bonds):              # utils/torsion.py:48-72: fp64 rotation, fp32 coordinates
                if updates[k] == 0:
                    continue
                axis = pos[u] - pos[v]
                rot = R.from_rotvec(axis * updates[k] / np.linalg.norm(axis)).as_matrix()
                pos[mask[k]] = (pos[mask[k]] - pos[v]) @ rot.T + pos[v]
            lig.pos = torch.from_numpy(pos.astype(np.float32))
    rec_sq = None
    for g in data_list:
        lig = g['ligand']
        centre = torch.mean(lig.pos, dim=0, keepdim=True)
        rot = torch.from_numpy(R.random().as_matrix()).float()
        lig.pos = (lig.pos - centre) @ rot.T + center_pocket
        if not no_random:
            rpos = g['receptor'].pos
            if choose_residue:
                idx = _random.randint(0, len(rpos) - 1)
                tr_update = torch.normal(mean=rpos[idx:idx + 1].cpu(), std=0.01)
            elif initial_noise_std_proportion >= 0.0:
                if rec_sq is None or g['receptor'] is not rec0:
                    rec_sq = torch.sqrt(torch.mean(torch.sum(rpos ** 2, dim=1))).cpu()
                tr_update = torch.normal(mean=0, std=rec_sq * initial_noise_std_proportion / 1.73, size=(1, 3))   # fp32 product
            else:
                tr_update = torch.normal(mean=0, std=-initial_noise_std_proportion * tr_sigma_max, size=(1, 3))
            lig.pos = lig.pos + tr_update


def rank_poses(data_list, confidence, original_center, rmsd_classification_cutoff=None):
    """The epilogue of a docking run, inference.py:274-283: absolute ligand coordinates of every pose (the graphs are centred
    on the receptor: + ``original_center``) ordered by decreasing confidence.  ``confidence``: what ``sampling`` returned (None:
    poses stay in sampling order); a list-valued ``rmsd_classification_cutoff`` (multi-threshold confidence head) ranks by the
    first output column, as the reference does.  Returns (ligand_pos [N, n_atoms, 3] float array, confidence [N] or None,
    re_order [N] or None).  ONE device->host copy for all poses instead of one per pose."""
    pos = torch.stack([g['ligand'].pos for g in data_list])
    ligand_pos = pos.cpu().numpy() + torch.as_tensor(original_center).cpu().numpy()
    if confidence is None:
        return ligand_pos, None, None
    if isinstance(rmsd_classification_cutoff, list):
        confidence = confidence[:, 0]
    confidence = confidence.cpu().numpy()
    re_order = np.argsort(confidence)[::-1]
    return ligand_pos[re_order], confidence[re_order], re_order


def is_iterable(arr):
    try:
        iter(arr)
        return True
    except TypeError:
        return False


def _triple(v):
    return list(v) if is_iterable(v) else [v] * 3


def _nan_guard(tr, rot, tor):
    """utils/sampling.py:117-131 without the host round trip: scores are only touched when a NaN shows up in the
    per-pose mean of the translation score."""
    cond = torch.isnan(tr.mean(dim=-1)).any()

    def fix(s):
        if s is None or s.numel() == 0:
            return s
        eps = 0.01 * torch.nanmean(s.abs())
        s = torch.where(cond & torch.isnan(s), eps, s)
        s = torch.where(cond & (s == float('inf')), eps, s)
        return torch.where(cond & (s == float('-inf')), -eps, s)

    return fix(tr), fix(rot), fix(tor)


def _nan_guard_packed(tr, rot, tor, pose_ptr, bond_ptr):
    """``_nan_guard`` per complex of a packed batch, still without a host read: the condition (a NaN in the per-pose mean of
    the translation score) and ``0.01 * nanmean(|s|)`` are taken over each complex's poses (tr, rot) and bonds (tor), as if
    it were sampled alone.  ``pose_ptr`` / ``bond_ptr`` [K + 1]: the pose and bond offsets of the complexes (device)."""
    K = pose_ptr.shape[0] - 1
    pose_id = torch.searchsorted(pose_ptr[1:], torch.arange(tr.shape[0], device=tr.device), right=True)
    cond = torch.zeros(K, device=tr.device).index_add_(0, pose_id, torch.isnan(tr.mean(dim=-1)).float()) > 0

    def fix(s, seg):
        if s is None or s.numel() == 0:
            return s
        ids = seg.view((-1,) + (1,) * (s.dim() - 1)).expand_as(s)
        a = s.abs()
        ok = ~torch.isnan(a)
        num = torch.zeros(K, device=s.device, dtype=s.dtype).index_add_(0, ids.reshape(-1), torch.where(ok, a, 0).reshape(-1))
        den = torch.zeros(K, device=s.device, dtype=s.dtype).index_add_(0, ids.reshape(-1), ok.to(s.dtype).reshape(-1))
        eps = (0.01 * (num / den))[ids]
        c = cond[ids]
        s = torch.where(c & torch.isnan(s), eps, s)
        s = torch.where(c & (s == float('inf')), eps, s)
        return torch.where(c & (s == float('-inf')), -eps, s)

    bond_id = None
    if tor is not None and tor.numel():
        bond_id = torch.searchsorted(bond_ptr[1:], torch.arange(tor.shape[0], device=tor.device), right=True)
    return fix(tr, pose_id), fix(rot, pose_id), fix(tor, bond_id)


def step_coefficients(t_idx, inference_steps, tr_schedule, rot_schedule, tor_schedule, t_to_sigma, model_args, ode,
                      temp_sampling, temp_psi, temp_sigma_data):
    """Host scalars (a, c) per degree of freedom such that  perturbation = a * score + c * z
    (utils/sampling.py:97-102,133-186)."""
    last = t_idx == inference_steps - 1
    ts, tp, tsd = _triple(temp_sampling), _triple(temp_psi), _triple(temp_sigma_data)
    out = []
    sig = t_to_sigma(tr_schedule[t_idx], rot_schedule[t_idx], tor_schedule[t_idx])
    lims = [(model_args.tr_sigma_min, model_args.tr_sigma_max), (model_args.rot_sigma_min, model_args.rot_sigma_max),
            (model_args.tor_sigma_min, model_args.tor_sigma_max)]
    for k, sched in enumerate((tr_schedule, rot_schedule, tor_schedule)):
        dt = float(sched[t_idx] - sched[t_idx + 1]) if not last else float(sched[t_idx])
        s_min, s_max = lims[k]
        sigma = float(sig[k])
        g = sigma * math.sqrt(2 * math.log(s_max / s_min))
        if ode:
            a, c = 0.5 * g * g * dt, 0.0
        else:
            a, c = g * g * dt, g * math.sqrt(dt)
        if ts[k] != 1.0:       # low-temperature sampling, :173-186 (uses the SDE form even when ode is set)
            sigma_data = math.exp(tsd[k] * math.log(s_max) + (1 - tsd[k]) * math.log(s_min))
            lam = (sigma_data + sigma) / (sigma_data + sigma / ts[k])
            a, c = g * g * dt * (lam + ts[k] * tp[k] / 2), g * math.sqrt(dt * (1 + tp[k]))
        out += [a, c]
    return out


def crop_receptor(g, cutoff):
    """Device-side ``crop_beyond`` (utils/utils.py:388-413, called per step at utils/sampling.py:104-109): a view of the
    batch whose receptor keeps only the residues within ``cutoff`` of some ligand atom of the same complex, contact edges
    restricted and relabelled.  The reference deep-copies the batch, splits it into a Python list, crops each complex
    and re-collates; here one neighbour-count kernel + index compaction does the same on the device.  The ligand store is
    shared with ``g`` (the sampler keeps updating ``g['ligand'].pos``); like the reference's fresh Batch, the returned
    graph carries no cached receptor embeddings."""
    from .hetero import HeteroGraph, Store
    if not isinstance(g, HeteroGraph):
        raise NotImplementedError("device-side crop_beyond is written against diffdock_b200.hetero.HeteroGraph batches")
    lig, rec, rr = g['ligand'], g['receptor'], g['receptor', 'receptor']
    B = g.num_graphs
    lig_ptr = ops.segment_ptr(lig.batch, B)
    _, _, count = ops.radius(lig.pos, rec.pos, lig_ptr, rec.batch, r=float(cutoff), max_num_neighbors=1)
    keep = count > 0
    out = HeteroGraph()
    out._nodes['ligand'] = lig
    for k, st in g._nodes.items():
        if k not in ('ligand', 'receptor'):
            out._nodes[k] = st
    new = Store()
    for k, v in rec.__dict__.items():
        if k in ('rec_node_attr', 'ptr', 'node_t') or k.startswith('_'):
            continue
        if torch.is_tensor(v) and v.dim() > 0 and v.shape[0] == keep.shape[0]:
            setattr(new, k, v[keep])
        else:
            setattr(new, k, v)
    out._nodes['receptor'] = new
    ei = rr.edge_index
    ok = keep[ei[0]] & keep[ei[1]]
    relabel = torch.cumsum(keep.long(), 0) - 1
    out._edges[('receptor', 'receptor')] = Store(edge_index=relabel[ei[:, ok]])
    for et, st in g._edges.items():
        if et != ('receptor', 'receptor'):
            out._edges[et] = st
    for k, v in g._globals.items():
        out._globals[k] = v
    return out


_GRAPH_POOLS = {}


def _graph_pool(device):
    """(memory pool, capture stream, warm-up stream) shared by the step graphs of one device.  torch releases a graph pool when
    the last graph captured into it dies, so a one-kernel anchor graph keeps it alive for the life of the process.  The two
    streams are persistent as well: the caching allocator keeps one block cache per stream, so a fresh side stream per batch
    (the usual warm-up recipe) made every batch cudaMalloc its working set again."""
    dev = torch.device(device)
    key = dev.index if dev.index is not None else torch.cuda.current_device()
    if key not in _GRAPH_POOLS:
        pool = torch.cuda.graph_pool_handle()
        anchor = torch.cuda.CUDAGraph()
        scratch = torch.zeros(8, device=dev)
        torch.cuda.synchronize(dev)
        with torch.cuda.graph(anchor, pool=pool):
            scratch.add_(1.0)
        _GRAPH_POOLS[key] = (pool, anchor, scratch, torch.cuda.Stream(device=dev), torch.cuda.Stream(device=dev))
    e = _GRAPH_POOLS[key]
    return e[0], e[3], e[4]


class GraphedSteps:
    """All reverse-diffusion steps of one batch as replays of ONE CUDA graph.

    The sync-free score model (diffdock_b200.CGModel._forward_sync_free) has static shapes for a given batch, the SDE
    coefficients and schedule times of every step sit in device tables indexed by a device-side step counter, and the pose
    update runs in place - so a step needs no host value at all: the 20 steps of utils/sampling.py:96-191 become 20 graph
    launches (about 500 kernel launches each) with the host idle."""

    def __init__(self, model, g, b, coef_rows, t_rows, bond_u, bond_v, mask_u8, use_torsion, device, draw_noise,
                 philox=None, warmup=1, consume_warmup=False, crop_rows=None, packed=None, frames=None):
        """``consume_warmup``: when a batch of new shapes needs an eager step before the capture, that step IS step 0 of the
        run (``steps_done`` = 1 afterwards) instead of being thrown away - ``run(n)`` then replays the remaining n - 1.
        ``crop_rows``: the squared receptor-crop cut-off of every step (``crop_cutoff2``); the model then crops the receptor
        on the device at each step (needs ``model.sync_free_crop_capable()``).
        ``packed``: a batch of several complexes (``hetero.collate_packed``; ``bond_u`` / ``bond_v`` / ``mask_u8`` are then
        unused): the NaN guard runs per complex and the pose update takes each pose's layout from ``g._pose_layout``.
        ``frames``: a device buffer [steps, n_atoms of the batch, 3]; every step copies the updated ligand coordinates
        into its row, indexed by the device step counter."""
        self.g, self.b, self.device, self.frames = g, b, device, frames
        lig = g['ligand']
        self.pos = lig.pos = lig.pos.float().contiguous().clone()         # static buffer, updated in place
        self.coef = torch.tensor(coef_rows, dtype=torch.float32, device=device).contiguous()        # [steps, 6]
        self.times = torch.tensor(t_rows, dtype=torch.float32, device=device).contiguous()          # [steps, 3]
        self.step = torch.zeros(1, dtype=torch.int32, device=device)
        self.crop = None
        if crop_rows is not None:
            self.crop = torch.tensor(crop_rows, dtype=torch.float32, device=device).contiguous()    # [steps]
            g._crop = (self.crop, self.step)
        n_lig, n_rec = lig.num_nodes, g['receptor'].num_nodes
        names = ('tr', 'rot', 'tor')

        def one_step():
            t = self.times.index_select(0, self.step.long())[0]                                     # [3] on the device
            for nt, n in (('ligand', n_lig), ('receptor', n_rec)):
                g[nt].node_t = {k: t[i].expand(n) for i, k in enumerate(names)}
            g.complex_t = {k: t[i].expand(b) for i, k in enumerate(names)}
            g._uniform_t = True                      # every graph of the batch is at the same diffusion time
            tr, rot, tor = model(g)[:3]
            if packed:
                tr, rot, tor = _nan_guard_packed(tr, rot, tor, g._complex_ptr, g._complex_bond_ptr)
            else:
                tr, rot, tor = _nan_guard(tr, rot, tor)
            has_tor = use_torsion and tor is not None and tor.numel() > 0
            if packed:
                _pose_update_packed(g, self.pos, tr, rot, tor if has_tor else None, self.coef, self.step, philox, has_tor)
            else:
                tr_z = rot_z = tor_z = None
                if draw_noise and philox is None:
                    tr_z = torch.normal(mean=0, std=1, size=(b, 3), device=device)
                    rot_z = torch.normal(mean=0, std=1, size=(b, 3), device=device)
                    if has_tor:
                        tor_z = torch.normal(mean=0, std=1, size=tuple(tor.shape), device=device)
                ops.pose_update_dev(self.pos, b, bond_u, bond_v, mask_u8, tr, rot, tor if has_tor else None, self.coef,
                                    step_dev=self.step, tr_z=tr_z, rot_z=rot_z, tor_z=tor_z,
                                    seed=philox[0] if philox else 0, pose_key=philox[1] if philox else None,
                                    use_torsion=has_tor, out=self.pos)
            if frames is not None:
                frames.index_copy_(0, self.step.long(), self.pos.unsqueeze(0))
            self.step.add_(1)

        pos0 = self.pos.clone()
        # Outside the capture: the per-batch constants (receptor embedding, static CSR; they read sizes back to the host)
        # and, the first time a model meets a batch of these shapes, one eager step: lazy library handles, table uploads,
        # and above all lazy module loading - a kernel variant (cuBLAS picks them by shape, the conv kernel has a single-CTA
        # and a CTA-pair form) that runs for the first time INSIDE a capture invalidates it.
        if hasattr(model, '_static'):
            model._static(g)
        sig = (b, n_lig, n_rec, int(g['ligand', 'ligand'].edge_index.shape[1]), int(g['receptor', 'receptor'].edge_index.shape[1]),
               int(g._pose_layout[1].shape[0]) if packed else int(bond_u.shape[0]) if bond_u is not None else 0, draw_noise,
               philox is not None, crop_rows is not None, frames is not None, ops.deterministic())
        if ops.deterministic():
            ops.fixed_error_word(device)         # the fixed-point scatter's error word exists before the capture
        seen = getattr(model, '_graph_warmed_shapes', None)
        if seen is None:
            seen = set()
            try:
                model._graph_warmed_shapes = seen
            except Exception:
                pass
        n_warm = 0 if sig in seen else warmup
        seen.add(sig)
        self.steps_done = 0
        pool, cap_stream, side = _graph_pool(device)
        cur = torch.cuda.current_stream(device)
        if n_warm:
            side.wait_stream(cur)
            with torch.cuda.stream(side):
                for _ in range(n_warm):
                    one_step()
            cur.wait_stream(side)
            try:
                model._graph_warmed = True
            except Exception:
                pass
        # One memory pool per device shared by all step graphs of this process: a sampling() call captures a new graph per
        # batch (shapes differ from complex to complex); with a private pool each capture would cudaMalloc its whole
        # footprint again (hundreds of ms for a 1500-residue x 40-pose batch) - the blocks of a finished batch's graph are
        # reused instead.  The capture is opened with capture_begin / capture_end on a persistent stream rather than with the
        # torch.cuda.graph context manager, which synchronises the device, runs gc.collect() and empties the allocator cache
        # on entry: measured on BASELINE config 5 that was 50 ms ... 1.9 s per batch (the collector walks every pose graph
        # the process holds; the emptied cache is re-allocated by the next batch) against 0.15-0.4 s of replays.
        self.graph = torch.cuda.CUDAGraph()
        cap_stream.wait_stream(cur)
        with torch.cuda.stream(cap_stream):
            self.graph.capture_begin(pool=pool)
            try:
                one_step()
            finally:
                self.graph.capture_end()
        cur.wait_stream(cap_stream)
        # the capture itself executes nothing.  An eager step that ran before it is either step 0 of this run (same kernels,
        # same device-side step counter and noise streams as a replay) or is undone.
        if n_warm == 1 and consume_warmup:
            self.steps_done = 1
        elif n_warm:
            self.pos.copy_(pos0)
            self.step.zero_()

    def run(self, n_steps):
        for _ in range(n_steps - self.steps_done):
            self.graph.replay()
        self.steps_done = n_steps
        return self.pos


def _collate_any(items, device):
    """diffdock_b200 graphs: shared-receptor collate; torch_geometric HeteroData (what inference.py passes, utils/sampling.py:80):
    PyG's own ``Batch.from_data_list`` - the score model only needs the attribute contract of SURVEY.md section 8(b)."""
    from .hetero import HeteroGraph
    if isinstance(items[0], HeteroGraph):
        return collate_shared_receptor(items, device)
    try:
        from torch_geometric.data import Batch
    except ImportError as e:
        raise TypeError(f"cannot batch {type(items[0]).__name__} objects: pass diffdock_b200.hetero.HeteroGraph items, or "
                        f"install torch_geometric for HeteroData lists") from e
    return Batch.from_data_list(items).to(device)


def _use_cuda_graph(model, model_args, noise_fn, visualization_list, N, batch_size, cuda_graph):
    if cuda_graph is False or os.environ.get('DDB200_CUDA_GRAPH', '1') == '0':
        return False
    crop_ok = getattr(model_args, 'crop_beyond', None) is None or \
        (hasattr(model, 'sync_free_crop_capable') and model.sync_free_crop_capable())
    ok = hasattr(model, 'sync_free_capable') and model.sync_free_capable() and noise_fn is None and crop_ok
    if cuda_graph is True and not ok:
        raise RuntimeError("cuda_graph=True needs the sync-free model path, no noise_fn, and a model that crops on the "
                           "device when crop_beyond is set")
    return ok


def _pose_update_packed(g, pos, tr, rot, tor, coef, step_dev, philox, has_tor):
    """One in-place ddb200_pose_update_packed step of the packed batch ``g`` (Philox noise keyed by ``philox = (seed,
    pose keys)``).  Out-of-range poses set ``g._pose_err``, which ``sample_packed`` reads once at the end."""
    layout, bu, bv, mask, max_atoms = g._pose_layout
    ops.pose_update_packed(pos, layout, max_atoms, bu, bv, mask, tr, rot, tor, coef, g._pose_err, step_dev=step_dev,
                           seed=philox[0], pose_key=philox[1], use_torsion=has_tor, out=pos)


def crop_cutoff2(t_to_sigma, t_tr, t_rot, t_tor, crop_beyond):
    """The squared receptor-crop cut-off of a step as a float32 value: (3 sigma_tr + crop_beyond)^2 in float64
    (utils/sampling.py:108), rounded as torch rounds a Python float compared with a float32 tensor (utils/utils.py:397)."""
    cutoff = float(t_to_sigma(t_tr, t_rot, t_tor)[0]) * 3 + crop_beyond
    return float(np.float32(cutoff ** 2))


def _eager_steps(g, b, model, inference_steps, tr_schedule, rot_schedule, tor_schedule, t_schedule, t_to_sigma, model_args,
                 coef_rows, device, bond_u, bond_v, mask_u8, use_torsion, ode, no_random, no_final_step_noise, noise_fn,
                 n_noise, philox, frames, packed=False):
    """The step loop launched op by op (utils/sampling.py:96-191): injected noise, a ``t_schedule``, or a score model whose
    shapes or cropping are outside the sync-free path.  ``frames``: as for ``GraphedSteps``.  ``packed``: a batch of several
    complexes (``GraphedSteps``), Philox noise only."""
    coef_dev = torch.tensor(coef_rows, dtype=torch.float32, device=device) if philox else None
    for t_idx in range(inference_steps):
        t_tr, t_rot, t_tor = tr_schedule[t_idx], rot_schedule[t_idx], tor_schedule[t_idx]
        if getattr(model_args, 'crop_beyond', None) is not None:
            tr_sigma = float(t_to_sigma(t_tr, t_rot, t_tor)[0])
            mod = crop_receptor(g, tr_sigma * 3 + model_args.crop_beyond)
        else:
            mod = g
        set_time(mod, t_schedule[t_idx] if t_schedule is not None else None, t_tr, t_rot, t_tor, b,
                 bool(getattr(model_args, 'all_atoms', False)), device)
        mod._uniform_t = True                        # set_time gives every graph of the batch the same diffusion time
        tr_score, rot_score, tor_score = model(mod)[:3]
        if packed:
            tr_score, rot_score, tor_score = _nan_guard_packed(tr_score, rot_score, tor_score, g._complex_ptr,
                                                               g._complex_bond_ptr)
        else:
            tr_score, rot_score, tor_score = _nan_guard(tr_score, rot_score, tor_score)
        has_tor = use_torsion and tor_score.numel() > 0
        if packed:
            step_dev = torch.full((1,), t_idx, dtype=torch.int32, device=device)
            g['ligand'].pos = g['ligand'].pos.float().contiguous()
            _pose_update_packed(g, g['ligand'].pos, tr_score, rot_score, tor_score if has_tor else None, coef_dev, step_dev,
                                philox, has_tor)
        elif philox:        # in-kernel counter-based noise: the same draws as the graphed path
            step_dev = torch.full((1,), t_idx, dtype=torch.int32, device=device)
            g['ligand'].pos = ops.pose_update_dev(
                g['ligand'].pos.float().contiguous(), b, bond_u, bond_v, mask_u8, tr_score, rot_score,
                tor_score if has_tor else None, coef_dev, step_dev=step_dev, seed=philox[0], pose_key=philox[1],
                use_torsion=has_tor)
        else:
            zero = no_random or (no_final_step_noise and t_idx == inference_steps - 1)
            tr_z = rot_z = tor_z = None
            if not ode and not zero:
                draw = (lambda kind, shape: noise_fn(kind, shape).to(device)) if noise_fn is not None else \
                    (lambda kind, shape: torch.normal(mean=0, std=1, size=shape, device=device))
                tr_z = draw('tr', (n_noise, 3))
                rot_z = draw('rot', (n_noise, 3))
                if use_torsion:
                    tor_z = draw('tor', tuple(tor_score.shape))
            coef = list(coef_rows[t_idx])
            g['ligand'].pos = ops.pose_update(g['ligand'].pos, b, bond_u, bond_v, mask_u8, tr_score, rot_score,
                                              tor_score if has_tor else None, coef, tr_z, rot_z, tor_z, use_torsion=has_tor)
        if frames is not None:
            frames[t_idx].copy_(g['ligand'].pos)


def _add_frames(visualization_list, data_list, b0, frames):
    """Hand the frames of the batch whose first pose is ``b0`` to the caller's visualisation objects (``add(coords, order,
    part=0, repeat=1)``, utils/visualise.py:PDBFile).  ``frames`` [steps, b, n_atoms, 3] on the host: the ligand
    coordinates after every step.  Leaves what the reference leaves: frame t + original_center at part 1, order t + 2
    (utils/sampling.py:193-197), except order 2, which the reference overwrites with each pose's final coordinates once
    its batch has run (:203-206) - so frame 0 is not kept.  Other entries of the objects are not touched."""
    steps = frames.shape[0]
    for i in range(frames.shape[1] if steps else 0):
        vis, center = visualization_list[b0 + i], data_list[b0 + i].original_center.detach().cpu()
        vis.add(frames[steps - 1, i] + center, part=1, order=2)
        for t in range(1, steps):
            vis.add(frames[t, i] + center, part=1, order=t + 2)


def _step_tables(inference_steps, tr_schedule, rot_schedule, tor_schedule, t_to_sigma, model_args, ode, no_random,
                 no_final_step_noise, temp_sampling, temp_psi, temp_sigma_data):
    """``(coef_rows [steps][6], t_rows [steps][3])``: the SDE coefficients (zero noise where the step draws none) and the
    schedule times of every step."""
    coef_rows, t_rows = [], []
    for t_idx in range(inference_steps):
        coef = step_coefficients(t_idx, inference_steps, tr_schedule, rot_schedule, tor_schedule, t_to_sigma,
                                 model_args, ode, temp_sampling, temp_psi, temp_sigma_data)
        if ode or no_random or (no_final_step_noise and t_idx == inference_steps - 1):
            coef[1] = coef[3] = coef[5] = 0.0          # no noise in this step (utils/sampling.py:136-145,158-161)
        coef_rows.append(coef)
        t_rows.append([float(tr_schedule[t_idx]), float(rot_schedule[t_idx]), float(tor_schedule[t_idx])])
    return coef_rows, t_rows


def _crop_rows(inference_steps, tr_schedule, rot_schedule, tor_schedule, t_to_sigma, model_args):
    crop_beyond = getattr(model_args, 'crop_beyond', None)
    return None if crop_beyond is None else [
        crop_cutoff2(t_to_sigma, tr_schedule[i], rot_schedule[i], tor_schedule[i], crop_beyond)
        for i in range(inference_steps)]


def _rank_batch(confidence_model, confidence_model_args, items, g, pos, b, device):
    """The confidence of ``b`` final poses (utils/sampling.py:197-227): ``items`` are their confidence graphs and ``pos``
    their final ligand coordinates; ``items`` None ranks the score batch ``g`` itself."""
    if items is None:
        out = confidence_model(g)
        return out[0] if type(out) is tuple else out
    crop = getattr(confidence_model_args, 'crop_beyond', None)
    if isinstance(items[0], HeteroGraph) and not (crop is not None and confidence_model_args.all_atoms):
        # one receptor copy uploaded and tiled on the device; the collate builds new stores, so the caller's
        # items are never written to, and the final positions stay on the device
        cg = collate_shared_receptor(items, device)
        cg['ligand'].pos = pos.clone()
    else:
        cg = collate(copy.deepcopy(items))
        cg['ligand'].pos = pos.cpu()
        cg = cg.to(device)
    if crop is not None:                                                    # utils/sampling.py:213-217
        cg = crop_receptor(cg, crop)
    return _confidence_at_t0(confidence_model, confidence_model_args, cg, device)


def _confidence_at_t0(confidence_model, confidence_model_args, cg, device):
    """One confidence forward of the collated batch ``cg`` with every graph at t = 0 (utils/sampling.py:218-227)."""
    set_time(cg, 0, 0, 0, 0, cg.num_graphs, confidence_model_args.all_atoms, device)
    cg._uniform_t = True                 # every graph of the batch is ranked at t = 0
    out = confidence_model(cg)
    return out[0] if type(out) is tuple else out


def _rank_route(confidence_model, confidence_model_args, confidence_data):
    """How ``sample_packed`` ranks: None without a confidence model; 'score': each score pack's own batch (no confidence
    graphs, as ``sampling`` ranks with ``confidence_data_list=None``); 'complex': one ``_rank_batch`` per complex, for a
    confidence ``crop_beyond`` (the eager ``crop_receptor`` keeps no receptor block layout) or confidence graphs that are
    not ``HeteroGraph``; else 'packed': ranking packs (``_rank_packed``)."""
    if confidence_model is None:
        return None
    if confidence_data is None:
        return 'score'
    if getattr(confidence_model_args, 'crop_beyond', None) is not None or \
            not all(isinstance(items[0], HeteroGraph) for items in confidence_data):
        return 'complex'
    return 'packed'


def _rank_packed(confidence_model, confidence_model_args, confidence_data, finals, max_pairs, device):
    """The confidences of several complexes' final poses, one confidence forward per ranking pack: the complexes' confidence
    graphs are packed greedily by their own ``pack_cost`` (receptor atoms counted for an all-atom ranker, whose graphs can
    cost far more than the score graphs) within ``max_pairs``, collated with ``hetero.collate_packed`` (each distinct
    receptor uploaded once), and given the final ligand coordinates ``finals[k]`` [poses x atoms, 3] by one device copy.
    Returns one ``nan_to_num(confidence, nan=-1000)`` per complex, in input order."""
    all_atoms = bool(getattr(confidence_model_args, 'all_atoms', False))
    out = [None] * len(confidence_data)
    for pack in pack_plan([pack_cost(items, all_atoms) for items in confidence_data], max_pairs):
        for k in pack:
            if finals[k].shape[0] != sum(int(d['ligand'].num_nodes) for d in confidence_data[k]):
                raise ValueError(f"complex {k}: the confidence graphs' ligands do not have the score graphs' atoms")
        cg = collate_packed([confidence_data[k] for k in pack], device)
        # the ligands are the same molecules in both batches: poses in the same order, atoms in the same order
        cg['ligand'].pos = torch.cat([finals[k] for k in pack])
        conf = torch.nan_to_num(_confidence_at_t0(confidence_model, confidence_model_args, cg, device), nan=-1000)
        for k, part in zip(pack, torch.split(conf, [len(confidence_data[k]) for k in pack])):
            out[k] = part
    return out


@torch.no_grad()
def sampling(data_list, model, inference_steps, tr_schedule, rot_schedule, tor_schedule, device, t_to_sigma, model_args,
             no_random=False, ode=False, visualization_list=None, confidence_model=None, confidence_data_list=None,
             confidence_model_args=None, t_schedule=None, batch_size=32, no_final_step_noise=False, pivot=None,
             return_full_trajectory=False, temp_sampling=1.0, temp_psi=0.0, temp_sigma_data=0.5, return_features=False,
             noise_fn=None, cuda_graph=None, rng=None, seed=0, pose_keys=None):
    """Same arguments and return value as ``utils/sampling.py:sampling``.  Extensions (all optional):
    ``noise_fn(kind, shape) -> tensor`` (kind in 'tr','rot','tor') replaces the device RNG - used by the injected-noise parity
    tests; otherwise torch.normal is drawn on ``device`` in the reference's order.
    ``cuda_graph``: None = capture the step in a CUDA graph whenever possible, True = require it, False = eager steps.
    ``rng='philox'``: noise from counter-based Philox streams keyed by (``seed``, ``pose_keys[i]``) and indexed by the step,
    so the result for a pose does not depend on batch composition or on how poses are sharded over GPUs (SURVEY.md 8(e));
    ``pose_keys`` [len(data_list)] int64 = (complex id << 32) | pose id, default 0..N-1."""
    assert not (return_full_trajectory or return_features or pivot), "Not implemented yet in new inference version"
    device = torch.device(device)
    if device.type != 'cuda':
        raise RuntimeError("diffdock_b200.sampling runs on a CUDA device only (no CPU fallback)")
    N = len(data_list)
    lig0 = data_list[0]['ligand']
    mask_rotate = np.asarray(lig0.mask_rotate[0] if isinstance(lig0.mask_rotate, list) else lig0.mask_rotate)
    mask_u8 = torch.from_numpy(mask_rotate.astype(np.uint8)).contiguous().to(device)
    ei0 = data_list[0]['ligand', 'ligand'].edge_index
    rot_bonds = ei0.T[lig0.edge_mask.cpu()] if ei0.numel() else ei0.T
    bond_u = rot_bonds[:, 0].to(torch.int32).contiguous().to(device)
    bond_v = rot_bonds[:, 1].to(torch.int32).contiguous().to(device)
    use_torsion = not model_args.no_torsion
    confidence = [] if confidence_model is not None else None
    conf_batches = None
    if confidence_model is not None and confidence_data_list is not None:
        conf_batches = [confidence_data_list[i:i + batch_size] for i in range(0, len(confidence_data_list), batch_size)]

    philox = rng == 'philox'
    assert rng in (None, 'philox'), "rng: None (torch.normal in the reference's order) or 'philox'"
    if philox:
        assert noise_fn is None
        keys_all = torch.arange(N, dtype=torch.int64) if pose_keys is None else torch.as_tensor(pose_keys, dtype=torch.int64)
    graphed = _use_cuda_graph(model, model_args, noise_fn, visualization_list, N, batch_size, cuda_graph)

    for batch_id, b0 in enumerate(range(0, N, batch_size)):
        g = _collate_any(data_list[b0:b0 + batch_size], device)
        b = g.num_graphs
        n = len(g['ligand'].pos) // b
        keys = keys_all[b0:b0 + b].to(device) if philox else None
        coef_rows, t_rows = _step_tables(inference_steps, tr_schedule, rot_schedule, tor_schedule, t_to_sigma, model_args,
                                         ode, no_random, no_final_step_noise, temp_sampling, temp_psi, temp_sigma_data)
        frames = None
        if visualization_list is not None:
            frames = torch.empty((inference_steps, b * n, 3), dtype=torch.float32, device=device)
        if graphed and t_schedule is None and b > 0:
            crop_rows = _crop_rows(inference_steps, tr_schedule, rot_schedule, tor_schedule, t_to_sigma, model_args)
            steps = GraphedSteps(model, g, b, coef_rows, t_rows, bond_u, bond_v, mask_u8, use_torsion, device,
                                 draw_noise=not (ode or no_random), philox=(seed, keys) if philox else None,
                                 consume_warmup=True, crop_rows=crop_rows, frames=frames)
            steps.run(inference_steps)
        else:
            _eager_steps(g, b, model, inference_steps, tr_schedule, rot_schedule, tor_schedule, t_schedule, t_to_sigma,
                         model_args, coef_rows, device, bond_u, bond_v, mask_u8, use_torsion, ode, no_random,
                         no_final_step_noise, noise_fn, min(batch_size, N), (seed, keys) if philox else None, frames)
        for i in range(b):
            data_list[b0 + i]['ligand'].pos = g['ligand'].pos[i * n:n * (i + 1)]
        if confidence_model is not None:
            items = conf_batches[batch_id] if conf_batches is not None else None
            confidence.append(_rank_batch(confidence_model, confidence_model_args, items, g, g['ligand'].pos, b, device))
        if frames is not None:                   # one device->host copy per batch
            _add_frames(visualization_list, data_list, b0, frames.view(inference_steps, b, n, 3).cpu())
    if confidence_model is not None:
        confidence = torch.nan_to_num(torch.cat(confidence, dim=0), nan=-1000)
    if ops.deterministic():
        ops.check_fixed_error(device)
    return data_list, confidence


def pack_cost(poses, all_atoms=False):
    """The cost of one complex in a pack: poses x ligand atoms x receptor nodes, the capacity of its ligand <- receptor
    cross graphs that sets a step's memory.  Receptor nodes are the residues, plus the receptor atoms for an all-atom score
    model (``all_atoms``; its ligand <- atom graph is the larger of the two)."""
    g = poses[0]
    n_rec = int(g['receptor'].num_nodes) + (int(g._nodes['atom'].num_nodes) if all_atoms else 0)
    return len(poses) * int(g['ligand'].num_nodes) * n_rec


def pack_plan(costs, max_pairs):
    """Greedy packing of complexes, in the given order, into batches whose summed cost (``pack_cost``: poses x ligand atoms x
    receptor nodes, the cross-graph capacity that sets a step's memory) stays within ``max_pairs``; a complex larger than
    the budget gets a batch of its own.  Returns lists of complex indices."""
    packs, cur, total = [], [], 0
    for i, cost in enumerate(costs):
        if cur and total + cost > max_pairs:
            packs.append(cur)
            cur, total = [], 0
        cur.append(i)
        total += cost
    if cur:
        packs.append(cur)
    return packs


PACK_MAX_PAIRS = 40 * 40 * 1500            # BASELINE config 3 (40 poses x 40 atoms x 1500 residues), a size bench.py runs


@torch.no_grad()
def sample_packed(complexes, model, inference_steps, tr_schedule, rot_schedule, tor_schedule, device, t_to_sigma, model_args,
                  *, seed, complex_ids=None, no_random=False, ode=False, no_final_step_noise=False, temp_sampling=1.0,
                  temp_psi=0.0, temp_sigma_data=0.5, confidence_model=None, confidence_data=None,
                  confidence_model_args=None, max_pairs=None, cuda_graph=None, noise_fn=None, visualization_list=None,
                  t_schedule=None):
    """Several docking jobs in one reverse-diffusion step.  ``complexes``: a list of pose lists, each what ``sampling`` takes
    as ``data_list`` for one complex (``HeteroGraph`` items; all-atom graphs for an ``AAModel``).  The complexes are packed
    greedily, in order, into batches of at most ``max_pairs`` poses x ligand atoms x receptor nodes (``pack_cost``: residues,
    plus receptor atoms for an all-atom model; default ``PACK_MAX_PAIRS``; ``pack_plan``); each batch is one
    ``hetero.collate_packed`` and runs its steps as one captured CUDA graph where ``sampling`` would, else eagerly, with
    the packed pose update (ddb200_pose_update_packed) and a per-complex NaN guard.  Noise is always Philox, keyed by
    ``(complex_ids[k] << 32) | pose`` (``complex_ids`` default 0 .. K-1).

    Ranking, after every score pack has run: ``confidence_data`` is one list of confidence graphs per complex.  They are
    packed on their own (``pack_plan`` over ``pack_cost(confidence_data[k], confidence_model_args.all_atoms)`` within the
    same ``max_pairs``: an all-atom confidence graph can cost far more than its score graph), each ranking pack is one
    ``hetero.collate_packed`` that takes its complexes' final ligand coordinates by a device copy, and ONE confidence
    forward at t = 0 ranks the whole pack.  Complexes are ranked one by one with ``sampling``'s code only where a pack
    cannot be formed: a confidence ``crop_beyond`` (the eager receptor crop keeps no receptor block layout) or confidence
    graphs that are not ``HeteroGraph``.  ``confidence_data=None`` ranks each score pack's own batch, as ``sampling``
    does with ``confidence_data_list=None``.  Measured on one H100 80GB HBM3 at a 700 W power limit (DESIGN section 6.5):
    at ``PACK_MAX_PAIRS`` an all-atom ranking graph of the README's screening run fills a ranking pack by itself, so that
    call takes the same time either way (12.39 s against 12.31 s ranking complex by complex); with an 8x budget its
    ranking stage alone takes 163 ms against 449 ms with an ``AAOldModel`` ranker at the trainer defaults.

    Score models: ``CGModel``, ``CGOldModel`` and ``AAModel``; an all-atom model without per-step cropping
    (``model_args.crop_beyond``), which is not built for receptor atoms.

    Returns ``[(data_list, confidence)]`` per complex, in input order: what ``sampling(poses, ..., rng='philox',
    pose_keys=keys, batch_size >= len(poses))`` returns for each complex, up to the summation order of atomics.  The
    ``fixed_center_conv=False`` centre convolution and the NaN guard behave as for a complex sampled alone."""
    if noise_fn is not None or visualization_list is not None or t_schedule is not None:
        raise NotImplementedError("sample_packed draws Philox noise in the pose update: noise_fn, visualization_list and "
                                  "t_schedule are sampling() options")
    from .aa_model import AAModel
    from .old_aa_model import AAOldModel
    all_atoms = isinstance(model, AAModel)
    if isinstance(model, AAOldModel) or (getattr(model_args, 'all_atoms', False) and not all_atoms):
        raise NotImplementedError("sample_packed runs the score models CGModel, CGOldModel and AAModel; model_args.all_atoms "
                                  "asks for an all-atom score model (AAModel)")
    if all_atoms and getattr(model_args, 'crop_beyond', None) is not None:
        raise NotImplementedError("sample_packed does not crop all-atom receptors per step (crop_beyond): the device-side "
                                  "crop covers residues only; sample such complexes one per sampling() call")
    K = len(complexes)
    if confidence_data is not None and len(confidence_data) != K:
        raise ValueError("one list of confidence graphs per complex")
    device = torch.device(device)
    if device.type != 'cuda':
        raise RuntimeError("diffdock_b200.sample_packed runs on a CUDA device only (no CPU fallback)")
    complex_ids = list(range(K)) if complex_ids is None else [int(i) for i in complex_ids]
    if len(complex_ids) != K:
        raise ValueError("one complex id per complex")
    rank = _rank_route(confidence_model, confidence_model_args, confidence_data)
    costs = [pack_cost(p, all_atoms) for p in complexes]
    budget = PACK_MAX_PAIRS if max_pairs is None else max_pairs
    packs = pack_plan(costs, budget)
    use_torsion = not model_args.no_torsion
    graphed = _use_cuda_graph(model, model_args, None, None, 0, 0, cuda_graph)
    coef_rows, t_rows = _step_tables(inference_steps, tr_schedule, rot_schedule, tor_schedule, t_to_sigma, model_args, ode,
                                     no_random, no_final_step_noise, temp_sampling, temp_psi, temp_sigma_data)
    crop_rows = _crop_rows(inference_steps, tr_schedule, rot_schedule, tor_schedule, t_to_sigma, model_args)
    finals, confidence = [None] * K, [None] * K
    errs = []
    for pack in packs:
        g = collate_packed([complexes[k] for k in pack], device)
        b = g.num_graphs
        keys = torch.cat([(complex_ids[k] << 32) + torch.arange(len(complexes[k]), dtype=torch.int64) for k in pack])
        philox = (seed, keys.to(device))
        g._pose_err = torch.zeros(1, dtype=torch.int32, device=device)
        errs.append(g._pose_err)
        if graphed:
            steps = GraphedSteps(model, g, b, coef_rows, t_rows, None, None, None, use_torsion, device,
                                 draw_noise=not (ode or no_random), philox=philox, consume_warmup=True, crop_rows=crop_rows,
                                 packed=True)
            steps.run(inference_steps)
        else:
            _eager_steps(g, b, model, inference_steps, tr_schedule, rot_schedule, tor_schedule, None, t_to_sigma,
                         model_args, coef_rows, device, None, None, None, use_torsion, ode, no_random, no_final_step_noise,
                         None, b, philox, None, packed=True)
        pos, layout = g['ligand'].pos, g._pose_layout[0].cpu()
        p0 = 0
        for k in pack:
            data_list = complexes[k]
            for i, d in enumerate(data_list):
                a0, n = int(layout[p0 + i, 0]), int(layout[p0 + i, 1])
                d['ligand'].pos = pos[a0:a0 + n]
            a1 = int(layout[p0 + len(data_list) - 1, 0] + layout[p0 + len(data_list) - 1, 1])
            finals[k] = pos[int(layout[p0, 0]):a1]           # a view: the final poses stay on the device until ranked
            p0 += len(data_list)
        if rank == 'score':
            conf = torch.nan_to_num(_rank_batch(confidence_model, confidence_model_args, None, g, pos, b, device), nan=-1000)
            for k, part in zip(pack, torch.split(conf, [len(complexes[k]) for k in pack])):
                confidence[k] = part
    if rank == 'packed':
        confidence = _rank_packed(confidence_model, confidence_model_args, confidence_data, finals, budget, device)
    elif rank == 'complex':
        confidence = [torch.nan_to_num(_rank_batch(confidence_model, confidence_model_args, confidence_data[k], None,
                                                   finals[k], len(complexes[k]), device), nan=-1000) for k in range(K)]
    if errs and int(torch.stack(errs).max()):
        raise RuntimeError("ddb200_pose_update_packed met a pose outside the declared layout")
    if ops.deterministic():
        ops.check_fixed_error(device)
    return [(complexes[k], confidence[k]) for k in range(K)]
