"""Duck-typed stand-in for the torch_geometric ``HeteroData`` / ``Batch`` objects the reference passes
to ``model(data)`` (utils/sampling.py:80,116).  torch_geometric is not installed in this image; the
score model only relies on the attribute contract listed in SURVEY.md section 8(b), which this class
provides.  A real PyG ``HeteroDataBatch`` satisfies the same contract and is accepted unchanged.

Edge-store keys follow PyG: a 2-tuple ``('ligand', 'ligand')`` resolves to the single edge type with
those endpoints (datasets/process_mols.py:202,294-295).
"""
from __future__ import annotations

import copy
from typing import Dict, List

import numpy as np
import torch


def _map(v, fn):
    if torch.is_tensor(v):
        return fn(v)
    if isinstance(v, dict):
        return {k: _map(x, fn) for k, x in v.items()}
    return v


class Store:
    """Attribute bag for one node or edge type."""

    def __init__(self, **kw):
        self.__dict__.update(kw)

    @property
    def num_nodes(self):
        for k in ('x', 'pos', 'batch'):
            if k in self.__dict__:
                return self.__dict__[k].shape[0]
        return 0

    @property
    def num_edges(self):
        return self.__dict__['edge_index'].shape[1] if 'edge_index' in self.__dict__ else 0

    def keys(self):
        return list(self.__dict__.keys())

    def __contains__(self, k):
        return k in self.__dict__

    def _apply(self, fn):
        for k, v in list(self.__dict__.items()):
            self.__dict__[k] = _map(v, fn)
        return self


class HeteroGraph:
    """One complex, or a batch of complexes (``num_graphs`` > 1, with per-node ``batch`` vectors)."""

    def __init__(self):
        object.__setattr__(self, '_nodes', {})
        object.__setattr__(self, '_edges', {})
        object.__setattr__(self, '_globals', {})

    # -- item access --------------------------------------------------------------------------
    def __getitem__(self, key):
        if isinstance(key, tuple):
            key = (key[0], key[-1])
            if key not in self._edges:
                self._edges[key] = Store()
            return self._edges[key]
        if key in self._globals:
            return self._globals[key]
        if key not in self._nodes:
            self._nodes[key] = Store()
        return self._nodes[key]

    def __setitem__(self, key, value):
        self._globals[key] = value

    def __getattr__(self, name):
        g = object.__getattribute__(self, '_globals')
        if name in g:
            return g[name]
        raise AttributeError(name)

    def __setattr__(self, name, value):
        self._globals[name] = value

    def __contains__(self, key):
        return key in self._globals or key in self._nodes

    @property
    def node_types(self):
        return list(self._nodes.keys())

    @property
    def edge_types(self):
        return list(self._edges.keys())

    # -- movement / copies --------------------------------------------------------------------
    def _apply(self, fn):
        for s in list(self._nodes.values()) + list(self._edges.values()):
            s._apply(fn)
        for k, v in list(self._globals.items()):
            self._globals[k] = _map(v, fn)
        return self

    def to(self, device, non_blocking=False):
        return self._apply(lambda t: t.to(device, non_blocking=non_blocking))

    def cpu(self):
        return self.to('cpu')

    def clone(self):
        return copy.deepcopy(self)

    def to_data_list(self):
        """Inverse of ``collate`` (torch_geometric Batch.to_data_list) for the attributes the path uses."""
        B = self._globals['num_graphs']
        ptr = {nt: st.ptr.tolist() if 'ptr' in st else None for nt, st in self._nodes.items()}
        for nt, st in self._nodes.items():
            if ptr[nt] is None:
                cnt = torch.bincount(st.batch, minlength=B)
                ptr[nt] = [0] + torch.cumsum(cnt, 0).tolist()
        out = []
        for b in range(B):
            g = HeteroGraph()
            for nt, st in self._nodes.items():
                lo, hi = ptr[nt][b], ptr[nt][b + 1]
                sl = st.__dict__.get('_slices', {})
                for k, v in st.__dict__.items():
                    if k in ('batch', 'ptr') or k.startswith('_'):
                        continue
                    if torch.is_tensor(v) and k in sl and sl[k][-1] == v.shape[0]:
                        setattr(g[nt], k, v[sl[k][b]:sl[k][b + 1]])
                    elif torch.is_tensor(v) and v.dim() > 0 and v.shape[0] == ptr[nt][-1]:
                        setattr(g[nt], k, v[lo:hi])
                    elif isinstance(v, dict):
                        setattr(g[nt], k, {a: t[lo:hi] for a, t in v.items()})
                    elif isinstance(v, list) and len(v) == B:
                        setattr(g[nt], k, v[b])
            for et, st in self._edges.items():
                ei = st.edge_index
                src_ptr, dst_ptr = ptr[et[0]], ptr[et[1]]
                sel = (ei[0] >= src_ptr[b]) & (ei[0] < src_ptr[b + 1])
                for k, v in st.__dict__.items():
                    if k == 'edge_index':
                        off = torch.tensor([[src_ptr[b]], [dst_ptr[b]]], dtype=ei.dtype, device=ei.device)
                        g[et].edge_index = ei[:, sel] - off
                    elif torch.is_tensor(v) and v.dim() > 0 and v.shape[0] == ei.shape[1]:
                        setattr(g[et], k, v[sel])
            for k, v in self._globals.items():
                if k == 'num_graphs':
                    continue
                if isinstance(v, list) and len(v) == B:
                    g._globals[k] = v[b]
                elif torch.is_tensor(v) and v.dim() > 0 and v.shape[0] == B:
                    g._globals[k] = v[b:b + 1]
                elif isinstance(v, dict):
                    g._globals[k] = {a: t[b:b + 1] for a, t in v.items()}
            out.append(g)
        return out

    def __deepcopy__(self, memo):
        g = HeteroGraph()
        for k, s in self._nodes.items():
            g._nodes[k] = Store(**{a: copy.deepcopy(v, memo) for a, v in s.__dict__.items()})
        for k, s in self._edges.items():
            g._edges[k] = Store(**{a: copy.deepcopy(v, memo) for a, v in s.__dict__.items()})
        for a, v in self._globals.items():
            g._globals[a] = copy.deepcopy(v, memo)
        return g


_LIST_ATTRS = ('mask_rotate', 'name', 'mol')


def collate(data_list: List[HeteroGraph]) -> HeteroGraph:
    """Equivalent of ``torch_geometric.data.Batch.from_data_list`` for the attributes the path uses:
    node tensors are concatenated, ``edge_index`` is offset by the cumulative node counts of its endpoint
    types, ``batch`` vectors and ``num_graphs`` are added, non-tensor attributes become lists."""
    out = HeteroGraph()
    B = len(data_list)
    offsets: Dict[str, List[int]] = {}
    for nt in data_list[0].node_types:
        counts = [d[nt].num_nodes for d in data_list]
        offs = [0]
        for c in counts:
            offs.append(offs[-1] + c)
        offsets[nt] = offs
        st = out[nt]
        slices = {}
        for attr in data_list[0][nt].keys():
            if attr.startswith('_'):
                continue
            vals = [getattr(d[nt], attr) for d in data_list]
            if attr in _LIST_ATTRS or not torch.is_tensor(vals[0]):
                setattr(st, attr, vals)
            else:
                setattr(st, attr, torch.cat(vals, 0))
                sizes = [0]
                for v in vals:
                    sizes.append(sizes[-1] + v.shape[0])
                slices[attr] = sizes
        st._slices = slices
        st.batch = torch.cat([torch.full((c,), i, dtype=torch.long) for i, c in enumerate(counts)])
        st.ptr = torch.tensor(offs, dtype=torch.long)
    for et in data_list[0].edge_types:
        st = out[et]
        for attr in data_list[0][et].keys():
            vals = [getattr(d[et], attr) for d in data_list]
            if attr == 'edge_index':
                o0, o1 = offsets[et[0]], offsets[et[1]]
                vals = [v + torch.tensor([[o0[i]], [o1[i]]], dtype=v.dtype) for i, v in enumerate(vals)]
                st.edge_index = torch.cat(vals, 1)
            elif torch.is_tensor(vals[0]):
                setattr(st, attr, torch.cat(vals, 0))
            else:
                setattr(st, attr, vals)
    for k in data_list[0]._globals.keys():
        vals = [d._globals[k] for d in data_list]
        if torch.is_tensor(vals[0]):
            out._globals[k] = torch.cat([v if v.dim() > 0 else v[None] for v in vals], 0)
        else:
            out._globals[k] = vals
    out._globals['num_graphs'] = B
    return out


_RECEPTOR_SIDE = ('receptor', 'atom')


def _receptor_side(g: HeteroGraph):
    """(node types, edge types) of the receptor side of a complex: residues, receptor atoms (all-atom graphs) and every
    edge type touching either."""
    nts = [k for k in _RECEPTOR_SIDE if k in g._nodes]
    return nts, [k for k in g._edges if k[0] in nts or k[1] in nts]


def _same_receptor(a: HeteroGraph, b: HeteroGraph) -> bool:
    """Exact equality of everything the model reads from the receptor side - residues, and receptor atoms with their edges
    when the graphs are all-atom ones (cheap identity checks first)."""
    nts, ets = _receptor_side(a)
    if (nts, ets) != _receptor_side(b) or 'receptor' not in nts:
        return False
    pairs = [(a._nodes[k], b._nodes[k]) for k in nts] + [(a._edges[k], b._edges[k]) for k in ets]
    for sa, sb in pairs:
        ka = [k for k in sa.keys() if not k.startswith('_')]
        if ka != [k for k in sb.keys() if not k.startswith('_')]:
            return False
        for k in ka:
            va, vb = getattr(sa, k), getattr(sb, k)
            if torch.is_tensor(va):
                if not torch.is_tensor(vb) or va.shape != vb.shape or va.dtype != vb.dtype:
                    return False
                if va.data_ptr() != vb.data_ptr() and not torch.equal(va, vb):
                    return False
            elif isinstance(va, (dict, list)):
                return False            # per-node dicts (node_t) / lists: take the general path
            elif va != vb:
                return False
    return True


def collate_shared_receptor(data_list: List[HeteroGraph], device, non_blocking=True) -> HeteroGraph:
    """``collate(data_list).to(device)`` for the sampler's usual input - N poses of ONE complex (inference.py:236-239 deep-
    copies the complex N times): when every item carries the same receptor, only ONE copy of the receptor tensors is
    concatenated on the host and uploaded (7.7 MB instead of 246 MB for 32 poses of a 1500-residue complex with 1280-wide
    language-model embeddings); the batch-level tensors are then tiled on the device, so the result is identical to the
    general path, and the receptor store carries ``_unique = (n_nodes_per_copy, n_edges_per_copy, copies)`` so that the
    score model embeds the receptor once (models/cg_model.py:272-295 recomputes the identical receptor per pose).

    All-atom graphs (the all-atom models' and the all-atom confidence model's input) get the same treatment for the
    receptor-atom store and the ('atom', 'atom') / ('atom', 'receptor') edges: one copy uploaded, tiled on the device with
    per-copy atom and residue offsets, and ``_unique = (n_atoms_per_copy, n_atom_atom_edges_per_copy, copies)`` on the atom
    store.  An edge type between the receptor side and the ligand takes the general path."""
    B = len(data_list)
    if B < 2:
        return collate(data_list).to(device, non_blocking=non_blocking)
    out = _collate_receptor_blocks([data_list], device, non_blocking)
    if out is None:
        return collate(data_list).to(device, non_blocking=non_blocking)
    for nt in _receptor_side(data_list[0])[0]:
        n1, e1, _, _ = out[nt]._blocks[0]
        out[nt]._unique = (n1, e1, B)
        del out[nt].__dict__['_blocks']
    return out


def _collate_receptor_blocks(complexes, device, non_blocking=True):
    """``collate(concatenated pose lists).to(device)`` with each DISTINCT receptor uploaded once and tiled on the device, or
    None when some complex's poses do not share one receptor (or an edge type joins the receptor side to the ligand).
    Consecutive complexes with the same receptor form one block; every receptor-side node store gets ``_blocks`` = one
    ``(nodes per copy, own edges per copy, copies, distinct receptor id)`` per block, in batch order."""
    items = [d for poses in complexes for d in poses]
    first = items[0]
    nts, ets = _receptor_side(first)
    if any(et[0] not in nts or et[1] not in nts for et in ets):
        return None
    if not all(_same_receptor(poses[0], d) for poses in complexes for d in poses[1:]):
        return None
    reps, blocks = [], []              # distinct receptors (one pose each); [distinct id, copies] per block
    for poses in complexes:
        if blocks and _same_receptor(reps[blocks[-1][0]], poses[0]):
            blocks[-1][1] += len(poses)
            continue
        uid = next((u for u, r in enumerate(reps) if _same_receptor(r, poses[0])), None)
        if uid is None:
            uid = len(reps)
            reps.append(poses[0])
        blocks.append([uid, len(poses)])
    B = len(items)
    stripped = []
    for d in items:                           # views without the receptor side: ligand stores are shared, not copied
        h = HeteroGraph()
        for k, st in d._nodes.items():
            if k not in nts:
                h._nodes[k] = st
        for k, st in d._edges.items():
            if k not in ets:
                h._edges[k] = st
        h._globals.update(d._globals)
        stripped.append(h)
    out = collate(stripped).to(device, non_blocking=non_blocking)
    up = {}                                   # (distinct id, store key, attribute) -> device tensor, uploaded once

    def dev(u, key, k, v):
        if (u, key, k) not in up:
            up[(u, key, k)] = v.to(device, non_blocking=non_blocking)
        return up[(u, key, k)]
    tile = lambda dv, c: dv.repeat((c,) + (1,) * (dv.dim() - 1)) if dv.dim() > 0 else dv
    n1 = {nt: [r._nodes[nt].num_nodes for r in reps] for nt in nts}
    for nt in nts:
        st = out[nt]
        for k in first._nodes[nt].keys():
            if k.startswith('_'):
                continue
            vals = [getattr(r._nodes[nt], k) for r in reps]
            if torch.is_tensor(vals[0]):
                setattr(st, k, torch.cat([tile(dev(u, nt, k, vals[u]), c) for u, c in blocks]))
            else:
                setattr(st, k, [vals[u] for u, c in blocks for _ in range(c)])
        per_copy = torch.tensor([n1[nt][u] for u, c in blocks for _ in range(c)], device=device)
        st.batch = torch.arange(B, device=device).repeat_interleave(per_copy)
        st.ptr = torch.cat([torch.zeros(1, dtype=per_copy.dtype, device=device), torch.cumsum(per_copy, 0)])
        own = [r._edges.get((nt, nt)) for r in reps]
        st._blocks = tuple((n1[nt][u], own[u].num_edges if own[u] is not None else 0, c, u) for u, c in blocks)
    for et in ets:
        st = out[et]
        for k in first._edges[et].keys():
            vals = [getattr(r._edges[et], k) for r in reps]
            if k == 'edge_index':
                parts, off0, off1 = [], 0, 0
                for u, c in blocks:
                    ei = dev(u, et, k, vals[u])
                    copy_id = torch.arange(c, device=device).repeat_interleave(ei.shape[1])
                    off = torch.stack([off0 + copy_id * n1[et[0]][u], off1 + copy_id * n1[et[1]][u]])
                    parts.append(ei.repeat(1, c) + off.to(ei.dtype))
                    off0, off1 = off0 + c * n1[et[0]][u], off1 + c * n1[et[1]][u]
                st.edge_index = torch.cat(parts, 1)
            elif torch.is_tensor(vals[0]):
                setattr(st, k, torch.cat([tile(dev(u, et, k, vals[u]), c) for u, c in blocks]))
            else:
                setattr(st, k, [vals[u] for u, c in blocks for _ in range(c)])
    return out


def receptor_blocks(st, num_graphs, n_edges):
    """The receptor block layout of a batch, ``[(node offset, edge offset, nodes per copy, edges per copy, copies, distinct
    id)]``, from ``_blocks`` (collate_packed) or ``_unique`` (collate_shared_receptor) when it describes this batch - every
    graph in exactly one copy, nodes and edges summing to the store's - else None."""
    blocks = getattr(st, '_blocks', None)
    if blocks is None:
        u = getattr(st, '_unique', None)
        blocks = None if u is None else ((u[0], u[1], u[2], 0),)
    if blocks is None:
        return None
    out, noff, eoff = [], 0, 0
    for n1, e1, c, uid in blocks:
        out.append((noff, eoff, n1, e1, c, uid))
        noff, eoff = noff + n1 * c, eoff + e1 * c
    if sum(b[4] for b in out) != num_graphs or noff != st.num_nodes or eoff != n_edges:
        return None
    return out


def pose_layout(complexes):
    """The per-pose descriptor of ddb200_pose_update_packed for the concatenated pose lists, on the host: ``(layout [n_poses,
    6] int32, bond_u int32, bond_v int32, mask uint8 (flat), max_atoms)``.  Rotatable bonds and masks are read from each
    complex's first pose, as ``sampling`` does; every pose must have the same atom and rotatable-bond counts."""
    rows, bu, bv, masks = [], [], [], []
    atom_off = tor_off = bond_off = mask_off = 0
    max_atoms = 0
    for poses in complexes:
        lig0 = poses[0]['ligand']
        n = int(lig0.num_nodes)
        ei = poses[0]['ligand', 'ligand'].edge_index
        rot = ei.T[lig0.edge_mask.cpu()] if ei.numel() else ei.T.reshape(0, 2)
        nb = int(rot.shape[0])
        mask = np.asarray(lig0.mask_rotate[0] if isinstance(lig0.mask_rotate, list) else lig0.mask_rotate)
        if nb:
            if mask.shape != (nb, n):
                raise ValueError(f"mask_rotate of shape {mask.shape} for {nb} rotatable bonds and {n} atoms")
            if int(rot.min()) < 0 or int(rot.max()) >= n:
                raise ValueError("rotatable bond outside the ligand")
            bu.append(rot[:, 0].to(torch.int32))
            bv.append(rot[:, 1].to(torch.int32))
            masks.append(torch.from_numpy(mask.astype(np.uint8).reshape(-1)))
        for d in poses:
            lig = d['ligand']
            if int(lig.num_nodes) != n or int(lig.edge_mask.sum()) != nb:
                raise ValueError("the poses of one complex must have the same atoms and rotatable bonds")
            rows.append([atom_off, n, bond_off, nb, tor_off, mask_off])
            atom_off, tor_off = atom_off + n, tor_off + nb
        bond_off, mask_off = bond_off + nb, mask_off + nb * n
        max_atoms = max(max_atoms, n)
    if max(atom_off, tor_off, mask_off) >= 2 ** 31:
        raise ValueError("packed batch too large for int32 offsets")
    cat = lambda ts, dt: torch.cat(ts) if ts else torch.zeros(0, dtype=dt)
    return (torch.tensor(rows, dtype=torch.int32).reshape(-1, 6), cat(bu, torch.int32), cat(bv, torch.int32),
            cat(masks, torch.uint8), max_atoms)


def collate_packed(complexes: List[List[HeteroGraph]], device, non_blocking=True) -> HeteroGraph:
    """One batch of several complexes: ``complexes`` is a list of pose lists (each what ``sampling`` takes as ``data_list``
    for one complex).  The result equals ``collate`` of the concatenated pose lists on ``device``, in the given order, with
    each distinct receptor uploaded once and tiled on the device (``_blocks`` on the receptor store, see
    ``_collate_receptor_blocks``), and these batch attributes:

    * ``_pose_layout``: ``(layout [n_poses, 6] int32, bond_u, bond_v, mask uint8, max_atoms)`` on the device, the
      descriptor of ddb200_pose_update_packed (``pose_layout``);
    * ``_center_node`` [n_poses]: the ligand node pose j of complex c reads in the centre convolution when
      ``fixed_center_conv=False`` - node ``lig_ptr[first pose of c] + j``, what it reads when its complex is sampled alone;
    * ``_complex_ptr`` [K + 1] and ``_complex_bond_ptr`` [K + 1]: the pose and rotatable-bond offsets of each complex."""
    if not complexes or any(len(p) == 0 for p in complexes):
        raise ValueError("collate_packed takes non-empty pose lists")
    layout, bu, bv, mask, max_atoms = pose_layout(complexes)
    out = _collate_receptor_blocks(complexes, device, non_blocking)
    if out is None:
        out = collate([d for poses in complexes for d in poses]).to(device, non_blocking=non_blocking)
    n_poses = [len(p) for p in complexes]
    pose_ptr = np.concatenate([[0], np.cumsum(n_poses)])
    first = pose_ptr[:-1]
    centre = [int(layout[f, 0]) + j for f, n in zip(first, n_poses) for j in range(n)]
    bond_ptr = [int(layout[f, 4]) for f in first] + [int(layout[-1, 4] + layout[-1, 3])]
    to = lambda t: t.to(device, non_blocking=non_blocking)
    out._pose_layout = (to(layout), to(bu), to(bv), to(mask), max_atoms)
    out._center_node = to(torch.tensor(centre, dtype=torch.long))
    out._complex_ptr = to(torch.from_numpy(pose_ptr.astype(np.int64)))
    out._complex_bond_ptr = to(torch.tensor(bond_ptr, dtype=torch.long))
    return out


def graph_to_dict(g: HeteroGraph) -> dict:
    """Plain nested dict (tensors / numpy / str) for fixtures."""
    return {'nodes': {k: dict(s.__dict__) for k, s in g._nodes.items()},
            'edges': {k: dict(s.__dict__) for k, s in g._edges.items()},
            'globals': dict(g._globals)}


def graph_from_dict(d: dict) -> HeteroGraph:
    g = HeteroGraph()
    for k, s in d['nodes'].items():
        g._nodes[k] = Store(**s)
    for k, s in d['edges'].items():
        g._edges[tuple(k)] = Store(**s)
    g._globals.update(d['globals'])
    return g
