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
    if B < 2 or not all(_same_receptor(data_list[0], d) for d in data_list[1:]):
        return collate(data_list).to(device, non_blocking=non_blocking)
    first = data_list[0]
    nts, ets = _receptor_side(first)
    if any(et[0] not in nts or et[1] not in nts for et in ets):
        return collate(data_list).to(device, non_blocking=non_blocking)
    stripped = []
    for d in data_list:                       # views without the receptor side: ligand stores are shared, not copied
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
    tile = lambda dv: dv.repeat((B,) + (1,) * (dv.dim() - 1)) if dv.dim() > 0 else dv
    n1 = {}
    for nt in nts:
        st1 = first._nodes[nt]
        n1[nt] = st1.num_nodes
        st = out[nt]
        for k in st1.keys():
            if k.startswith('_'):
                continue
            v = getattr(st1, k)
            setattr(st, k, tile(v.to(device, non_blocking=non_blocking)) if torch.is_tensor(v) else [v] * B)
        st.batch = torch.arange(B, device=device).repeat_interleave(n1[nt])
        st.ptr = torch.arange(B + 1, device=device) * n1[nt]
        own = first._edges.get((nt, nt))
        st._unique = (n1[nt], own.num_edges if own is not None else 0, B)
    for et in ets:
        st1, st = first._edges[et], out[et]
        for k in st1.keys():
            v = getattr(st1, k)
            if k == 'edge_index':
                ei = v.to(device, non_blocking=non_blocking)
                copy_id = torch.arange(B, device=device).repeat_interleave(ei.shape[1])
                off = torch.stack([copy_id * n1[et[0]], copy_id * n1[et[1]]])
                st.edge_index = ei.repeat(1, B) + off.to(ei.dtype)
            elif torch.is_tensor(v):
                setattr(st, k, tile(v.to(device, non_blocking=non_blocking)))
            else:
                setattr(st, k, [v] * B)
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
