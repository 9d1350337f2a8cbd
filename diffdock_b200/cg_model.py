"""Drop-in for the reference's coarse-grained model ``models/cg_model.py:CGModel`` in score and confidence mode.

Same constructor keywords, ``forward(data) -> (tr_pred, rot_pred, tor_pred, sidechain_pred)`` contract (confidence mode:
``(confidence, atom_confidence)``, the times used as sigmas, the head in one ddb200_confidence_head launch), ``state_dict``
keys and side effects on ``data`` (SURVEY.md section 8(b)); ``utils/sampling.py:116`` can call it unchanged.  What runs
underneath is H100-native: neighbour search and the tensor-product convolutions (SH + Clebsch-Gordan contraction +
segmented reduction + BatchNorm/residual epilogue) are hand-written sm_90a kernels behind the C ABI
(include/diffdock_b200.h); every edge list is produced already CSR-sorted by its convolution target; the score-norm
tables are device buffers (no host round trips for so3/torus look-ups).

CUDA only, inference only.  No CPU fallback.
"""
from __future__ import annotations

import math
import os

import numpy as np
import torch
from torch import nn

from . import ops
from .irreps import irreps_str, sh_irreps
from .hetero import receptor_blocks
from .layers import (AtomEncoder, GaussianSmearing, _mlp, check_confidence_widths, check_forward, confidence_head, cross_cutoff,
                     cross_graph, edge_cutoff, edge_weight, ligand_graph, score_heads)
from .synthetic import LIG_FEATURE_DIMS as lig_feature_dims, REC_RESIDUE_FEATURE_DIMS as rec_residue_feature_dims
from .tensor_layers import TensorProductConvLayer, get_irrep_seq
from .tp_table import full_tensor_product

_TABLES = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'tables', 'score_norm_tables.npz')
# utils/so3.py:6 and utils/torus.py:25-26
SO3_MIN_EPS, SO3_MAX_EPS, SO3_N_EPS = 0.0005, 4, 2000
TORUS_SIGMA_MIN, TORUS_SIGMA_MAX, TORUS_SIGMA_N = 3e-3, 2, 5000


def _i32(t):
    return t.to(torch.int32).contiguous()


def _flat(w):
    """Per-edge weights as the flat vector the kernels take; None for the scalar weight 1."""
    return w.reshape(-1).contiguous() if torch.is_tensor(w) else None


def _rr_joint(c, n_lig):
    """(target, source) of the static receptor graph as int32 in the joint numbering [ligand | residues], once per batch."""
    if n_lig not in c.setdefault('rr_tgt32', {}):
        c['rr_tgt32'][n_lig] = (_i32(c['rr_tgt'] + n_lig), _i32(c['rr_src'] + n_lig))
    return c['rr_tgt32'][n_lig]


def _block_maps(spans, dev):
    """``spans`` = [(batch offset, rows per copy, copies, distinct id)] in batch order, the copies of a span back to back:
    ``(rows, row_map, offsets)`` - the batch rows of copy 0 of each distinct id's first span, concatenated in order of first
    appearance; the distinct row of every batch row; the distinct offset of each id."""
    ar = lambda a, b: torch.arange(a, b, device=dev)
    rows, uoff, n_u = [], {}, 0
    for off, n1, _, uid in spans:
        if uid not in uoff:
            uoff[uid] = n_u
            rows.append(ar(off, off + n1))
            n_u += n1
    row_map = torch.cat([(uoff[uid] + ar(0, n1)).repeat(cp) for _, n1, cp, uid in spans])
    return torch.cat(rows), row_map, uoff


def receptor_tiles(rec, B, ei):
    """Index maps between a batch whose receptor store carries a block layout (``hetero.receptor_blocks``) and its distinct
    receptors, numbered by concatenating copy 0 of each one's first block; None without a layout.  ``nodes`` / ``edges``:
    batch rows of those copies; ``edge_index``: their contact edges in the distinct numbering; ``node_map`` [n_rec] /
    ``edge_map`` [E]: the distinct row of every batch node / edge; ``sorted_rows`` / ``sorted_shift``: the rows of the copies
    in the contact graph sorted stably by target (targets of a copy sort together, copies in batch order) and what turns
    their batch node numbers into distinct ones.  Works for any receptor-side node store with its own edges (residues and
    their contact graph, receptor atoms and the ('atom', 'atom') edges)."""
    blocks = receptor_blocks(rec, B, ei.shape[1])
    if blocks is None:
        return None
    dev = ei.device
    nodes, node_map, uoff = _block_maps([(noff, n1, cp, uid) for noff, _, n1, _, cp, uid in blocks], dev)
    edges, edge_map, _ = _block_maps([(eoff, e1, cp, uid) for _, eoff, _, e1, cp, uid in blocks], dev)
    seen, shift = set(), []
    for noff, _, _, e1, _, uid in blocks:
        if uid not in seen:
            seen.add(uid)
            shift.append(torch.full((e1,), noff - uoff[uid], dtype=torch.long, device=dev))
    shift = torch.cat(shift)
    return dict(nodes=nodes, edges=edges, edge_index=ei[:, edges] - shift, node_map=node_map, edge_map=edge_map,
                sorted_rows=edges, sorted_shift=shift)


def linked_edge_tiles(src, src_tiles, dst_tiles, ei, B):
    """Index maps of the edges between two tiled receptor-side stores (the ('atom', 'receptor') edges of all-atom graphs:
    row 0 an atom, row 1 its residue), which the block layout does not describe by itself: the batch collates them copy by
    copy in the order of the ``src`` store's blocks, so the edges of a copy are those whose row-0 node lies in it.
    ``(edges, edge_index, edge_map)`` - batch rows of copy 0 of each distinct receptor, those edges in the two stores'
    distinct numberings, the distinct row of every batch edge - or None when the batch's edges do not follow that layout.
    Two host reads (the per-graph edge counts, the check)."""
    blocks = receptor_blocks(src, B, src_tiles['edge_map'].shape[0])
    cnt = torch.bincount(src.batch[ei[0]], minlength=B).tolist() if ei.shape[1] else [0] * B
    spans, g, eoff, per_uid = [], 0, 0, {}
    for _, _, _, _, cp, uid in blocks:
        e1 = cnt[g]
        if any(c != e1 for c in cnt[g:g + cp]) or per_uid.setdefault(uid, e1) != e1:
            return None
        spans.append((eoff, e1, cp, uid))
        g, eoff = g + cp, eoff + e1 * cp
    edges, edge_map, _ = _block_maps(spans, ei.device)
    ends = torch.stack([src_tiles['node_map'][ei[0]], dst_tiles['node_map'][ei[1]]])    # every batch edge, distinct ends
    edge_index = ends[:, edges]
    if not torch.equal(edge_index[:, edge_map], ends):                  # each edge is the same edge of its copy 0
        return None
    return dict(edges=edges, edge_map=edge_map, edge_index=edge_index)


class CGModel(nn.Module):
    def __init__(self, t_to_sigma, device, timestep_emb_func, in_lig_edge_features=4, sigma_embed_dim=32, sh_lmax=2,
                 ns=16, nv=4, num_conv_layers=2, lig_max_radius=5, rec_max_radius=30, cross_max_distance=250,
                 center_max_distance=30, distance_embed_dim=32, cross_distance_embed_dim=32, no_torsion=False,
                 scale_by_sigma=True, norm_by_sigma=True, use_second_order_repr=False, batch_norm=True,
                 dynamic_max_cross=False, dropout=0.0, smooth_edges=False, odd_parity=False,
                 separate_noise_schedule=False, lm_embedding_type=None, confidence_mode=False,
                 confidence_dropout=0, confidence_no_batchnorm=False,
                 asyncronous_noise_schedule=False, affinity_prediction=False, parallel=1,
                 parallel_aggregators="mean max min std", num_confidence_outputs=1, atom_num_confidence_outputs=1,
                 fixed_center_conv=False, no_aminoacid_identities=False, include_miscellaneous_atoms=False,
                 differentiate_convolutions=True, tp_weights_layers=2, num_prot_emb_layers=0, reduce_pseudoscalars=False,
                 embed_also_ligand=False, atom_confidence=False, sidechain_pred=False, depthwise_convolution=False):
        super().__init__()
        assert parallel == 1, "not implemented"
        unsupported = dict(separate_noise_schedule=separate_noise_schedule,
                           asyncronous_noise_schedule=asyncronous_noise_schedule,
                           include_miscellaneous_atoms=include_miscellaneous_atoms, sidechain_pred=sidechain_pred,
                           depthwise_convolution=depthwise_convolution)
        bad = [k for k, v in unsupported.items() if v]
        if bad:
            raise NotImplementedError(f"{bad}: outside the hot path built so far (SURVEY.md section 8)")
        if lm_embedding_type not in (None, 'precomputed'):
            raise NotImplementedError("on-the-fly ESM embeddings are preprocessing (out of scope); use 'precomputed'")
        self.t_to_sigma, self.device, self.timestep_emb_func = t_to_sigma, device, timestep_emb_func
        self.in_lig_edge_features, self.sigma_embed_dim = in_lig_edge_features, sigma_embed_dim
        self.lig_max_radius, self.rec_max_radius = lig_max_radius, rec_max_radius
        self.cross_max_distance, self.dynamic_max_cross = cross_max_distance, dynamic_max_cross
        self.center_max_distance = center_max_distance
        self.distance_embed_dim, self.cross_distance_embed_dim = distance_embed_dim, cross_distance_embed_dim
        self.sh_lmax = sh_lmax
        self.sh_irreps = irreps_str(sh_irreps(sh_lmax))
        self.ns, self.nv = ns, nv
        self.scale_by_sigma, self.norm_by_sigma = scale_by_sigma, norm_by_sigma
        self.no_torsion, self.smooth_edges, self.odd_parity = no_torsion, smooth_edges, odd_parity
        self.confidence_mode, self.affinity_prediction = confidence_mode, affinity_prediction
        self.atom_confidence, self.atom_num_confidence_outputs = atom_confidence, atom_num_confidence_outputs
        self.num_conv_layers, self.num_prot_emb_layers = num_conv_layers, num_prot_emb_layers
        self.fixed_center_conv, self.no_aminoacid_identities = fixed_center_conv, no_aminoacid_identities
        self.differentiate_convolutions, self.reduce_pseudoscalars = differentiate_convolutions, reduce_pseudoscalars
        self.embed_also_ligand = embed_also_ligand
        self.lm_embedding_type = lm_embedding_type
        lm_dim = 1280 if lm_embedding_type == 'precomputed' else 0
        S, D, Dx = sigma_embed_dim, distance_embed_dim, cross_distance_embed_dim

        self.lig_node_embedding = AtomEncoder(emb_dim=ns, feature_dims=lig_feature_dims, sigma_embed_dim=S)
        self.lig_edge_embedding = _mlp(in_lig_edge_features + S + D, ns, ns, dropout)
        self.rec_node_embedding = AtomEncoder(emb_dim=ns, feature_dims=rec_residue_feature_dims, sigma_embed_dim=0,
                                              lm_embedding_dim=lm_dim)
        self.rec_edge_embedding = _mlp(D, ns, ns, dropout)
        self.rec_sigma_embedding = _mlp(S, ns, ns, dropout)
        self.cross_edge_embedding = _mlp(S + Dx, ns, ns, dropout)
        self.lig_distance_expansion = GaussianSmearing(0.0, lig_max_radius, D)
        self.rec_distance_expansion = GaussianSmearing(0.0, rec_max_radius, D)
        self.cross_distance_expansion = GaussianSmearing(0.0, cross_max_distance, Dx)

        self._irrep_seq = get_irrep_seq(ns, nv, use_second_order_repr, reduce_pseudoscalars)
        self._conv_kw = dict(sh_irreps=self.sh_irreps, n_edge_features=3 * ns, hidden_features=3 * ns, residual=True,
                             batch_norm=batch_norm, dropout=dropout, faster=sh_lmax == 1 and not use_second_order_repr,
                             tp_weights_layers=tp_weights_layers)
        self.rec_emb_layers = nn.ModuleList([self.conv(i, 1) for i in range(num_prot_emb_layers)])
        if embed_also_ligand:
            self.lig_emb_layers = nn.ModuleList([self.conv(i, 1) for i in range(num_prot_emb_layers)])
        self.conv_layers = self._interaction_stack(4, 2)
        self._sync_free = None
        # the sync-free forward drops receptor <- receptor messages that cannot reach a ligand atom (_pruned_contact_groups);
        # False runs every contact edge in every layer, for comparisons only
        self._prune_receptor = True
        if confidence_mode:
            self._confidence_heads(confidence_dropout, confidence_no_batchnorm, num_confidence_outputs)
            return

        # translation / rotation head
        self.center_distance_expansion = GaussianSmearing(0.0, center_max_distance, D)
        self.center_edge_embedding = _mlp(D + S, ns, ns, dropout)
        self.final_conv = TensorProductConvLayer(in_irreps=self.conv_layers[-1].out_irreps, sh_irreps=self.sh_irreps,
                                                 out_irreps='2x1o + 2x1e' if not odd_parity else '1x1o + 1x1e',
                                                 n_edge_features=2 * ns, residual=False, dropout=dropout,
                                                 batch_norm=batch_norm)
        self.tr_final_layer = nn.Sequential(nn.Linear(1 + S, ns), nn.Dropout(dropout), nn.ReLU(), nn.Linear(ns, 1))
        self.rot_final_layer = nn.Sequential(nn.Linear(1 + S, ns), nn.Dropout(dropout), nn.ReLU(), nn.Linear(ns, 1))
        if not no_torsion:
            self.final_edge_embedding = _mlp(D, ns, ns, dropout)
            T, tor_sh = full_tensor_product(self.sh_irreps, '1x2e')       # o3.FullTensorProduct(sh, "2e"), :240
            self.register_buffer('_tor_tp', torch.from_numpy(T).float(), persistent=False)
            self.tor_bond_conv = TensorProductConvLayer(in_irreps=self.conv_layers[-1].out_irreps,
                                                        sh_irreps=irreps_str(tor_sh),
                                                        out_irreps=f'{ns}x0o + {ns}x0e' if not odd_parity else f'{ns}x0o',
                                                        n_edge_features=3 * ns, residual=False, dropout=dropout,
                                                        batch_norm=batch_norm)
            self.tor_final_layer = nn.Sequential(nn.Linear(2 * ns if not odd_parity else ns, ns, bias=False), nn.Tanh(),
                                                 nn.Dropout(dropout), nn.Linear(ns, 1, bias=False))
        # score-norm tables (utils/so3.py:59, utils/torus.py:72-76) as device buffers; not part of the state_dict
        z = np.load(_TABLES)
        self.register_buffer('_so3_table', torch.from_numpy(z['so3_exp_score_norms']).float(), persistent=False)
        self.register_buffer('_torus_table', torch.from_numpy(z['torus_score_norm']).float(), persistent=False)

    def _confidence_heads(self, dropout, no_batchnorm, num_confidence_outputs):
        """``atom_confidence_predictor`` (with atom_confidence) and ``confidence_predictor`` (models/cg_model.py:181-208 =
        models/aa_model.py:177-211).  The pooled input is the first ns columns of the ligand features and, after three or
        more convolutions in all (embedding + interaction layers), the last nv (reduce_pseudoscalars) or ns columns."""
        ns = self.ns
        self._conf_tail = (self.nv if self.reduce_pseudoscalars else ns) \
            if self.num_conv_layers + self.num_prot_emb_layers >= 3 else 0
        n_in = ns + self._conf_tail

        def head(i, o):
            bn = (lambda: nn.Identity()) if no_batchnorm else (lambda: nn.BatchNorm1d(ns))
            return nn.Sequential(nn.Linear(i, ns), bn(), nn.ReLU(), nn.Dropout(dropout), nn.Linear(ns, ns), bn(), nn.ReLU(),
                                 nn.Dropout(dropout), nn.Linear(ns, o))
        if self.atom_confidence:
            self.atom_confidence_predictor = head(n_in, self.atom_num_confidence_outputs + ns)
            n_in = ns
        self.confidence_predictor = head(n_in, num_confidence_outputs + (1 if self.affinity_prediction else 0))
        check_confidence_widths(self)

    def conv(self, i, groups):
        """Convolution ``i`` of the stack (protein embedding layers first) with ``groups`` radial MLPs."""
        seq = self._irrep_seq
        return TensorProductConvLayer(in_irreps=seq[min(i, len(seq) - 1)], out_irreps=seq[min(i + 1, len(seq) - 1)],
                                      edge_groups=groups, **self._conv_kw)

    def _interaction_stack(self, groups, last_groups):
        """The interaction layers: ``groups`` radial MLPs per layer, ``last_groups`` in the last one, one without
        differentiate_convolutions."""
        P, L = self.num_prot_emb_layers, self.num_conv_layers
        return nn.ModuleList([self.conv(i, 1 if not self.differentiate_convolutions else
                                        (last_groups if i == P + L - 1 else groups)) for i in range(P, P + L)])

    # ---------------------------------------------------------------------------------------------------------
    def load_state_dict(self, state_dict, strict=True, **kw):
        """Accepts reference checkpoints: e3nn's TensorProduct modules register buffers (``*.tp.weight``,
        ``*.tp.output_mask``, ``final_tp_tor.*``, compiled ``_w3j_*`` constants) that have no counterpart here."""
        drop = [k for k in state_dict if '.tp.' in k or k.startswith('final_tp_tor.') or '_w3j' in k]
        if drop:
            state_dict = {k: v for k, v in state_dict.items() if k not in drop}
        return super().load_state_dict(state_dict, strict=strict, **kw)

    def set_score_norm_tables(self, so3_exp_score_norms, torus_score_norm):
        """Install the tables of the caller's reference installation (torus.score_norm_ is a Monte-Carlo estimate that
        differs per machine, SURVEY.md section 5)."""
        self._so3_table.copy_(torch.as_tensor(so3_exp_score_norms, dtype=torch.float32))
        self._torus_table.copy_(torch.as_tensor(torus_score_norm, dtype=torch.float32))

    # ---------------------------------------------------------------------------------------------------------
    def get_edge_weight(self, edge_vec, max_norm):
        return edge_weight(edge_vec, max_norm, self.smooth_edges)

    def _so3_score_norm(self, eps):
        """utils/so3.py:89-93 evaluated on the device (fp32 index arithmetic, round-half-even like np.around)."""
        lo, hi = math.log10(SO3_MIN_EPS), math.log10(SO3_MAX_EPS)
        idx = (torch.log10(eps.float()) - np.float32(lo)) / np.float32(hi - lo) * SO3_N_EPS
        idx = torch.round(idx).clamp(0, SO3_N_EPS - 1).long()
        return self._so3_table[idx]

    def _torus_score_norm(self, sigma):
        """utils/torus.py:79-83 on the device."""
        lo, hi = math.log(TORUS_SIGMA_MIN), math.log(TORUS_SIGMA_MAX)
        s = torch.log(sigma.float() / np.float32(np.pi))
        s = (s - np.float32(lo)) / np.float32(hi - lo) * TORUS_SIGMA_N
        s = torch.round(s.clamp(0, TORUS_SIGMA_N)).long()
        return self._torus_table[s]

    # ---------------------------------------------------------------------------------------------------------
    def _static(self, data):
        """Pose-independent quantities, cached on ``data`` like the reference does (models/cg_model.py:273,292-295)."""
        rec, rr, lig, ll = data['receptor'], data['receptor', 'receptor'], data['ligand'], data['ligand', 'ligand']
        if hasattr(rec, 'rec_node_attr') and hasattr(rr, '_b200'):
            return rr._b200
        B = data.num_graphs
        c = {}
        ei = rr.edge_index.long()
        # copies of the same receptor (N poses of one complex, inference.py:236-239, or several ligands against one protein
        # in a packed batch): embed each distinct receptor ONCE and tile the result; the reference recomputes the identical
        # 1280-wide embedding for every pose of the batch (models/cg_model.py:272-295)
        tiles = receptor_tiles(rec, B, ei)
        c['tiles'] = tiles
        if tiles is None:
            x1, pos1, ei1 = rec.x, rec.pos, ei
        else:
            x1, pos1, ei1 = rec.x[tiles['nodes']], rec.pos[tiles['nodes']], tiles['edge_index']
        vec = (pos1[ei1[1]] - pos1[ei1[0]]).float()
        rec_edge_attr = self.rec_edge_embedding(self.rec_distance_expansion(vec.norm(dim=-1)))
        rec_node_attr = self.rec_node_embedding(x1)
        if self.rec_emb_layers:     # input of the embedding layers: a cropped step runs them over its own contact graph
            c['rec_node_pre'] = rec_node_attr[tiles['node_map']] if tiles is not None else rec_node_attr
        ew = self.get_edge_weight(vec, self.rec_max_radius)
        for layer in self.rec_emb_layers:
            ea_ = torch.cat([rec_edge_attr, rec_node_attr[ei1[0], :self.ns], rec_node_attr[ei1[1], :self.ns]], -1)
            rec_node_attr = layer(rec_node_attr, ei1, ea_, None, edge_weight=ew, edge_vec=vec)
        if tiles is not None:
            em = tiles['edge_map']
            vec, rec_edge_attr, rec_node_attr = vec[em], rec_edge_attr[em], rec_node_attr[tiles['node_map']]
            ew = ew[em] if torch.is_tensor(ew) else ew
        rec.rec_node_attr, rr.rec_edge_attr, rr.edge_weight = rec_node_attr, rec_edge_attr, ew
        rr.edge_sh = None   # evaluated inside the convolution kernel from the edge vectors; kept for attribute parity
        # CSR order of the static receptor graph (target = edge_index[0])
        tgt, order = torch.sort(ei[0], stable=True)
        c['rr_tgt'], c['rr_src'] = tgt, ei[1][order]
        c['rr_vec'] = vec[order].contiguous()
        c['rr_ea'] = rec_edge_attr[order].contiguous()
        c['rr_ew'] = ew[order].contiguous() if torch.is_tensor(ew) else None
        c['rr_tgt_batch'] = rec.batch[tgt]
        c['rec_ptr'] = ops.segment_ptr(rec.batch, B)
        c['lig_ptr'] = ops.segment_ptr(lig.batch, B)
        # rotatable bonds are static too
        mask = lig.edge_mask
        bonds = ll.edge_index[:, mask].long()
        c['bonds'], c['n_bonds'] = bonds, int(bonds.shape[1])
        c['bond_batch'] = lig.batch[bonds[0]] if bonds.shape[1] else None
        self._static_sync_free(data, c)
        rr._b200 = c
        return c

    def _static_sync_free(self, data, c):
        """Per-batch constants of the sync-free forward: node counts, the bond edges as a CSR by target atom, capacities of
        the per-step edge buffers (upper bounds that hold for ANY pose), int32 views.  One host read per batch."""
        rec, lig, ll = data['receptor'], data['ligand'], data['ligand', 'ligand']
        B, dev = data.num_graphs, lig.pos.device
        n_lig, n_rec = lig.batch.shape[0], rec.batch.shape[0]
        lig_cnt = (c['lig_ptr'][1:] - c['lig_ptr'][:-1])
        rec_cnt = (c['rec_ptr'][1:] - c['rec_ptr'][:-1])
        host = torch.stack([lig_cnt, rec_cnt]).cpu()                       # the one host read of the batch
        c['lig_cnt_f'] = lig_cnt.float().unsqueeze(1)
        c['rec_max'] = int(host[1].max()) if B else 0
        c['cap_cross'] = int((host[0].long() * host[1].long()).sum())      # every ligand atom x every residue of its complex
        c['lig_batch32'], c['rec_batch32'] = _i32(lig.batch), _i32(rec.batch)
        c['rr_gid32'] = _i32(c['rr_tgt_batch'])
        # bond edges sorted by their convolution target (edge_index[0]), original order kept inside a target
        ei = ll.edge_index.long()
        order = torch.sort(ei[0], stable=True).indices
        c['pre_tgt'], c['pre_col'] = _i32(ei[0][order]), _i32(ei[1][order])
        attr = ll.edge_attr.float()[order] if ei.shape[1] else torch.zeros((0, self.in_lig_edge_features), device=dev)
        c['pre_attr'] = torch.cat([attr, torch.zeros((1, attr.shape[1]), device=dev)], 0)     # row -1: "not a bond"
        # radius_graph(max_num_neighbors=32) = radius with cap 33 minus the self hit: a centre atom whose own index is not
        # among its first 33 hits keeps 33 neighbours
        c['cap_ll'] = int(ei.shape[1]) + 33 * n_lig
        c['bond_lig_batch'] = lig.batch[c['bonds'][0]] if c['n_bonds'] else None
        c['cap_tor'] = 32 * c['n_bonds']
        c['bond_batch32'] = _i32(c['bond_batch']) if c['n_bonds'] else None

    def _ligand_graph(self, data, c):
        """Bond edges + radius graph, sorted stably by convolution target (models/cg_model.py:467-497)."""
        tgt, src, attr, vec, ew, node = ligand_graph(self, data, c['lig_ptr'])
        tgt, order = torch.sort(tgt, stable=True)
        return node, tgt, src[order], attr[order], vec[order], ew[order] if torch.is_tensor(ew) else ew

    # ---------------------------------------------------------------------------------------------------------
    def sync_free_capable(self):
        """The forward can run without any host synchronisation (and so inside a CUDA graph) when every convolution of the
        stack has a shape the fully fused kernel supports; otherwise the neighbour-list sizes go through the host."""
        if self._sync_free is None:
            ok = os.environ.get('DDB200_SYNC_FREE', '1') != '0'
            ok = ok and self.embed_also_ligand
            for layer in list(self.conv_layers) + list(getattr(self, 'lig_emb_layers', [])):
                ok = ok and layer.fused_capable(self.ns, self.ns)
            self._sync_free = bool(ok)
        return self._sync_free

    def sync_free_crop_capable(self):
        """The sync-free forward can also crop the receptor per step (``data._crop``, set by the sampler's graphed step): the
        receptor embedding layers then run on every step over the cropped contact graph, so they need the fused kernel too."""
        return self.sync_free_capable() and all(layer.fused_capable(self.ns, self.ns) for layer in self.rec_emb_layers)

    @torch.no_grad()
    def forward(self, data):
        check_forward(self, data)
        c = self._static(data)
        # the cap of the cross graphs (models/cg_model.py:546, models/aa_model.py:595,610) must not bind
        if self.sync_free_capable() and max(c['rec_max'], c.get('atom_max', 0)) <= 10000:
            return self._forward_sync_free(data, c)
        if getattr(data, '_crop', None) is not None:
            raise RuntimeError("per-step receptor cropping (data._crop) runs on the sync-free forward only, which this "
                               "batch cannot take (more than 10000 residues in a complex)")
        return self._forward_host_sized(data, c)

    def _interaction_layers(self, node, groups, n_last, merge=False, shared=None, per_layer=None):
        """The interaction layers over the joint graph; the last one only takes the first ``n_last`` groups, the edges that
        end on ligand atoms (models/cg_model.py:347-349).  ``merge``: one radial MLP for all edge types runs them as a
        single group (exactly-sized lists only).  ``shared = (accumulators, k)``: layer 0 starts from messages computed
        elsewhere instead of running group ``k`` (an int, or a tuple of group indices).  ``per_layer = (k, [group | None per
        layer])``: layer l runs the given group in place of group ``k`` where one is given."""
        L = len(self.conv_layers)
        for l, layer in enumerate(self.conv_layers):
            use, init = (groups if l < L - 1 else groups[:n_last]), None
            if per_layer is not None and per_layer[1][l] is not None:
                k = per_layer[0]
                use = use[:k] + [per_layer[1][l]] + use[k + 1:]
            if l == 0 and shared is not None:
                init, skip = shared
                skip = (skip,) if isinstance(skip, int) else skip
                use = [None if k in skip else g for k, g in enumerate(use)]
            if merge:
                use = [tuple(torch.cat([g[k] for g in use]) if use[0][k] is not None else None for k in range(5))]
            node = layer.forward_groups(node, use, gather_scalars=self.ns, init=init)
        return node

    # ---------------------------------------------------------------------------------------------------------
    def _forward_sync_free(self, data, c):
        """The whole forward without a device->host read: every per-step neighbour list is written into an upper-bound
        buffer by ddb200_graph_fill with its live length kept in device memory, the reverse direction of the cross graph is
        an index permutation of the forward one, the ligand-receptor edge embedding is one kernel, and the convolutions
        take (capacity, device count).  Shapes are static for a given batch, so a reverse-diffusion step can be captured in
        a CUDA graph (diffdock_b200/sampling.py)."""
        lig, rec = data['ligand'], data['receptor']
        ns, n_lig = self.ns, lig.batch.shape[0]
        tr_sigma, rot_sigma, tor_sigma = self._sigmas(data)

        # -- embeddings (models/cg_model.py:272-306) --------------------------------------------------------------
        sig = self.rec_sigma_embedding(self.timestep_emb_func(data.complex_t['tr'])).contiguous()      # [B, ns]
        crop = getattr(data, '_crop', None)
        prune = self._prune_receptor and len(self.conv_layers) > 1
        keep = None
        if crop is None:
            rec_node, rec_pos = rec.rec_node_attr.clone(), rec.pos.float().contiguous()
            rr_tgt32 = _rr_joint(c, n_lig)
            g_rr = (rr_tgt32[0], rr_tgt32[1], c['rr_ea'], c['rr_vec'], _flat(c['rr_ew']),
                    dict(ea_add=sig, ea_add_idx=c['rr_gid32']))
        else:
            rec_node, rec_pos, g_rr, keep = self._cropped_receptor(data, c, crop, sig, n_lig, select=not prune)
        rec_node[:, :ns] += sig[rec.batch]
        lig_node, g_ll = self._ligand_graph_sync_free(data, c)

        # -- cross graph, both directions (:321-327, :539-562) ------------------------------------------------------------
        r, rpg = cross_cutoff(self, tr_sigma)
        g_lr, g_rl = self._cross_graph_sync_free(data, c, rec_pos, c['rec_ptr'], c['rec_batch32'],
                                                 c['rec_max'], c['cap_cross'], r, rpg, n_lig, self.cross_edge_embedding,
                                                 self.cross_distance_expansion, vec_sign=-1.0)

        # -- joint graph: four edge groups (:329-338) ---------------------------------------------------------------
        node = torch.cat([lig_node, rec_node], 0)
        groups = [g_ll,                                                                                   # lig <- lig
                  g_lr,                                                                                   # lig <- rec
                  g_rr,                                                                                   # rec <- rec
                  g_rl]                                                                                   # rec <- lig, Y(-v)
        # the shared layer-0 messages assume every pose keeps every residue
        shared = self._shared_receptor_messages(data, c, rec, rec_node, sig, n_lig) \
            if len(self.conv_layers) > 1 and crop is None else None
        pruned = self._pruned_contact_groups(c, g_rl, keep, sig, n_lig, rec_node.shape[0], shared is not None) \
            if prune else None
        node = self._interaction_layers(node, groups, 2, shared=(shared, 2) if shared is not None else None,
                                        per_layer=(2, pruned) if pruned is not None else None)
        return self._heads(data, c, node[:n_lig], tr_sigma, rot_sigma, tor_sigma, sync_free=True)

    def _need_levels(self, L, shared):
        """Per interaction layer l, the k of the need set R_k its receptor <- receptor group is restricted to, or None: the
        last layer has no such group, and layer 0 keeps the shared messages when they apply.  Layer l's output reaches the
        ligand through L - 1 - l more layers, one contact hop each, the last of which ends on ligand atoms."""
        return [None if l == L - 1 or (l == 0 and shared) else L - 1 - l for l in range(L)]

    def _pruned_contact_groups(self, c, g_rl, keep, sig, n_lig, n_rec, shared):
        """The receptor <- receptor group of every interaction layer restricted to targets that can still pass a message to
        a ligand atom (None where the layer keeps its group).  Only the ligand's final features reach the outputs, so a
        residue's features after layer l matter only through a chain of messages into the ligand in layers l+1 .. L-1:
        R_1 = the targets of this step's receptor <- ligand edges (g_rl, the edges the convolutions use), R_{k+1} = R_k and
        the sources of the contact edges into R_k (under a crop, only the edges whose two ends are kept), and layer l needs
        its targets in R_{L-1-l}.

        Invariant: a residue outside layer l's set gets no contact messages in that layer, so its row of the layer output
        is wrong, and no later layer or head reads it - the contact and receptor -> ligand messages of later layers only
        gather from R_{L-1-l} (the ligand graph, the cross groups and the heads never see other residues).  Every buffer
        lives in ``c``, so a captured step allocates nothing."""
        levels = self._need_levels(len(self.conv_layers), shared)
        n_levels = max((k for k in levels if k is not None), default=0)
        if n_levels == 0:
            return None
        if 'rr_tgt32l' not in c:
            c['rr_tgt32l'] = (_i32(c['rr_tgt']), _i32(c['rr_src']))
        tgt32, src32 = c['rr_tgt32l']
        key = ('prune', n_lig, n_levels)
        if key not in c:
            c[key] = (torch.empty((n_levels, n_rec), dtype=torch.uint8, device=tgt32.device),
                      [ops.select_edges_buffers(tgt32.shape[0], tgt32.device) for _ in range(n_levels)])
        need_buf, bufs = c[key]
        need = ops.receptor_need(g_rl[0], g_rl[5]['n_edges_dev'], n_lig, tgt32, src32, n_rec, n_levels, keep=keep,
                                 out=need_buf)
        ew, sel = _flat(c['rr_ew']), {}
        for k in sorted({k for k in levels if k is not None}):
            t, s_, perm, gid, n_dev = ops.crop_select_edges(tgt32, src32, keep, c['rr_gid32'], offset=n_lig,
                                                            need=need[k - 1], out=bufs[k - 1])
            sel[k] = (t, s_, c['rr_ea'], c['rr_vec'], ew,
                      dict(n_edges_dev=n_dev, edge_perm=perm, ea_add=sig, ea_add_idx=gid))
        return [sel[k] if k is not None else None for k in levels]

    def _cropped_receptor(self, data, c, crop, sig, n_lig, select=True):
        """utils/sampling.py:104-109 in masked form: the residues farther than the step's cut-off from every ligand atom of
        their complex keep their rows but lose every edge.  ``crop = (cutoff2_table, step_dev)``.  Returns the receptor node
        features (the embedding layers rerun over the cropped contact graph, as the reference embeds its cropped batch),
        the positions for the cross-graph search (+inf at dropped residues), the rec <- rec edge group (None when
        ``select`` is False and no embedding layer needs it: the pruned layers select their own) and the keep flags."""
        if not self.sync_free_crop_capable():
            raise RuntimeError("per-step receptor cropping needs every receptor embedding layer on the fused kernel "
                               "(CGModel.sync_free_crop_capable)")
        lig, rec = data['ligand'], data['receptor']
        keep, rec_pos = ops.crop_flags(lig.pos.float().contiguous(), c['lig_ptr'], rec.pos.float().contiguous(),
                                       c['rec_batch32'], crop[0], crop[1])
        if 'rr_tgt32l' not in c:
            c['rr_tgt32l'] = (_i32(c['rr_tgt']), _i32(c['rr_src']))
        if not select and not len(self.rec_emb_layers):
            return rec.rec_node_attr.clone(), rec_pos, None, keep
        tgt, src, perm, gid, n_dev = ops.crop_select_edges(*c['rr_tgt32l'], keep, c['rr_gid32'], offset=n_lig)
        ew = _flat(c['rr_ew'])
        if len(self.rec_emb_layers):
            node = c['rec_node_pre']
            g = (tgt - n_lig, src - n_lig, c['rr_ea'], c['rr_vec'], ew, dict(n_edges_dev=n_dev, edge_perm=perm))
            for layer in self.rec_emb_layers:
                node = layer.forward_groups(node, [g], gather_scalars=self.ns)
        else:
            node = rec.rec_node_attr.clone()
        g_rr = (tgt, src, c['rr_ea'], c['rr_vec'], ew, dict(n_edges_dev=n_dev, edge_perm=perm, ea_add=sig, ea_add_idx=gid))
        return node, rec_pos, g_rr, keep

    def _ligand_graph_sync_free(self, data, c):
        """Bonds + radius graph, CSR by target, built on the device (models/cg_model.py:467-497), and the ligand embedding
        layers over it: ``(ligand node features, edge group)``."""
        lig = data['ligand']
        g = self._ligand_edges_sync_free(data, c)
        node = self.lig_node_embedding(torch.cat([lig.x.float(), lig.node_sigma_emb], 1))
        for layer in self.lig_emb_layers:
            node = layer.forward_groups(node, [g], gather_scalars=self.ns)
        return node, g

    def _ligand_edges_sync_free(self, data, c):
        """The edge group of the ligand graph (bonds + radius graph, CSR by target) in a capacity buffer; sets
        ``node_sigma_emb`` on the ligand.

        radius_graph caps the neighbours of each CENTRE atom at 32, and its edges point from the centre to the neighbour,
        which is the convolution's target (edge_index = [neighbour, centre], models/cg_model.py:478-483).  Where the cap
        binds, an atom can be the target of more than 32 edges, so the search runs per centre and the pairs are then
        sorted by target: the bonds of each target first (in their original order), then its radius edges by centre, the
        order of the reference's concatenation sorted stably by target."""
        lig = data['ligand']
        pos = lig.pos.float().contiguous()
        n_lig = pos.shape[0]
        lig.node_sigma_emb = self.timestep_emb_func(lig.node_t['tr'])
        cnt = ops.radius_count(pos, pos, c['lig_ptr'], c['lig_batch32'], r=self.lig_max_radius, max_num_neighbors=33,
                               exclude_self=True)
        incl = torch.cumsum(cnt, 0, dtype=torch.int32)
        n_b = c['pre_col'].shape[0]
        centre, nbr, _, _, _ = ops.graph_fill(
            pos, pos, c['lig_ptr'], c['lig_batch32'], (incl - cnt).contiguous(), c['cap_ll'] - n_b, r=self.lig_max_radius,
            max_num_neighbors=33, exclude_self=True, want_vec=False, fill_row=0)
        # rows past the live count get the key n_lig, so that they sort last
        live = torch.arange(centre.shape[0], dtype=torch.int32, device=pos.device) < incl[-1:]
        key = torch.cat([c['pre_tgt'], torch.where(live, nbr, n_lig)])
        tgt, perm, _ = ops.csr_sort_by_target(key.contiguous(), n_lig + 1)
        src = torch.cat([c['pre_col'], centre])[perm].contiguous()
        eid = torch.cat([torch.arange(n_b, device=pos.device), torch.full_like(centre, -1, dtype=torch.long)])[perm]
        tgt = torch.where(tgt < n_lig, tgt, 0).contiguous()              # padded rows: any valid node
        vec = (pos[src.long()] - pos[tgt.long()]).contiguous()
        attr = torch.cat([c['pre_attr'][eid], lig.node_sigma_emb[tgt.long()],
                          self.lig_distance_expansion(vec.norm(dim=-1))], 1)
        return (tgt, src, self.lig_edge_embedding(attr), vec, _flat(self.get_edge_weight(vec, self.lig_max_radius)),
                dict(n_edges_dev=incl[-1:] + n_b))

    def _cross_graph_sync_free(self, data, c, xpos, x_ptr, x_batch32, x_max, cap, r, rpg, col_off, mlp, gs, vec_sign):
        """Ligand <- x edges (x: residues or receptor atoms at ``xpos``, numbered from ``col_off`` in the joint graph) in a
        capacity buffer, and the x <- ligand direction as a permutation of them with the edge vector times ``vec_sign``:
        ``(forward group, reverse group)`` (models/cg_model.py:539-562)."""
        lig = data['ligand']
        pos = lig.pos.float().contiguous()
        n_lig = pos.shape[0]
        cnt = ops.radius_count(xpos, pos, x_ptr, c['lig_batch32'], r=r, r_per_graph=rpg, max_num_neighbors=10000)
        incl = torch.cumsum(cnt, 0, dtype=torch.int32)
        n_dev = incl[-1:]
        # the reverse search below has no cap and reads each pair's forward position from slot[ligand atom, x], so it is
        # only right while the forward cap cannot bind; past that the reverse list is the forward one sorted by x
        slot = torch.empty((n_lig, max(x_max, 1)), dtype=torch.int32, device=pos.device) if x_max <= 10000 else None
        # rows beyond the live count must be valid (zero) when library ops gather over the whole buffer: the smooth edge
        # weight, or the embedding MLP when its shape is outside the edge-embedding kernel's templates
        padded_valid = self.smooth_edges or not self._edge_embed_in_kernel(mlp, gs)
        f_tgt, f_src, vec, _, _ = ops.graph_fill(
            xpos, pos, x_ptr, c['lig_batch32'], (incl - cnt).contiguous(), cap, r=r, r_per_graph=rpg,
            max_num_neighbors=10000, slot_out=slot, slot_ld=slot.shape[1] if slot is not None else 0, col_offset=col_off,
            fill_row=0 if padded_valid else None)
        if slot is not None:
            cnt_r = ops.radius_count(pos, xpos, c['lig_ptr'], x_batch32, r=r, r_per_graph=rpg, max_num_neighbors=1 << 30)
            incl_r = torch.cumsum(cnt_r, 0, dtype=torch.int32)
            b_tgt, b_src, _, _, perm = ops.graph_fill(
                pos, xpos, c['lig_ptr'], x_batch32, (incl_r - cnt_r).contiguous(), cap, r=r, r_per_graph=rpg,
                max_num_neighbors=1 << 30, want_vec=False, slot_in=slot, y_ptr=x_ptr, slot_ld=slot.shape[1], want_perm=True,
                row_offset=col_off)
        else:
            # stable sort by the x end; rows past the live count get a key above every x, so they sort last
            n_rows = col_off + xpos.shape[0]
            live = torch.arange(f_src.shape[0], dtype=torch.int32, device=pos.device) < n_dev
            b_tgt, perm, _ = ops.csr_sort_by_target(torch.where(live, f_src, n_rows), n_rows + 1)
            b_src, perm = f_tgt[perm], perm.int()
        ea = self._cross_edge_embedding(lig.node_sigma_emb, vec, f_tgt, n_dev, mlp, gs)
        ew = None
        if self.smooth_edges:
            ew = _flat(self.get_edge_weight(vec, edge_cutoff(r, rpg, lig.batch, f_tgt.long())))
        return ((f_tgt, f_src, ea, vec, ew, dict(n_edges_dev=n_dev)),
                (b_tgt, b_src, ea, vec, ew, dict(n_edges_dev=n_dev, edge_perm=perm, vec_sign=vec_sign)))

    def _shared_receptor_messages(self, data, c, rec, rec_node, sig, n_lig):
        """Layer-0 receptor<-receptor messages when the batch holds copies of the same receptors (``c['tiles']``) at ONE
        diffusion time: the residue features entering the first interaction layer (static embedding + sigma embedding) and
        the contact graph are then the same in every copy of a receptor, so the messages are computed once per distinct
        receptor - one accumulation over the concatenated copy-0 graphs - and added to all copies' accumulators.  The
        reference recomputes them per pose (models/cg_model.py:342-349 over the B-fold receptor).  Needs the sampler's
        promise that all graphs of the batch share t (``data._uniform_t``; the model API allows per-graph times)."""
        tiles = c['tiles']
        if tiles is None or not getattr(data, '_uniform_t', False) or not self.differentiate_convolutions:
            return None
        n_u = tiles['nodes'].shape[0]
        if n_u == rec_node.shape[0]:
            return None                        # no receptor repeats: nothing to share
        layer = self.conv_layers[0]
        if 'rr0' not in c:          # copy 0 of each distinct receptor's CSR-sorted contact graph, numbered as tiles['nodes']
            rows = tiles['sorted_rows']
            c['rr0'] = (_i32(c['rr_tgt'][rows] - tiles['sorted_shift']), _i32(c['rr_src'][rows] - tiles['sorted_shift']),
                        c['rr_ea'][rows].contiguous(), c['rr_vec'][rows].contiguous(),
                        _flat(c['rr_ew'][rows]) if c['rr_ew'] is not None else None)
        t0, s0, ea0, vec0, ew0 = c['rr0']
        zero_idx = c.setdefault('rr0_zero', torch.zeros(t0.shape[0], dtype=torch.int32, device=ea0.device))
        g0 = (t0, s0, ea0, vec0, ew0, dict(ea_add=sig[:1].contiguous(), ea_add_idx=zero_idx))
        sum0, cnt0 = layer.accumulate_group(rec_node[tiles['nodes']], g0, 2, n_u, gather_scalars=self.ns)
        N = n_lig + rec_node.shape[0]
        sum_buf, cnt_buf = ops.new_accumulators(N, layer.out_size, sum0.device)
        sum_buf[n_lig:].add_(sum0[tiles['node_map']])
        cnt_buf[n_lig:].add_(cnt0[tiles['node_map']])
        return sum_buf, cnt_buf

    def _edge_embed_in_kernel(self, mlp, gs):
        return (gs.offset.shape[0], self.ns) in ops.EDGE_EMBED_SHAPES and len(mlp) == 4

    def _cross_edge_embedding(self, node_sigma_emb, vec, row, n_dev, mlp, gs):
        """``mlp(cat[sigma_emb[lig], gs(d)])`` (models/cg_model.py:326,553-554): the sigma half of the first Linear is
        applied per ligand NODE, the rest per edge in one kernel (ddb200_edge_embed)."""
        l1, l2 = mlp[0], mlp[-1]
        S = node_sigma_emb.shape[1]
        if self._edge_embed_in_kernel(mlp, gs):
            u = torch.addmm(l1.bias, node_sigma_emb, l1.weight[:, :S].t()).contiguous()
            return ops.edge_embed(vec, row, u, l1.weight[:, S:].contiguous(), l2.weight.contiguous(), l2.bias.contiguous(),
                                  gs.offset.contiguous(), float(gs.coeff), n_dev)
        attr = torch.cat([node_sigma_emb[row.long()], gs(vec.norm(dim=-1))], 1)      # library path on the padded buffer
        return mlp(attr)

    # ---------------------------------------------------------------------------------------------------------
    def _forward_host_sized(self, data, c):
        """Forward with exactly-sized neighbour lists (one host read of each edge count): convolution shapes outside the
        fused kernel's templates, or more than 10000 residues per complex."""
        rec, ns = data['receptor'], self.ns
        tr_sigma, rot_sigma, tor_sigma = self._sigmas(data)

        # -- embeddings (models/cg_model.py:272-306) --------------------------------------------------------------
        sig = self.rec_sigma_embedding(self.timestep_emb_func(data.complex_t['tr']))
        rec_node = rec.rec_node_attr.clone()
        rec_node[:, :ns] += sig[rec.batch]
        rr_ea = c['rr_ea'] + sig[c['rr_tgt_batch']]
        lig_x, ll_tgt, ll_src, ll_ea, ll_vec, ll_ew = self._ligand_graph(data, c)
        lig_node = self.lig_node_embedding(lig_x)
        ll_ea = self.lig_edge_embedding(ll_ea)
        assert self.embed_also_ligand, "otherwise reimplement padding"
        ll_ei = torch.stack([ll_tgt, ll_src])
        for layer in self.lig_emb_layers:
            ea_ = torch.cat([ll_ea, lig_node[ll_tgt, :ns], lig_node[ll_src, :ns]], -1)
            lig_node = layer(lig_node, ll_ei, ea_, None, edge_weight=ll_ew, edge_vec=ll_vec, assume_sorted=True)

        # -- cross graph (:321-327) ---------------------------------------------------------------------------------
        r, rpg = cross_cutoff(self, tr_sigma)
        li, ri, lr_ea, lr_vec, lr_ew = cross_graph(self, data, rec.pos.float(), c['rec_ptr'], r, rpg,
                                                   self.cross_distance_expansion, self.cross_edge_embedding)

        # -- joint graph: four edge groups, each CSR-sorted by target (:329-338) ------------------------------------
        n_lig = lig_node.shape[0]
        node = torch.cat([lig_node, rec_node], 0)
        rl_tgt, rev = torch.sort(ri, stable=True)            # receptor <- ligand direction: same pairs, sorted by residue
        rr_tgt32 = _rr_joint(c, n_lig)
        groups = [   # (target, gathered node, edge attr, edge vector, edge weight): int32, CSR-sorted, built once per forward
            (_i32(ll_tgt), _i32(ll_src), ll_ea, ll_vec.contiguous(), _flat(ll_ew)),                      # lig <- lig
            (_i32(li), _i32(ri + n_lig), lr_ea, lr_vec.contiguous(), _flat(lr_ew)),                      # lig <- rec
            (rr_tgt32[0], rr_tgt32[1], rr_ea, c['rr_vec'], _flat(c['rr_ew'])),                           # rec <- rec
            (_i32(rl_tgt + n_lig), _i32(li[rev]), lr_ea[rev], (-lr_vec[rev]).contiguous(),
             _flat(lr_ew[rev]) if torch.is_tensor(lr_ew) else None),                                     # rec <- lig, SH(-v)
        ]
        node = self._interaction_layers(node, groups, 2, merge=not self.differentiate_convolutions)
        return self._heads(data, c, node[:n_lig], tr_sigma, rot_sigma, tor_sigma, sync_free=False)

    def _sigmas(self, data):
        """(tr, rot, tor) sigma per complex; the confidence model takes the times as sigmas (models/cg_model.py:312-315)."""
        t = [data.complex_t[k] for k in ('tr', 'rot', 'tor')]
        return t if self.confidence_mode else self.t_to_sigma(*t)

    def _heads(self, data, c, lig_node, tr_sigma, rot_sigma, tor_sigma, sync_free):
        """Score mode: ``(tr, rot, tor, None)``; confidence mode: ``(confidence, atom_confidence)``."""
        if self.confidence_mode:
            return confidence_head(self, lig_node, c['lig_ptr'])
        return score_heads(self, data, c, lig_node, tr_sigma, rot_sigma, tor_sigma, sync_free) + (None,)
