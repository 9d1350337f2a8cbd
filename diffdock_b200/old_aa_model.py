"""Drop-in for the reference's ALL-ATOM confidence model ``models/old_aa_model.py:AAOldModel`` in confidence mode - what
``inference.py:192,209`` builds when the confidence model's parameters say ``all_atoms`` (the released DiffDock-L ranking
model) and ``utils/sampling.py:208-227`` calls once per batch of final poses (SURVEY.md section 8, rows f2 / f3).

Same constructor keywords, ``forward(data) -> confidence [B]`` (``[B, 2]`` with affinity_prediction) and ``state_dict`` keys
as the reference class for: confidence_mode=True, use_old_atom_encoder=True (the only encoder the reference class can be
built with - its new AtomEncoder rejects the ``lm_embedding_type`` keyword, models/old_aa_model.py:71), one noise schedule,
parallel=1.  Three node types and nine convolutions per interaction layer (:105-121, :229-266), all on the same sm_90a
kernels as the score model: neighbour lists from ddb200_radius_*, spherical harmonics evaluated in-kernel from the edge
vectors, OldTensorProductConvLayer on the fully fused wgmma kernel when its shapes allow.  The reversed directions
(atom<-ligand, residue<-ligand, residue<-atom) reuse the forward edge attributes AND the forward vector's harmonics, as the
reference does (:246-266).

Where every convolution has a fused-kernel shape and no complex has more than 10 000 residues or atoms, the forward makes
no device->host read after the per-batch constants (``_static``, ``_forward_sync_free``), as CGOldModel's score mode does:

1. The residue and atom node embeddings are computed once per batch with the sigma embedding set to zero; each call adds
   ``M . sigma_emb`` per complex (the encoders are affine in the sigma embedding).  A batch whose residue and atom stores
   carry a block layout - B poses of one receptor (``_unique``, diffdock_b200.hetero.collate_shared_receptor) or several
   complexes (``_blocks``, diffdock_b200.hetero.collate_packed) - embeds each distinct receptor once and gathers the rows
   onto the batch through ``node_map`` (diffdock_b200.cg_model.receptor_tiles / linked_edge_tiles).
2. The three static edge sets (residue-residue, atom-atom, atom-residue) are CSR-sorted by target once per batch; the
   residue<-atom group is the atom<-residue list sorted by residue, reading its attributes through ``edge_perm``.  Their
   edge attributes depend on sigma and are embedded per call: per batch edge, or - for a block layout at one time - per
   distinct receptor edge, read by every copy through ``edge_perm``.
3. The ligand graph and the ligand<-residue / ligand<-atom graphs go into capacity buffers with device counts; the
   atom<-ligand and residue<-ligand groups are permutations of those lists with the forward vector (``vec_sign = +1``).
4. Nine fused launches per layer, each with its own radial MLP, into one accumulator per (target type, convolution);
   three chained ddb200_tpconv_finalize calls per target type give ``pad(x) + up + up + up`` in the reference's order.
5. In a batch of repeated receptors at one time (``_uniform_t``: the sampler's ranking call at t = 0) the four layer-0
   groups that end on residues or atoms and start from them (residue<-residue, residue<-atom, atom<-atom, atom<-residue)
   see the same inputs in every copy: their messages are computed over the distinct receptors' edges and gathered onto
   every copy's rows.

CUDA only, inference only.  No CPU fallback.
"""
from __future__ import annotations

import os
import weakref

import torch
import torch.nn.functional as F
from torch import nn

from . import ops
from .aa_model import AAModel
from .cg_model import CGModel, _flat, _i32
from .hetero import receptor_blocks
from .irreps import irreps_str, sh_irreps
from .layers import (GaussianSmearing, OldAtomEncoder, _mlp, check_confidence_widths, check_forward, confidence_head,
                     cross_cutoff, cross_graph, edge_weight, ligand_graph)
from .old_cg_model import CGOldModel, sigma_map
from .synthetic import (LIG_FEATURE_DIMS as lig_feature_dims, REC_ATOM_FEATURE_DIMS as rec_atom_feature_dims,
                        REC_RESIDUE_FEATURE_DIMS as rec_residue_feature_dims)
from .tensor_layers import OldTensorProductConvLayer

# target-type rows of each interaction layer: (node type, its three convolutions in the order the reference adds them,
# models/old_aa_model.py:280-285); convolution k of layer l is conv_layers[9 l + k]
_LIG_SUM, _REC_SUM, _ATOM_SUM = (0, 2, 1), (6, 8, 7), (3, 4, 5)


def _uniq(st, B, n_edges):
    """True when ``st`` carries ``_unique = (nodes, edges, copies)`` for this batch of B copies: the one-block case of
    ``hetero.receptor_blocks``, which the forward reads for every block layout."""
    return getattr(st, '_unique', None) is not None and receptor_blocks(st, B, n_edges) is not None


def _csr(tgt, n_rows):
    """(target int32 sorted stably, order int64) of an edge list."""
    if tgt.shape[0] == 0:
        return _i32(tgt), torch.zeros(0, dtype=torch.long, device=tgt.device)
    t32, order, _ = ops.csr_sort_by_target(_i32(tgt), n_rows)
    return t32, order


class AAOldModel(nn.Module):
    # the ligand graph, the cross graphs and the per-batch constants of the sync-free path are the score models'
    _static_sync_free = CGModel._static_sync_free
    _ligand_edges_sync_free = CGModel._ligand_edges_sync_free
    _cross_graph_sync_free = CGModel._cross_graph_sync_free
    _cross_edge_embedding = CGModel._cross_edge_embedding
    _edge_embed_in_kernel = CGModel._edge_embed_in_kernel
    _receptor_tiles = staticmethod(AAModel._receptor_tiles)      # the all-atom block layout's index maps
    _bn = staticmethod(CGOldModel._bn)

    def __init__(self, t_to_sigma, device, timestep_emb_func, in_lig_edge_features=4, sigma_embed_dim=32, sh_lmax=2,
                 ns=16, nv=4, num_conv_layers=2, lig_max_radius=5, rec_max_radius=30, cross_max_distance=250,
                 center_max_distance=30, distance_embed_dim=32, cross_distance_embed_dim=32, no_torsion=False,
                 scale_by_sigma=True, norm_by_sigma=True, use_second_order_repr=False, batch_norm=True,
                 dynamic_max_cross=False, dropout=0.0, smooth_edges=False, odd_parity=False,
                 separate_noise_schedule=False, lm_embedding_type=False, confidence_mode=False, confidence_dropout=0,
                 confidence_no_batchnorm=False, asyncronous_noise_schedule=False, affinity_prediction=False, parallel=1,
                 parallel_aggregators="mean max min std", num_confidence_outputs=1, fixed_center_conv=False,
                 no_aminoacid_identities=False, include_miscellaneous_atoms=False, use_old_atom_encoder=False,
                 lm_embedding_dim=1280):
        super().__init__()
        lm_embedding_type = lm_embedding_type or None
        assert (not no_aminoacid_identities) or (lm_embedding_type is None), "no language model emb without identities"
        if parallel != 1:
            raise NotImplementedError("parallel > 1 (affinity aggregation over several poses) is outside the hot-path scope")
        if not confidence_mode:
            raise NotImplementedError("diffdock_b200.AAOldModel is built in confidence mode only (SURVEY.md rows f2/f3); "
                                      "the score model is diffdock_b200.cg_model.CGModel")
        if not use_old_atom_encoder:
            raise NotImplementedError("models/old_aa_model.py can only be constructed with use_old_atom_encoder=True")
        if include_miscellaneous_atoms or separate_noise_schedule or asyncronous_noise_schedule or use_second_order_repr:
            raise NotImplementedError("misc atoms / separate or asynchronous noise schedules / second-order irreps are "
                                      "outside the hot-path scope (SURVEY.md section 8)")
        self.t_to_sigma, self.device, self.timestep_emb_func = t_to_sigma, device, timestep_emb_func
        self.in_lig_edge_features, self.sigma_embed_dim = in_lig_edge_features, sigma_embed_dim
        self.lig_max_radius, self.rec_max_radius = lig_max_radius, rec_max_radius
        self.cross_max_distance, self.dynamic_max_cross = cross_max_distance, dynamic_max_cross
        self.sh_lmax, self.sh_irreps = sh_lmax, irreps_str(sh_irreps(sh_lmax))
        self.ns, self.nv, self.smooth_edges = ns, nv, smooth_edges
        self.confidence_mode, self.num_conv_layers = confidence_mode, num_conv_layers
        self.affinity_prediction, self.no_aminoacid_identities = affinity_prediction, no_aminoacid_identities
        S, D, Dx = sigma_embed_dim, distance_embed_dim, cross_distance_embed_dim
        kw = dict(lm_embedding_dim=lm_embedding_dim) if lm_embedding_type is not None else {}
        self.lig_node_embedding = OldAtomEncoder(ns, lig_feature_dims, S)
        self.lig_edge_embedding = _mlp(in_lig_edge_features + S + D, ns, ns, dropout)
        self.rec_node_embedding = OldAtomEncoder(ns, rec_residue_feature_dims, S, lm_embedding_type=lm_embedding_type, **kw)
        self.rec_edge_embedding = _mlp(S + D, ns, ns, dropout)
        self.atom_node_embedding = OldAtomEncoder(ns, rec_atom_feature_dims, S)
        self.atom_edge_embedding = _mlp(S + D, ns, ns, dropout)
        self.lr_edge_embedding = _mlp(S + Dx, ns, ns, dropout)
        self.ar_edge_embedding = _mlp(S + D, ns, ns, dropout)
        self.la_edge_embedding = _mlp(S + Dx, ns, ns, dropout)
        self.lig_distance_expansion = GaussianSmearing(0.0, lig_max_radius, D)
        self.rec_distance_expansion = GaussianSmearing(0.0, rec_max_radius, D)
        self.cross_distance_expansion = GaussianSmearing(0.0, cross_max_distance, Dx)
        seq = [f'{ns}x0e', f'{ns}x0e + {nv}x1o', f'{ns}x0e + {nv}x1o + {nv}x1e',
               f'{ns}x0e + {nv}x1o + {nv}x1e + {ns}x0o']
        convs = []
        for i in range(num_conv_layers):
            p = dict(in_irreps=seq[min(i, 3)], sh_irreps=self.sh_irreps, out_irreps=seq[min(i + 1, 3)],
                     n_edge_features=3 * ns, residual=False, batch_norm=batch_norm, dropout=dropout)
            convs += [OldTensorProductConvLayer(**p) for _ in range(9)]       # 3 intra & 6 inter per layer (:119-120)
        self.conv_layers = nn.ModuleList(convs)
        bn = (lambda: nn.Identity()) if confidence_no_batchnorm else (lambda: nn.BatchNorm1d(ns))
        out_dim = (num_confidence_outputs + 1) if affinity_prediction else num_confidence_outputs
        self.confidence_predictor = nn.Sequential(
            nn.Linear(2 * ns if num_conv_layers >= 3 else ns, ns), bn(), nn.ReLU(), nn.Dropout(confidence_dropout),
            nn.Linear(ns, ns), bn(), nn.ReLU(), nn.Dropout(confidence_dropout), nn.Linear(ns, out_dim))
        self._conf_tail = ns if num_conv_layers >= 3 else 0
        check_confidence_widths(self)
        self._sync_free = None

    def load_state_dict(self, state_dict, strict=True, **kw):
        """Reference checkpoints carry e3nn's tensor-product buffers (``*.tp.*``): dropped, the kernels have their own tables."""
        sd = {k: v for k, v in state_dict.items() if '.tp.' not in k}
        return super().load_state_dict(sd, strict=strict, **kw)

    def get_edge_weight(self, edge_vec, max_norm):                      # models/old_aa_model.py:352-356
        return edge_weight(edge_vec, max_norm, self.smooth_edges)

    def _static_graph(self, data, nt, pos, edge_embedding, node_embedding, expansion, max_r):
        """Receptor-residue / receptor-atom graph on precomputed edges (:400-445); row 0 = target, row 1 = gathered node."""
        st = data[nt]
        st.node_sigma_emb = self.timestep_emb_func(st.node_t['tr'])
        ei = data[nt, nt].edge_index.long()
        vec = pos[ei[1]] - pos[ei[0]]
        ea = edge_embedding(torch.cat([st.node_sigma_emb[ei[0]], expansion(vec.norm(dim=-1))], 1))
        node = node_embedding(torch.cat([st.x.float(), st.node_sigma_emb], 1))
        return node, ei, ea, vec, self.get_edge_weight(vec, max_r)

    @torch.no_grad()
    def forward(self, data):                                            # models/old_aa_model.py:202-286
        check_forward(self, data)
        if self.sync_free_capable():
            c = self._static(data)
            if max(c['rec_max'], c['atom_max']) <= 10000:      # the cross graphs' cap (:454, :470) must not bind
                return confidence_head(self, self._forward_sync_free(data, c), c['lig_ptr'])[0]
        return self._forward_host_sized(data)

    def sync_free_capable(self):
        """The forward runs without a device->host read after the per-batch constants when every one of the 9 L
        convolutions has a shape the fully fused kernel supports."""
        if self._sync_free is None:
            ok = os.environ.get('DDB200_SYNC_FREE', '1') != '0'
            self._sync_free = bool(ok and all(layer.fused_capable(self.ns, self.ns) for layer in self.conv_layers))
        return self._sync_free

    # ---------------------------------------------------------------------------------------------------------
    def _static(self, data):
        """Per-batch constants, cached on ``data`` (host reads of the node counts): the sigma-free residue and atom node
        embeddings with their sigma maps, the static edge sets CSR-sorted by target in the joint numbering
        [ligand | residues | atoms] with the complex of each edge, and the ligand / cross-graph constants of
        CGModel._static_sync_free.  A batch whose residue and atom stores carry a block layout (``AAModel._receptor_tiles``:
        ``collate_shared_receptor``'s one receptor, ``collate_packed``'s distinct receptors) also gets the distinct
        receptors' edge vectors with the distinct row of every sorted edge (``perm``), and - when some receptor is
        repeated - their four static groups in the local numbering [distinct residues | distinct atoms] (``shared``)."""
        rec, atom, lig = data['receptor'], data['atom'], data['ligand']
        rr, aa, ar, ll = data['receptor', 'receptor'], data['atom', 'atom'], data['atom', 'receptor'], data['ligand', 'ligand']
        hit = getattr(rr, '_b200_v10aa', None)
        if hit is not None and hit[0]() is self:
            return hit[1]
        B, S = data.num_graphs, self.sigma_embed_dim
        n_lig, n_rec, n_atom = lig.batch.shape[0], rec.pos.shape[0], atom.pos.shape[0]
        o_r, o_a = n_lig, n_lig + n_rec
        N = o_a + n_atom
        rr_ei, aa_ei, ar_ei = rr.edge_index.long(), aa.edge_index.long(), ar.edge_index.long()
        tiles = self._receptor_tiles(data, B, rr_ei, aa_ei, ar_ei)
        rt, at, lt = (tiles['rec'], tiles['atom'], tiles['ar']) if tiles is not None else (None, None, None)
        c = {}
        # node embeddings with the sigma embedding set to zero (:401, :424), once per distinct receptor, the LM layer included
        for key, st, enc, t in (('rec', rec, self.rec_node_embedding, rt), ('atom', atom, self.atom_node_embedding, at)):
            x1 = (st.x[t['nodes']] if t is not None else st.x).float()
            base = enc(torch.cat([x1, x1.new_zeros((x1.shape[0], S))], 1))
            c[key + '_base'] = base[t['node_map']] if t is not None else base
            c[key + '_sigma_map'] = sigma_map(enc, S, st.x.shape[1])
        c['rec_gid'], c['atom_gid'] = rec.batch, atom.batch
        # static edge sets (:404-445, :486): row 0 = convolution target, vector gathered - target, sigma of the target's complex
        rp, ap = rec.pos.float(), atom.pos.float()
        spec = {'rr': (rr_ei[0] + o_r, rr_ei[1] + o_r, rp[rr_ei[1]] - rp[rr_ei[0]], rec.batch[rr_ei[0]], self.rec_max_radius, rt),
                'aa': (aa_ei[0] + o_a, aa_ei[1] + o_a, ap[aa_ei[1]] - ap[aa_ei[0]], atom.batch[aa_ei[0]], self.lig_max_radius, at),
                'ar': (ar_ei[0] + o_a, ar_ei[1] + o_r, rp[ar_ei[1]] - ap[ar_ei[0]], atom.batch[ar_ei[0]], None, lt)}
        ew = lambda vec, max_r: _flat(self.get_edge_weight(vec, max_r)) if max_r is not None else None
        for k, (tgt, src, vec, gid, max_r, t) in spec.items():
            t32, order = _csr(tgt, N)
            vs = vec[order].contiguous()
            c[k] = dict(tgt=t32, src=_i32(src[order]), vec=vs, gid=_i32(gid[order]), ew=ew(vs, max_r))
            if t is not None:       # the distinct receptors' edges, and the distinct row of every sorted edge
                vu = vec[t['edges']].contiguous()
                c[k].update(perm=_i32(t['edge_map'][order]), vec_u=vu, ew_u=ew(vu, max_r),
                            row_u=torch.zeros(vu.shape[0], dtype=torch.int32, device=vu.device))
        # residue <- atom (:264-266): the atom <- residue edges sorted by residue, forward attributes and vector
        t32, order = _csr(c['ar']['src'].long(), N)
        c['ra'] = dict(tgt=t32, src=c['ar']['tgt'][order].contiguous(), perm=_i32(order))
        if tiles is not None:
            c['ra']['perm_u'] = c['ar']['perm'][order].contiguous()
            nr_u, na_u = rt['nodes'].shape[0], at['nodes'].shape[0]
            if nr_u + na_u < n_rec + n_atom and self.num_conv_layers > 1:
                # the four layer-0 groups between residues and atoms over the distinct receptors, numbered [residues |
                # atoms]; each reads the attributes of its distinct edge (the atom-residue edges' for residue <- atom)
                n_u = nr_u + na_u
                loc = {'rr': (rt['edge_index'][0], rt['edge_index'][1]),
                       'aa': (at['edge_index'][0] + nr_u, at['edge_index'][1] + nr_u),
                       'ar': (lt['edge_index'][0] + nr_u, lt['edge_index'][1]),
                       'ra': (lt['edge_index'][1], lt['edge_index'][0] + nr_u)}
                groups = {}
                for k, (tgt, src) in loc.items():
                    t32, order = _csr(tgt, n_u)
                    groups[k] = (t32, _i32(src[order]), _i32(order))
                c['shared'] = (rt['nodes'], at['nodes'], rt['node_map'], at['node_map'], groups)
        # ligand graph and cross-graph constants (CGModel._static_sync_free) and the atom side of the ligand<-atom graph
        c['rec_ptr'], c['atom_ptr'], c['lig_ptr'] = (ops.segment_ptr(s.batch, B) for s in (rec, atom, lig))
        c['rr_tgt_batch'] = rec.batch[rr_ei[0]]
        bonds = ll.edge_index[:, lig.edge_mask].long()
        c['bonds'], c['n_bonds'] = bonds, int(bonds.shape[1])
        c['bond_batch'] = lig.batch[bonds[0]] if bonds.shape[1] else None
        self._static_sync_free(data, c)
        atom_cnt, lig_cnt = c['atom_ptr'][1:] - c['atom_ptr'][:-1], c['lig_ptr'][1:] - c['lig_ptr'][:-1]
        c['atom_max'] = int(atom_cnt.max()) if B else 0
        c['cap_la'] = int((lig_cnt.long() * atom_cnt.long()).sum())      # every ligand atom x every atom of its complex
        c['atom_batch32'] = _i32(atom.batch)
        rr._b200_v10aa = (weakref.ref(self), c)
        return c

    def _static_edge_attr(self, sig, vec, row, mlp, gs):
        """``mlp(cat[sigma_emb of the edge's complex, gs(|vec|)])`` (:409-410, :431-432, :489) with ``sig`` [rows, S] and
        ``row`` the sigma row of each edge; an empty edge set (e.g. a receptor without contact edges) has none."""
        if vec.shape[0] == 0:
            return vec.new_zeros((0, self.ns))
        return self._cross_edge_embedding(sig, vec, row, None, mlp, gs)

    def _forward_sync_free(self, data, c):
        """Ligand node features after the interaction layers without a device->host read (module docstring, 1-5)."""
        lig, rec, atom = data['ligand'], data['receptor'], data['atom']
        ns, n_lig = self.ns, lig.batch.shape[0]
        o_r, o_a = n_lig, n_lig + rec.pos.shape[0]
        N = o_a + atom.pos.shape[0]
        # distinct receptors at one time: every copy's static edge attributes and layer-0 messages are its distinct one's
        uniform = 'perm_u' in c['ra'] and getattr(data, '_uniform_t', False)
        tr_sigma = data.complex_t['tr']                                      # confidence mode: the times are the sigmas
        sig = self.timestep_emb_func(tr_sigma)                               # [B, S], per complex

        # -- residue / atom embeddings and the static groups (:400-445, :486-491) ----------------------------------------
        rec_node = c['rec_base'] + (sig @ c['rec_sigma_map'].t())[c['rec_gid']]
        atom_node = c['atom_base'] + (sig @ c['atom_sigma_map'].t())[c['atom_gid']]
        emb = {'rr': (self.rec_edge_embedding, self.rec_distance_expansion),
               'aa': (self.atom_edge_embedding, self.lig_distance_expansion),
               'ar': (self.ar_edge_embedding, self.rec_distance_expansion)}
        g = {}
        for k, (mlp, gs) in emb.items():
            d = c[k]
            if uniform:     # the distinct receptors' attributes; every edge reads its distinct row through edge_perm
                ea = self._static_edge_attr(sig[:1], d['vec_u'], d['row_u'], mlp, gs)
                g[k] = (d['tgt'], d['src'], ea, d['vec_u'], d['ew_u'], dict(edge_perm=d['perm']))
            else:
                ea = self._static_edge_attr(sig, d['vec'], d['gid'], mlp, gs)
                g[k] = (d['tgt'], d['src'], ea, d['vec'], d['ew'], {})
        ra = c['ra']
        g['ra'] = (ra['tgt'], ra['src'], g['ar'][2], g['ar'][3], None,
                   dict(edge_perm=ra['perm_u'] if uniform else ra['perm']))
        shared = uniform and 'shared' in c

        # -- ligand graph (:358-398) and ligand cross graphs (:447-485) --------------------------------------------------
        g_ll = self._ligand_edges_sync_free(data, c)
        lig_node = self.lig_node_embedding(torch.cat([lig.x.float(), lig.node_sigma_emb], 1))
        r, rpg = cross_cutoff(self, tr_sigma)
        # atom <- ligand and residue <- ligand reuse the forward attributes and harmonics (:254, :262): vec_sign = +1
        g_lr, g_rl = self._cross_graph_sync_free(data, c, rec.pos.float().contiguous(), c['rec_ptr'], c['rec_batch32'],
                                                 c['rec_max'], c['cap_cross'], r, rpg, o_r, self.lr_edge_embedding,
                                                 self.cross_distance_expansion, vec_sign=1.0)
        g_la, g_al = self._cross_graph_sync_free(data, c, atom.pos.float().contiguous(), c['atom_ptr'], c['atom_batch32'],
                                                 c['atom_max'], c['cap_la'], float(self.lig_max_radius), None, o_a,
                                                 self.la_edge_embedding, self.cross_distance_expansion, vec_sign=1.0)
        groups = {0: (g_ll, n_lig), 1: (g_lr, n_lig), 2: (g_la, n_lig), 3: (g['aa'], N), 4: (g_al, N), 5: (g['ar'], N),
                  6: (g['rr'], o_a), 7: (g_rl, o_a), 8: (g['ra'], o_a)}

        # -- interaction layers (:229-286) --------------------------------------------------------------------------------
        x = torch.cat([lig_node, rec_node, atom_node], 0)
        L, C = self.num_conv_layers, self.conv_layers
        for l in range(L):
            last = l == L - 1
            convs = C[9 * l:9 * l + 9]
            ks = (0, 1, 2) if last else range(9)
            acc = self._shared_static_messages(x, c, g, o_r, o_a, N, convs) if (l == 0 and shared and not last) else {}
            for k in ks:        # raw sums per convolution; rows of a sum: its target type's rows in the joint numbering
                if k not in acc:
                    acc[k] = convs[k].accumulate_group(x, groups[k][0], 0, groups[k][1], ns)
            rows = [(0, n_lig, _LIG_SUM)] + ([] if last else [(o_r, o_a, _REC_SUM), (o_a, N, _ATOM_SUM)])
            out = torch.empty((n_lig if last else N, convs[0].out_size), device=x.device)
            for lo, hi, order in rows:      # pad(x) + up_a + up_b + up_c (:280-285)
                part = x[lo:hi]
                for j, k in enumerate(order):
                    s, n = acc[k]
                    part = ops.tpconv_finalize(s[lo:hi], n[lo:hi], True, *self._bn(convs[k]), residual=part,
                                               out=out[lo:hi] if j == 2 else None)
            x = out
        return x

    def _shared_static_messages(self, x, c, g, o_r, o_a, N, convs):
        """Layer-0 sums of the four groups between residues and atoms (residue<-residue, residue<-atom, atom<-atom,
        atom<-residue) for a batch of copies of the same receptors at ONE time: their node features and edge attributes are
        the same in every copy, so the sums are computed once over the distinct receptors (local numbering [distinct
        residues | distinct atoms], ``c['shared']``) and gathered onto every copy's rows through the node maps.  ``g``:
        the batch's static groups, whose attribute arrays are already the distinct edges'."""
        rows_r, rows_a, map_r, map_a, local = c['shared']
        nr_u = rows_r.shape[0]
        x0 = torch.cat([x[o_r + rows_r], x[o_a + rows_a]], 0)
        n_u = x0.shape[0]
        D = convs[0].out_size
        acc = {}
        for k, key, lo, hi, part, node_map in ((6, 'rr', o_r, o_a, slice(0, nr_u), map_r),
                                               (8, 'ra', o_r, o_a, slice(0, nr_u), map_r),
                                               (3, 'aa', o_a, N, slice(nr_u, n_u), map_a),
                                               (5, 'ar', o_a, N, slice(nr_u, n_u), map_a)):
            tgt, src, perm = local[key]
            s0, n0 = convs[k].accumulate_group(x0, (tgt, src, *g[key][2:5], dict(edge_perm=perm)), 0, n_u, self.ns)
            s, n = ops.new_accumulators(hi, D, x.device)
            s[lo:] = s0[part][node_map]
            n[lo:] = n0[part][node_map]
            acc[k] = (s, n)
        return acc

    def _forward_host_sized(self, data):
        """Exactly-sized neighbour lists (one host read of each edge count), every convolution through
        OldTensorProductConvLayer.forward: layer shapes outside the fused kernel, or more than 10 000 residues / atoms."""
        lig_s, rec_s, atom_s = data['ligand'], data['receptor'], data['atom']
        B, ns, L, C = data.num_graphs, self.ns, self.num_conv_layers, self.conv_layers
        tr_sigma = data.complex_t['tr']                                 # confidence mode: times are used as they are (:209)
        rp, ap = rec_s.pos.float(), atom_s.pos.float()

        # ligand graph (:358-398): bonds + radius graph
        tgt, src, lig_ea, lig_vec, lig_w, lig_x = ligand_graph(self, data, ops.segment_ptr(lig_s.batch, B))
        lig_ei = torch.stack([tgt, src])
        lig = self.lig_node_embedding(lig_x)
        lig_ea = self.lig_edge_embedding(lig_ea)

        rec, rec_ei, rec_ea, rec_vec, rec_w = self._static_graph(data, 'receptor', rp, self.rec_edge_embedding,
                                                                 self.rec_node_embedding, self.rec_distance_expansion,
                                                                 self.rec_max_radius)
        atom, at_ei, at_ea, at_vec, at_w = self._static_graph(data, 'atom', ap, self.atom_edge_embedding,
                                                              self.atom_node_embedding, self.lig_distance_expansion,
                                                              self.lig_max_radius)

        # cross graphs (:447-491): ligand-residue (cut-off per complex), ligand-atom (lig_max_radius), atom-residue (given)
        r, rpg = cross_cutoff(self, tr_sigma)
        li, ri, lr_ea, lr_vec, lr_w = cross_graph(self, data, rp, ops.segment_ptr(rec_s.batch, B), r, rpg,
                                                  self.cross_distance_expansion, self.lr_edge_embedding)
        la_l, la_a, la_ea, la_vec, la_w = cross_graph(self, data, ap, ops.segment_ptr(atom_s.batch, B),
                                                      float(self.lig_max_radius), None, self.cross_distance_expansion,
                                                      self.la_edge_embedding)
        lr, la = torch.stack([li, ri]), torch.stack([la_l, la_a])
        ar = data['atom', 'receptor'].edge_index.long()
        ar_vec = rp[ar[1]] - ap[ar[0]]
        ar_ea = self.ar_edge_embedding(torch.cat([atom_s.node_sigma_emb[ar[0]],
                                                  self.rec_distance_expansion(ar_vec.norm(dim=-1))], 1))

        cat = lambda e, a, b: torch.cat([e, a[:, :ns], b[:, :ns]], -1)
        flip = lambda ei: torch.flip(ei, dims=[0])
        for l in range(L):
            k = 9 * l
            lig_up = C[k](lig, lig_ei, cat(lig_ea, lig[lig_ei[0]], lig[lig_ei[1]]), None, edge_weight=lig_w, edge_vec=lig_vec)
            lr_up = C[k + 1](rec, lr, cat(lr_ea, lig[lr[0]], rec[lr[1]]), None, out_nodes=lig.shape[0], edge_weight=lr_w,
                             edge_vec=lr_vec, assume_sorted=True)
            la_up = C[k + 2](atom, la, cat(la_ea, lig[la[0]], atom[la[1]]), None, out_nodes=lig.shape[0], edge_weight=la_w,
                             edge_vec=la_vec, assume_sorted=True)
            if l != L - 1:
                at_up = C[k + 3](atom, at_ei, cat(at_ea, atom[at_ei[0]], atom[at_ei[1]]), None, edge_weight=at_w, edge_vec=at_vec)
                al_up = C[k + 4](lig, flip(la), cat(la_ea, atom[la[1]], lig[la[0]]), None, out_nodes=atom.shape[0],
                                 edge_weight=la_w, edge_vec=la_vec)
                ar_up = C[k + 5](rec, ar, cat(ar_ea, atom[ar[0]], rec[ar[1]]), None, out_nodes=atom.shape[0], edge_weight=1.0,
                                 edge_vec=ar_vec)
                rec_up = C[k + 6](rec, rec_ei, cat(rec_ea, rec[rec_ei[0]], rec[rec_ei[1]]), None, edge_weight=rec_w,
                                  edge_vec=rec_vec)
                rl_up = C[k + 7](lig, flip(lr), cat(lr_ea, rec[lr[1]], lig[lr[0]]), None, out_nodes=rec.shape[0],
                                 edge_weight=lr_w, edge_vec=lr_vec)
                ra_up = C[k + 8](atom, flip(ar), cat(ar_ea, rec[ar[1]], atom[ar[0]]), None, out_nodes=rec.shape[0],
                                 edge_weight=1.0, edge_vec=ar_vec)
            lig = F.pad(lig, (0, lig_up.shape[-1] - lig.shape[-1])) + lig_up + la_up + lr_up
            if l != L - 1:
                atom = F.pad(atom, (0, at_up.shape[-1] - atom.shape[-1])) + at_up + al_up + ar_up
                rec = F.pad(rec, (0, rec_up.shape[-1] - rec.shape[-1])) + rec_up + ra_up + rl_up
        return confidence_head(self, lig, ops.segment_ptr(lig_s.batch, B))[0]
