"""Drop-in for the reference's all-atom model ``models/aa_model.py:AAModel`` (score mode; confidence mode as in
diffdock_b200/cg_model.py) - SURVEY.md section 8, row f3.

Same constructor keywords, ``forward(data) -> (tr_pred, rot_pred, tor_pred, None)`` contract, ``state_dict`` keys and side
effects on ``data`` (the cached receptor / atom embeddings of models/aa_model.py:319-333) as the reference class.  It is the
coarse-grained model (diffdock_b200/cg_model.py) with a third node type - receptor atoms - and nine edge groups per
interaction layer instead of four (three in the last layer, models/aa_model.py:401-430); every group runs on the same
sm_90a convolution kernels through ``TensorProductConvLayer.forward_groups`` (fully fused wgmma kernel when the shape
allows), neighbour lists come from ddb200_radius_*, spherical harmonics are evaluated in-kernel.

Two reference behaviours are reproduced on purpose: the reversed groups (residue<-ligand, residue<-atom, atom<-ligand) reuse
the FORWARD direction's spherical harmonics (:405-406; the coarse-grained model evaluates Y(-v) instead, cg_model.py:556-557),
and ligand-atom distances go through the ligand distance expansion (:613) into an MLP sized for the cross expansion (:108).

CUDA only, inference only.  No CPU fallback.  Like the coarse-grained model the forward has a sync-free
form (``_forward_sync_free``: every per-step neighbour list in a capacity buffer with its live count on the device, the three
reversed groups as permutations of the forward lists, sigma terms of the four static groups added inside the kernel), so the
sampler captures the all-atom step in a CUDA graph too; ``_forward_host_sized`` reads the neighbour-list sizes back and is
used for shapes outside the fused kernel or more than 10000 residues / atoms per complex."""
from __future__ import annotations

import torch
from torch import nn

from . import ops
from .cg_model import CGModel, _i32, linked_edge_tiles, receptor_tiles
from .layers import AtomEncoder, _mlp, cross_cutoff, cross_graph
from .synthetic import REC_ATOM_FEATURE_DIMS as rec_atom_feature_dims


class AAModel(CGModel):
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
                 embed_also_ligand=False, atom_confidence=False, sidechain_pred=False, depthwise_convolution=False,
                 crop_beyond=None):
        if crop_beyond is not None:
            raise NotImplementedError("models/aa_model.py:366-368 raises for crop_beyond too")
        if smooth_edges:
            raise NotImplementedError("the reference AAModel cannot run with smooth_edges (it concatenates the integer "
                                      "atom-residue edge weight with tensors, models/aa_model.py:413-416)")
        super().__init__(t_to_sigma, device, timestep_emb_func, in_lig_edge_features=in_lig_edge_features,
                         sigma_embed_dim=sigma_embed_dim, sh_lmax=sh_lmax, ns=ns, nv=nv, num_conv_layers=num_conv_layers,
                         lig_max_radius=lig_max_radius, rec_max_radius=rec_max_radius,
                         cross_max_distance=cross_max_distance, center_max_distance=center_max_distance,
                         distance_embed_dim=distance_embed_dim, cross_distance_embed_dim=cross_distance_embed_dim,
                         no_torsion=no_torsion, scale_by_sigma=scale_by_sigma, norm_by_sigma=norm_by_sigma,
                         use_second_order_repr=use_second_order_repr, batch_norm=batch_norm,
                         dynamic_max_cross=dynamic_max_cross, dropout=dropout, smooth_edges=False, odd_parity=odd_parity,
                         separate_noise_schedule=separate_noise_schedule, lm_embedding_type=lm_embedding_type,
                         confidence_mode=confidence_mode, confidence_dropout=confidence_dropout,
                         confidence_no_batchnorm=confidence_no_batchnorm, num_confidence_outputs=num_confidence_outputs,
                         atom_num_confidence_outputs=atom_num_confidence_outputs,
                         asyncronous_noise_schedule=asyncronous_noise_schedule,
                         affinity_prediction=affinity_prediction, parallel=parallel, fixed_center_conv=fixed_center_conv,
                         no_aminoacid_identities=no_aminoacid_identities,
                         include_miscellaneous_atoms=include_miscellaneous_atoms,
                         differentiate_convolutions=differentiate_convolutions, tp_weights_layers=tp_weights_layers,
                         num_prot_emb_layers=num_prot_emb_layers, reduce_pseudoscalars=reduce_pseudoscalars,
                         embed_also_ligand=embed_also_ligand, atom_confidence=atom_confidence, sidechain_pred=sidechain_pred,
                         depthwise_convolution=depthwise_convolution)
        S, D, Dx = sigma_embed_dim, distance_embed_dim, cross_distance_embed_dim
        del self.cross_edge_embedding
        self.atom_node_embedding = AtomEncoder(emb_dim=ns, feature_dims=rec_atom_feature_dims, sigma_embed_dim=0)
        self.atom_edge_embedding = _mlp(D, ns, ns, dropout)
        self.lr_edge_embedding = _mlp(S + Dx, ns, ns, dropout)
        self.ar_edge_embedding = _mlp(D, ns, ns, dropout)
        self.la_edge_embedding = _mlp(S + Dx, ns, ns, dropout)
        self.rec_emb_layers = nn.ModuleList([self.conv(i, 4 if differentiate_convolutions else 1)
                                             for i in range(num_prot_emb_layers)])
        self.conv_layers = self._interaction_stack(9, 3)

    def sync_free_capable(self):
        """As CGModel.sync_free_capable; additionally every edge type must have its own radial MLP (the merged single-group
        form concatenates edge lists, which needs their sizes on the host)."""
        return self.differentiate_convolutions and super().sync_free_capable()

    def sync_free_crop_capable(self):
        """No per-step cropping on the sync-free path: the reference crops the receptor atoms too (utils/utils.py:388-413),
        which the masked crop of CGModel does not cover; the sampler keeps the eager crop for this model."""
        return False

    # ---------------------------------------------------------------------------------------------------------
    @staticmethod
    def _csr(tgt, src, n_rows, *payload):
        """(tgt32, src32, payload...) sorted stably by target."""
        t32, order, _ = ops.csr_sort_by_target(_i32(tgt), n_rows)
        return (t32, _i32(src[order])) + tuple(p[order].contiguous() for p in payload)

    @staticmethod
    def _receptor_tiles(data, B, rr_ei, aa_ei, ar_ei):
        """Index maps between a batch whose residue and atom stores carry a block layout (``_blocks`` / ``_unique``) and its
        distinct receptors: ``{'rec': .., 'atom': ..}`` from ``receptor_tiles``, ``'ar'`` from ``linked_edge_tiles`` for the
        atom-residue edges; None without a layout."""
        rt = receptor_tiles(data['receptor'], B, rr_ei)
        at = receptor_tiles(data['atom'], B, aa_ei) if rt is not None else None
        lt = linked_edge_tiles(data['atom'], at, rt, ar_ei, B) if at is not None else None
        return None if lt is None else dict(rec=rt, atom=at, ar=lt)

    def _static(self, data):
        """Pose-independent part, cached on ``data`` like models/aa_model.py:276-333: residue / atom node embeddings, the
        edge embeddings of the three static graphs (residue-residue, atom-atom, atom-residue), the optional protein
        embedding layers over their four groups, and the CSR-sorted static edge groups of the joint graph.

        When the batch holds copies of the same receptors (the poses of one complex, ``collate_shared_receptor``, or several
        complexes of a packed batch, ``collate_packed``), the embeddings and the protein embedding layers run once per
        distinct receptor and are mapped onto the batch rows; the reference recomputes them for every pose
        (models/aa_model.py:276-333 over the B-fold receptor)."""
        rec, atom, lig = data['receptor'], data['atom'], data['ligand']
        rr, aa, ar, ll = data['receptor', 'receptor'], data['atom', 'atom'], data['atom', 'receptor'], data['ligand', 'ligand']
        if hasattr(rec, 'rec_node_attr') and hasattr(rr, '_b200aa'):
            return rr._b200aa
        ns, B = self.ns, data.num_graphs
        rp, ap = rec.pos.float(), atom.pos.float()
        n_rec, n_atom, n_lig = rp.shape[0], ap.shape[0], lig.pos.shape[0]
        rr_ei, aa_ei, ar_ei = rr.edge_index.long(), aa.edge_index.long(), ar.edge_index.long()
        rr_vec, aa_vec = rp[rr_ei[1]] - rp[rr_ei[0]], ap[aa_ei[1]] - ap[aa_ei[0]]
        ar_vec = rp[ar_ei[1]] - ap[ar_ei[0]]
        tiles = self._receptor_tiles(data, B, rr_ei, aa_ei, ar_ei)
        if tiles is None:
            xr, xa, rr_u, aa_u, ar_u, vecs = rec.x, atom.x, rr_ei, aa_ei, ar_ei, (rr_vec, aa_vec, ar_vec)
        else:
            rt, at, lt = tiles['rec'], tiles['atom'], tiles['ar']
            xr, xa = rec.x[rt['nodes']], atom.x[at['nodes']]
            rr_u, aa_u, ar_u = rt['edge_index'], at['edge_index'], lt['edge_index']
            vecs = (rr_vec[rt['edges']], aa_vec[at['edges']], ar_vec[lt['edges']])
        rr_vec_u, aa_vec_u, ar_vec_u = vecs
        nr_u, na_u = xr.shape[0], xa.shape[0]
        rr_ea = self.rec_edge_embedding(self.rec_distance_expansion(rr_vec_u.norm(dim=-1)))
        aa_ea = self.atom_edge_embedding(self.lig_distance_expansion(aa_vec_u.norm(dim=-1)))
        ar_ea = self.ar_edge_embedding(self.rec_distance_expansion(ar_vec_u.norm(dim=-1)))
        r_node, a_node = self.rec_node_embedding(xr), self.atom_node_embedding(xa)
        # layer-0 messages of the static groups can be shared by the copies (_shared_static_messages)
        shareable = tiles is not None and nr_u + na_u < n_rec + n_atom and self.differentiate_convolutions \
            and len(self.conv_layers) > 1
        u_groups = None
        if len(self.rec_emb_layers) or shareable:
            # joint numbering [residues | atoms] (:301-311): residue<-residue, atom<-residue, atom<-atom, residue<-atom
            n = nr_u + na_u
            u_groups = [self._csr(rr_u[0], rr_u[1], n, rr_ea, rr_vec_u),
                        self._csr(ar_u[0] + nr_u, ar_u[1], n, ar_ea, ar_vec_u),
                        self._csr(aa_u[0] + nr_u, aa_u[1] + nr_u, n, aa_ea, aa_vec_u),
                        self._csr(ar_u[1], ar_u[0] + nr_u, n, ar_ea, ar_vec_u)]       # reversed: forward harmonics
        if len(self.rec_emb_layers):
            node = torch.cat([r_node, a_node], 0)
            for layer in self.rec_emb_layers:
                node = layer.forward_groups(node, [g + (None,) for g in u_groups], gather_scalars=ns)
            r_node, a_node = node[:nr_u], node[nr_u:]
        if tiles is not None:
            r_node, a_node = r_node[rt['node_map']], a_node[at['node_map']]
            rr_ea, aa_ea, ar_ea = rr_ea[rt['edge_map']], aa_ea[at['edge_map']], ar_ea[lt['edge_map']]
        rec.rec_node_attr, rr.rec_edge_attr, rr.edge_sh, rr.edge_weight = r_node, rr_ea, None, 1.0
        atom.atom_node_attr, aa.atom_edge_attr, aa.edge_sh, aa.edge_weight = a_node, aa_ea, None, 1.0
        ar.edge_attr, ar.edge_sh, ar.edge_weight = ar_ea, None, 1
        c = {}
        N = n_lig + n_rec + n_atom
        o_r, o_a = n_lig, n_lig + n_rec
        # static groups of the joint graph [ligand | residues | atoms], CSR by target, with the graph id of the sigma term
        gid = lambda b: b.to(torch.int64)
        c['rr'] = self._csr(rr_ei[0] + o_r, rr_ei[1] + o_r, N, rr_ea, rr_vec, gid(rec.batch[rr_ei[0]]))
        c['ra'] = self._csr(ar_ei[1] + o_r, ar_ei[0] + o_a, N, ar_ea, ar_vec, gid(atom.batch[ar_ei[0]]))    # residue <- atom
        c['aa'] = self._csr(aa_ei[0] + o_a, aa_ei[1] + o_a, N, aa_ea, aa_vec, gid(atom.batch[aa_ei[0]]))
        c['ar'] = self._csr(ar_ei[0] + o_a, ar_ei[1] + o_r, N, ar_ea, ar_vec, gid(atom.batch[ar_ei[0]]))    # atom <- residue
        c['rec_ptr'], c['atom_ptr'] = ops.segment_ptr(rec.batch, B), ops.segment_ptr(atom.batch, B)
        c['lig_ptr'] = ops.segment_ptr(lig.batch, B)
        bonds = ll.edge_index[:, lig.edge_mask].long()
        c['bonds'], c['n_bonds'] = bonds, int(bonds.shape[1])
        c['bond_batch'] = lig.batch[bonds[0]] if bonds.shape[1] else None
        # CGModel's constants (ligand / residue counts, bond CSR, capacities, lig_cnt_f, bond_lig_batch) + the atom side
        c['rr_tgt_batch'] = rec.batch[rr_ei[0]]
        self._static_sync_free(data, c)
        atom_cnt = c['atom_ptr'][1:] - c['atom_ptr'][:-1]
        lig_cnt = c['lig_ptr'][1:] - c['lig_ptr'][:-1]
        c['atom_max'] = int(atom_cnt.max()) if B else 0
        c['cap_la'] = int((lig_cnt.long() * atom_cnt.long()).sum())      # every ligand atom x every atom of its complex
        c['atom_batch32'] = _i32(atom.batch)
        c['gid32'] = {k: _i32(c[k][4]) for k in ('rr', 'ra', 'aa', 'ar')}
        if shareable:
            # the four static groups of the distinct receptors with their layer-0 group index in the nine-group list
            # (forward_groups order: ll, lr, la, rr, rl, ra, aa, al, ar) and a zero sigma row per edge
            zero = lambda g: torch.zeros(g[0].shape[0], dtype=torch.int32, device=rp.device)
            c['shared_static'] = (rt['nodes'], at['nodes'], rt['node_map'], at['node_map'],
                                  [(k, g, zero(g)) for k, g in zip((3, 8, 6, 5), u_groups) if g[0].shape[0]])
        rr._b200aa = c
        return c

    def _forward_sync_free(self, data, c):
        """The forward without a device->host read (see CGModel._forward_sync_free): ligand graph, ligand-residue and
        ligand-atom graphs written into upper-bound buffers with device-side counts; the reversed groups (residue<-ligand,
        atom<-ligand) are permutations of the forward lists and - as in the reference, models/aa_model.py:405-406 - keep the
        FORWARD direction's edge vector (vec_sign = +1); the four static groups get their sigma term inside the kernel."""
        lig, rec, atom = data['ligand'], data['receptor'], data['atom']
        ns, n_lig = self.ns, lig.batch.shape[0]
        o_r, o_a = n_lig, n_lig + rec.batch.shape[0]
        tr_sigma, rot_sigma, tor_sigma = self._sigmas(data)

        sig = self.rec_sigma_embedding(self.timestep_emb_func(data.complex_t['tr'])).contiguous()
        rec_node, atom_node = rec.rec_node_attr.clone(), atom.atom_node_attr.clone()
        rec_node[:, :ns] += sig[rec.batch]
        atom_node[:, :ns] += sig[atom.batch]
        lig_node, g_ll = self._ligand_graph_sync_free(data, c)        # models/aa_model.py:538-568 = cg_model.py:467-497

        # -- ligand cross graphs (:588-623): residues within the (per-complex) cut-off, atoms within lig_max_radius ---------
        r, rpg = cross_cutoff(self, tr_sigma)
        g_lr, g_rl = self._cross_graph_sync_free(data, c, rec.pos.float().contiguous(), c['rec_ptr'], c['rec_batch32'],
                                                 c['rec_max'], c['cap_cross'], r, rpg, o_r, self.lr_edge_embedding,
                                                 self.cross_distance_expansion, vec_sign=1.0)
        g_la, g_al = self._cross_graph_sync_free(data, c, atom.pos.float().contiguous(), c['atom_ptr'], c['atom_batch32'],
                                                 c['atom_max'], c['cap_la'], float(self.lig_max_radius), None, o_a,
                                                 self.la_edge_embedding, self.lig_distance_expansion, vec_sign=1.0)

        # -- joint graph [ligand | residues | atoms]: nine groups in the reference's order (:401-417) --------------------
        node = torch.cat([lig_node, rec_node, atom_node], 0)
        stat = lambda k: (c[k][0], c[k][1], c[k][2], c[k][3], None, dict(ea_add=sig, ea_add_idx=c['gid32'][k]))
        groups = [g_ll, g_lr, g_la, stat('rr'), g_rl, stat('ra'), stat('aa'), g_al, stat('ar')]
        shared = self._shared_static_messages(data, c, node, sig, o_r, o_a)
        node = self._interaction_layers(node, groups, 3, shared=(shared, (3, 5, 6, 8)) if shared is not None else None)
        return self._heads(data, c, node[:n_lig], tr_sigma, rot_sigma, tor_sigma, sync_free=True)

    def _shared_static_messages(self, data, c, node, sig, o_r, o_a):
        """Layer-0 messages of the four static groups (residue<-residue, residue<-atom, atom<-atom, atom<-residue) when the
        batch holds copies of the same receptors at ONE diffusion time (``data._uniform_t``, the sampler's promise): their
        node features (static embedding + sigma embedding) and edge attributes are then the same in every copy, so they
        are accumulated once over the distinct receptors and added to every copy's rows (CGModel._shared_receptor_messages
        does the same for the residue graph).  ``node``: the joint features [ligand | residues | atoms] entering layer 0.
        None when there is nothing to share."""
        if 'shared_static' not in c or not getattr(data, '_uniform_t', False):
            return None
        rows_r, rows_a, map_r, map_a, u_groups = c['shared_static']
        layer = self.conv_layers[0]
        x0 = torch.cat([node[o_r + rows_r], node[o_a + rows_a]], 0)
        n_u, nr_u = x0.shape[0], rows_r.shape[0]
        acc = ops.new_accumulators(n_u, layer.out_size, x0.device)
        s0 = sig[:1].contiguous()
        for k, g, zero in u_groups:
            acc = layer.accumulate_group(x0, g + (None, dict(ea_add=s0, ea_add_idx=zero)), k, n_u, gather_scalars=self.ns,
                                         init=acc)
        sum_buf, cnt_buf = ops.new_accumulators(node.shape[0], layer.out_size, x0.device)
        sum_buf[o_r:o_a].add_(acc[0][:nr_u][map_r])
        sum_buf[o_a:].add_(acc[0][nr_u:][map_a])
        cnt_buf[o_r:o_a].add_(acc[1][:nr_u][map_r])
        cnt_buf[o_a:].add_(acc[1][nr_u:][map_a])
        return sum_buf, cnt_buf

    def _forward_host_sized(self, data, c):
        """Forward with exactly-sized neighbour lists (the sizes are read back to the host)."""
        lig, rec, atom = data['ligand'], data['receptor'], data['atom']
        ns = self.ns
        tr_sigma, rot_sigma, tor_sigma = self._sigmas(data)
        n_lig, n_rec = lig.pos.shape[0], rec.pos.shape[0]
        o_r, o_a = n_lig, n_lig + n_rec

        # -- embeddings (:335-362): sigma term on residue / atom scalars and on the three static edge-attribute sets ----
        sig = self.rec_sigma_embedding(self.timestep_emb_func(data.complex_t['tr']))
        rec_node, atom_node = rec.rec_node_attr.clone(), atom.atom_node_attr.clone()
        rec_node[:, :ns] += sig[rec.batch]
        atom_node[:, :ns] += sig[atom.batch]
        lig_x, ll_tgt, ll_src, ll_ea, ll_vec, _ = self._ligand_graph(data, c)
        lig_node = self.lig_node_embedding(lig_x)
        ll_ea = self.lig_edge_embedding(ll_ea)
        assert self.embed_also_ligand, "otherwise reimplement padding"
        g_ll = (_i32(ll_tgt), _i32(ll_src), ll_ea, ll_vec.contiguous(), None)
        for layer in self.lig_emb_layers:
            lig_node = layer.forward_groups(lig_node, [g_ll], gather_scalars=ns)

        # -- ligand cross graphs (:588-623): residues within the (per-complex) cut-off, atoms within lig_max_radius ---------
        r, rpg = cross_cutoff(self, tr_sigma)
        li, ri, lr_ea, lr_vec, _ = cross_graph(self, data, rec.pos.float(), c['rec_ptr'], r, rpg,
                                               self.cross_distance_expansion, self.lr_edge_embedding)
        la_l, la_a, la_ea, la_vec, _ = cross_graph(self, data, atom.pos.float(), c['atom_ptr'], float(self.lig_max_radius),
                                                   None, self.lig_distance_expansion, self.la_edge_embedding)

        # -- joint graph [ligand | residues | atoms]: nine groups in the reference's order (:401-417) --------------------
        node = torch.cat([lig_node, rec_node, atom_node], 0)
        rl_tgt, rl_rev = torch.sort(ri, stable=True)                 # residue <- ligand: same pairs sorted by residue
        al_tgt, al_rev = torch.sort(la_a, stable=True)               # atom <- ligand
        stat = lambda k: (c[k][0], c[k][1], c[k][2] + sig[c[k][4]], c[k][3], None)
        groups = [
            g_ll,                                                                                        # ligand <- ligand
            (_i32(li), _i32(ri + o_r), lr_ea, lr_vec.contiguous(), None),                                # ligand <- residue
            (_i32(la_l), _i32(la_a + o_a), la_ea, la_vec.contiguous(), None),                            # ligand <- atom
            stat('rr'),                                                                                  # residue <- residue
            (_i32(rl_tgt + o_r), _i32(li[rl_rev]), lr_ea[rl_rev], lr_vec[rl_rev].contiguous(), None),    # residue <- ligand (forward Y)
            stat('ra'),                                                                                  # residue <- atom   (forward Y)
            stat('aa'),                                                                                  # atom <- atom
            (_i32(al_tgt + o_a), _i32(la_l[al_rev]), la_ea[al_rev], la_vec[al_rev].contiguous(), None),  # atom <- ligand    (forward Y)
            stat('ar'),                                                                                  # atom <- residue
        ]
        node = self._interaction_layers(node, groups, 3, merge=not self.differentiate_convolutions)
        return self._heads(data, c, node[:n_lig], tr_sigma, rot_sigma, tor_sigma, sync_free=False)
