"""Drop-in for the reference's ``models/old_cg_model.py:CGOldModel``, the DiffDock v1.0 architecture, in both modes:

* confidence mode - the ranking model ``utils/sampling.py:208-227`` calls once per batch of final poses (SURVEY.md
  section 8, row f2): ``forward(data) -> confidence [B]`` (``[B, 2]`` with affinity_prediction);
* score mode - the v1.0 score model (``inference.py --old_score_model``): ``forward(data) -> (tr [B, 3], rot [B, 3],
  tor [n_rotatable_bonds])``, the reference's 3-tuple.

Same constructor keywords and ``state_dict`` keys as the reference class for: use_old_atom_encoder=True (the only encoder the
reference class can be built with - its new AtomEncoder rejects the ``lm_embedding_type`` keyword,
models/old_cg_model.py:63-66), no miscellaneous atoms, one noise schedule.  The convolutions are the same sm_90a kernels as
the v1.1 score model's: every OldTensorProductConvLayer call goes through the fully fused wgmma kernel (csrc/fused_conv.cu)
when its shapes allow, neighbour lists come from ddb200_radius_* / ddb200_graph_fill, spherical harmonics are evaluated
in-kernel from the edge vectors.

Score mode follows diffdock_b200.cg_model.CGModel: per-batch constants in ``_static``, a forward without any device->host
read (``_forward_sync_free``, capturable in a CUDA graph by diffdock_b200.sampling) when every convolution has a fused-kernel
shape, else ``_forward_host_sized``.  What the v1.0 wiring changes on that path (models/old_cg_model.py:203-351):

1. sigma enters the receptor embeddings.  The node encoder is affine in the sigma embedding, so its sigma-free part
   (including the 1280-wide language-model Linear) is computed once per batch and each step adds ``M . sigma_emb`` per
   complex (``M`` [ns, S] folded from the encoder's weights); the contact-edge embedding runs in ddb200_edge_embed with
   the sigma half of its first Linear applied per complex.  A batch of B poses of one receptor at one time embeds one
   copy's contact graph and the copies read it through ``edge_perm``.
2. Four convolutions per layer, each with its own radial MLP, mean and BatchNorm, residual=False: each is one fused launch
   over the joint [ligand | residues] numbering into one of two accumulators (intra: lig<-lig and rec<-rec; inter:
   lig<-rec and rec<-lig), and two chained ddb200_tpconv_finalize calls per node type give
   ``pad(x) + BN_intra(mean_intra) + BN_inter(mean_inter)``.  The receptor is not updated in the last layer.
3. The rec<-lig convolution reads ``[ea | node[lig] | node[rec]]`` while its target is the residue: the two node blocks of
   its first Linear are swapped in the kernel plan (TensorProductConvLayer._fused_plan).
4. rec<-lig uses Y(rec - lig) unnegated (:265): the reverse permutation of the cross list with ``vec_sign = +1``.
5. Layer-0 rec<-rec messages of a batch of repeated receptors at one time are computed once per distinct receptor and
   added to all copies.

Confidence mode runs the same sync-free forward with the times as sigmas, then the one-kernel confidence head; where its
conditions fail it keeps the host-sized forward.

CUDA only, inference only.  No CPU fallback.
"""
from __future__ import annotations

import os
import weakref

import numpy as np
import torch
import torch.nn.functional as F
from torch import nn

from . import ops
from .cg_model import _TABLES, CGModel, _flat, _i32, receptor_tiles
from .irreps import irreps_str, sh_irreps
from .layers import (GaussianSmearing, OldAtomEncoder, _mlp, check_confidence_widths, check_forward, confidence_head,
                     cross_cutoff, cross_graph, edge_weight, ligand_graph, score_heads)
from .synthetic import LIG_FEATURE_DIMS as lig_feature_dims, REC_RESIDUE_FEATURE_DIMS as rec_residue_feature_dims
from .tensor_layers import OldTensorProductConvLayer
from .tp_table import full_tensor_product


def sigma_map(enc, S, x_cols):
    """``M`` [ns, S] with enc(cat[x, s]) = enc(cat[x, 0]) + M s for the OldAtomEncoder ``enc`` and its input
    ``cat[x (x_cols columns), sigma embedding (S columns)]``: the encoder reads its scalar columns and (with an LM embedding)
    the last ``lm_embedding_dim`` columns of that input (models/layers.py:103-116); the sigma columns can fall in either."""
    nc, nsf = enc.num_categorical_features, enc.num_scalar_features
    cols = torch.arange(x_cols, x_cols + S)                              # where the sigma embedding sits
    W = enc.linear.weight.detach()
    m = W.new_zeros((W.shape[0], S))
    j = cols - nc
    ok = (j >= 0) & (j < nsf)
    m[:, ok] = W[:, j[ok]]
    if enc.lm_embedding_type is not None:
        W_lm, lm = enc.lm_embedding_layer.weight.detach(), enc.lm_embedding_dim
        m = W_lm[:, :W.shape[0]] @ m
        j = cols - (x_cols + S - lm)
        ok = j >= 0
        m[:, ok] += W_lm[:, W.shape[0] + j[ok]]
    return m.contiguous()


class CGOldModel(nn.Module):
    # The ligand and cross graphs, the score-norm look-ups and the per-batch constants of the sync-free path are the v1.1
    # score model's (models/old_cg_model.py:361-391,439-461 = models/cg_model.py:467-497,539-562).
    _static_sync_free = CGModel._static_sync_free
    _ligand_edges_sync_free = CGModel._ligand_edges_sync_free
    _cross_graph_sync_free = CGModel._cross_graph_sync_free
    _cross_edge_embedding = CGModel._cross_edge_embedding
    _edge_embed_in_kernel = CGModel._edge_embed_in_kernel
    _so3_score_norm, _torus_score_norm = CGModel._so3_score_norm, CGModel._torus_score_norm
    set_score_norm_tables = CGModel.set_score_norm_tables

    def __init__(self, t_to_sigma, device, timestep_emb_func, in_lig_edge_features=4, sigma_embed_dim=32, sh_lmax=2,
                 ns=16, nv=4, num_conv_layers=2, lig_max_radius=5, rec_max_radius=30, cross_max_distance=250,
                 center_max_distance=30, distance_embed_dim=32, cross_distance_embed_dim=32, no_torsion=False,
                 scale_by_sigma=True, norm_by_sigma=True, use_second_order_repr=False, batch_norm=True,
                 dynamic_max_cross=False, dropout=0.0, smooth_edges=False, odd_parity=False,
                 separate_noise_schedule=False, lm_embedding_type=None, confidence_mode=False, confidence_dropout=0,
                 confidence_no_batchnorm=False, asyncronous_noise_schedule=False, affinity_prediction=False, parallel=1,
                 parallel_aggregators="mean max min std", num_confidence_outputs=1, fixed_center_conv=False,
                 no_aminoacid_identities=False, include_miscellaneous_atoms=False, use_old_atom_encoder=False,
                 lm_embedding_dim=1280):
        super().__init__()
        assert parallel == 1, "not implemented"
        assert (not no_aminoacid_identities) or (lm_embedding_type is None), "no language model emb without identities"
        if not use_old_atom_encoder:
            raise NotImplementedError("models/old_cg_model.py can only be constructed with use_old_atom_encoder=True")
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
        self.scale_by_sigma, self.no_torsion, self.odd_parity = scale_by_sigma, no_torsion, odd_parity
        self.fixed_center_conv = fixed_center_conv
        kw = dict(lm_embedding_dim=lm_embedding_dim) if lm_embedding_type is not None else {}
        self.lig_node_embedding = OldAtomEncoder(ns, lig_feature_dims, sigma_embed_dim)
        self.lig_edge_embedding = _mlp(in_lig_edge_features + sigma_embed_dim + distance_embed_dim, ns, ns, dropout)
        self.rec_node_embedding = OldAtomEncoder(ns, rec_residue_feature_dims, sigma_embed_dim,
                                                 lm_embedding_type=lm_embedding_type, **kw)
        self.rec_edge_embedding = _mlp(sigma_embed_dim + distance_embed_dim, ns, ns, dropout)
        self.cross_edge_embedding = _mlp(sigma_embed_dim + cross_distance_embed_dim, ns, ns, dropout)
        self.lig_distance_expansion = GaussianSmearing(0.0, lig_max_radius, distance_embed_dim)
        self.rec_distance_expansion = GaussianSmearing(0.0, rec_max_radius, distance_embed_dim)
        self.cross_distance_expansion = GaussianSmearing(0.0, cross_max_distance, cross_distance_embed_dim)
        seq = [f'{ns}x0e', f'{ns}x0e + {nv}x1o', f'{ns}x0e + {nv}x1o + {nv}x1e',
               f'{ns}x0e + {nv}x1o + {nv}x1e + {ns}x0o']
        lig, rec, l2r, r2l = [], [], [], []
        for i in range(num_conv_layers):
            p = dict(in_irreps=seq[min(i, 3)], sh_irreps=self.sh_irreps, out_irreps=seq[min(i + 1, 3)],
                     n_edge_features=3 * ns, hidden_features=3 * ns, residual=False, batch_norm=batch_norm,
                     dropout=dropout)
            lig.append(OldTensorProductConvLayer(**p))           # creation order of the reference (:118-125)
            rec.append(OldTensorProductConvLayer(**p))
            l2r.append(OldTensorProductConvLayer(**p))
            r2l.append(OldTensorProductConvLayer(**p))
        self.lig_conv_layers, self.rec_conv_layers = nn.ModuleList(lig), nn.ModuleList(rec)
        self.lig_to_rec_conv_layers, self.rec_to_lig_conv_layers = nn.ModuleList(l2r), nn.ModuleList(r2l)
        self._sync_free = None
        if confidence_mode:
            bn = (lambda: nn.Identity()) if confidence_no_batchnorm else (lambda: nn.BatchNorm1d(ns))
            self.confidence_predictor = nn.Sequential(
                nn.Linear(2 * ns if num_conv_layers >= 3 else ns, ns), bn(), nn.ReLU(), nn.Dropout(confidence_dropout),
                nn.Linear(ns, ns), bn(), nn.ReLU(), nn.Dropout(confidence_dropout),
                nn.Linear(ns, 2 if affinity_prediction else 1))
            self._conf_tail = ns if num_conv_layers >= 3 else 0
            check_confidence_widths(self)
            return
        # score mode: translation / rotation and torsion heads (:156-201)
        S, D = sigma_embed_dim, distance_embed_dim
        self.center_distance_expansion = GaussianSmearing(0.0, center_max_distance, D)
        self.center_edge_embedding = _mlp(D + S, ns, ns, dropout)
        self.final_conv = OldTensorProductConvLayer(in_irreps=self.lig_conv_layers[-1].out_irreps, sh_irreps=self.sh_irreps,
                                                    out_irreps='2x1o + 2x1e' if not odd_parity else '1x1o + 1x1e',
                                                    n_edge_features=2 * ns, residual=False, dropout=dropout,
                                                    batch_norm=batch_norm)
        self.tr_final_layer = nn.Sequential(nn.Linear(1 + S, ns), nn.Dropout(dropout), nn.ReLU(), nn.Linear(ns, 1))
        self.rot_final_layer = nn.Sequential(nn.Linear(1 + S, ns), nn.Dropout(dropout), nn.ReLU(), nn.Linear(ns, 1))
        if not no_torsion:
            self.final_edge_embedding = _mlp(D, ns, ns, dropout)
            T, tor_sh = full_tensor_product(self.sh_irreps, '1x2e')       # o3.FullTensorProduct(sh, "2e"), :186
            self.register_buffer('_tor_tp', torch.from_numpy(T).float(), persistent=False)
            self.tor_bond_conv = OldTensorProductConvLayer(in_irreps=self.lig_conv_layers[-1].out_irreps,
                                                           sh_irreps=irreps_str(tor_sh),
                                                           out_irreps=f'{ns}x0o + {ns}x0e' if not odd_parity else f'{ns}x0o',
                                                           n_edge_features=3 * ns, residual=False, dropout=dropout,
                                                           batch_norm=batch_norm)
            self.tor_final_layer = nn.Sequential(nn.Linear(2 * ns if not odd_parity else ns, ns, bias=False), nn.Tanh(),
                                                 nn.Dropout(dropout), nn.Linear(ns, 1, bias=False))
        z = np.load(_TABLES)        # score-norm tables (utils/so3.py:59, utils/torus.py:72-76), not in the state_dict
        self.register_buffer('_so3_table', torch.from_numpy(z['so3_exp_score_norms']).float(), persistent=False)
        self.register_buffer('_torus_table', torch.from_numpy(z['torus_score_norm']).float(), persistent=False)

    def load_state_dict(self, state_dict, strict=True, **kw):
        """Reference checkpoints carry e3nn's tensor-product buffers (``*.tp.*``, and ``final_tp_tor.*`` in score mode):
        dropped, the kernels have their own tables."""
        sd = {k: v for k, v in state_dict.items() if '.tp.' not in k and not k.startswith('final_tp_tor.')}
        return super().load_state_dict(sd, strict=strict, **kw)

    def get_edge_weight(self, edge_vec, max_norm):                      # models/old_cg_model.py:353-359
        return edge_weight(edge_vec, max_norm, self.smooth_edges)

    @torch.no_grad()
    def forward(self, data):                                            # models/old_cg_model.py:203-351
        check_forward(self, data)
        if self.confidence_mode:                                        # times are used as they are (:210)
            if self.sync_free_capable():
                c = self._static(data)
                if c['rec_max'] <= 10000:
                    return confidence_head(self, self._forward_sync_free(data, c, data.complex_t['tr']), c['lig_ptr'])[0]
            lig_node = self._forward_host_sized(data, data.complex_t['tr'])
            return confidence_head(self, lig_node, ops.segment_ptr(data['ligand'].batch, data.num_graphs))[0]
        c = self._static(data)
        tr_sigma, rot_sigma, tor_sigma = self.t_to_sigma(*[data.complex_t[k] for k in ('tr', 'rot', 'tor')])
        sync_free = self.sync_free_capable() and c['rec_max'] <= 10000      # the cross graph's cap (:445) must not bind
        lig_node = self._forward_sync_free(data, c, tr_sigma) if sync_free else self._forward_host_sized(data, tr_sigma)
        return score_heads(self, data, c, lig_node, tr_sigma, rot_sigma, tor_sigma, sync_free)

    def sync_free_capable(self):
        """The forward runs without any host synchronisation after the per-batch constants (and so, in score mode, inside
        a CUDA graph) when every convolution of the stack has a shape the fully fused kernel supports."""
        if self._sync_free is None:
            ok = os.environ.get('DDB200_SYNC_FREE', '1') != '0'
            for convs in (self.lig_conv_layers, self.rec_conv_layers, self.lig_to_rec_conv_layers, self.rec_to_lig_conv_layers):
                ok = ok and all(layer.fused_capable(self.ns, self.ns) for layer in convs)
            self._sync_free = bool(ok)
        return self._sync_free

    def sync_free_crop_capable(self):
        """Per-step receptor cropping is not built into the sync-free v1.0 forward: ``crop_beyond`` runs the eager
        ``sampling.crop_receptor`` path."""
        return False

    # ---------------------------------------------------------------------------------------------------------
    def _static(self, data):
        """Per-batch constants of the score model, cached on ``data`` (one host read per batch): the sigma-free part of the
        receptor node embedding, the contact graph in CSR order by target, and those of CGModel._static_sync_free."""
        rec, rr, lig, ll = data['receptor'], data['receptor', 'receptor'], data['ligand'], data['ligand', 'ligand']
        hit = getattr(rr, '_b200_v10', None)
        if hit is not None and hit[0]() is self:      # per model: the score and confidence models may share the batch
            return hit[1]
        B, n_lig, ns = data.num_graphs, lig.batch.shape[0], self.ns
        ei = rr.edge_index.long()
        tiles = receptor_tiles(rec, B, ei)        # copies of the same receptors: each distinct one is embedded once
        c = {'tiles': tiles}
        # receptor node embedding with the sigma embedding set to zero (:401, :221), 1280-wide LM layer included
        x1 = rec.x[tiles['nodes']].float() if tiles is not None else rec.x.float()
        base = self.rec_node_embedding(torch.cat([x1, x1.new_zeros((x1.shape[0], self.sigma_embed_dim))], 1))
        c['rec_base'] = base[tiles['node_map']] if tiles is not None else base
        c['rec_sigma_map'] = sigma_map(self.rec_node_embedding, self.sigma_embed_dim, rec.x.shape[1])
        c['rec_gid'] = rec.batch                # complex of each residue: the sigma terms are per complex, not per batch
        # contact graph in CSR order by target (edge_index[0]); vector gathered - target (:406)
        tgt, order = torch.sort(ei[0], stable=True)
        src = ei[1][order]
        pos = rec.pos.float()
        vec = (pos[src] - pos[tgt]).contiguous()
        ew = self.get_edge_weight(vec, self.rec_max_radius)
        c['rr_tgt'], c['rr_src'], c['rr_vec'] = tgt, src, vec
        c['rr_ew'] = _flat(ew)
        c['rr_tgt_batch'] = rec.batch[tgt]
        c['rr_joint'] = (_i32(tgt + n_lig), _i32(src + n_lig))
        if tiles is not None:   # copy 0 of each distinct receptor's sorted contact graph, numbered as tiles['nodes']
            rows, shift = tiles['sorted_rows'], tiles['sorted_shift']
            c['rr0'] = (_i32(tgt[rows] - shift), _i32(src[rows] - shift), vec[rows].contiguous(),
                        c['rr_ew'][rows].contiguous() if c['rr_ew'] is not None else None)
            c['rr0_row'] = torch.zeros(rows.shape[0], dtype=torch.int32, device=vec.device)
            c['rr_perm'] = _i32(tiles['edge_map'])     # sorted row -> copy-0 row (a copy's sorted order is copy 0's)
        c['rec_ptr'] = ops.segment_ptr(rec.batch, B)
        c['lig_ptr'] = ops.segment_ptr(lig.batch, B)
        bonds = ll.edge_index[:, lig.edge_mask].long()
        c['bonds'], c['n_bonds'] = bonds, int(bonds.shape[1])
        c['bond_batch'] = lig.batch[bonds[0]] if bonds.shape[1] else None
        self._static_sync_free(data, c)
        rr._b200_v10 = (weakref.ref(self), c)
        return c

    def _forward_sync_free(self, data, c, tr_sigma):
        """Ligand node features after the interaction layers without a device->host read: capacity buffers with device
        counts for the ligand and cross graphs (as CGModel._forward_sync_free), the receptor embeddings from the per-batch
        constants plus the per-complex sigma terms, four fused convolutions per layer finalised per node type."""
        lig, rec = data['ligand'], data['receptor']
        ns, n_lig, B = self.ns, lig.batch.shape[0], data.num_graphs
        shared = c['tiles'] is not None and getattr(data, '_uniform_t', False)     # repeated receptors at one time
        sig = self.timestep_emb_func(data.complex_t['tr'])                    # [B, S], per complex

        # -- receptor embeddings (:393-414) -------------------------------------------------------------------------------
        rec_node = c['rec_base'] + (sig @ c['rec_sigma_map'].t())[c['rec_gid']]
        if shared:      # one copy's contact edges; the other copies read them through edge_perm
            t0, s0, vec0, ew0 = c['rr0']
            ea0 = self._rec_edge_attr(sig[:1], vec0, c['rr0_row'])
            g_rr = (*c['rr_joint'], ea0, vec0, ew0, dict(edge_perm=c['rr_perm']))
        else:
            g_rr = (*c['rr_joint'], self._rec_edge_attr(sig, c['rr_vec'], c['rr_gid32']), c['rr_vec'], c['rr_ew'], {})

        # -- ligand graph (:361-391) and cross graph (:439-461) ----------------------------------------------------------
        g_ll = self._ligand_edges_sync_free(data, c)
        lig_node = self.lig_node_embedding(torch.cat([lig.x.float(), lig.node_sigma_emb], 1))
        r, rpg = cross_cutoff(self, tr_sigma)
        # rec <- lig reuses the lig <- rec attributes and harmonics Y(rec - lig) (:264-265): vec_sign = +1
        g_lr, g_rl = self._cross_graph_sync_free(data, c, rec.pos.float().contiguous(), c['rec_ptr'], c['rec_batch32'],
                                                 c['rec_max'], c['cap_cross'], r, rpg, n_lig, self.cross_edge_embedding,
                                                 self.cross_distance_expansion, vec_sign=1.0)

        # -- interaction layers (:247-294) --------------------------------------------------------------------------------
        x = torch.cat([lig_node, rec_node], 0)
        L = len(self.lig_conv_layers)
        for l in range(L):
            last = l == L - 1
            n_out = n_lig if last else x.shape[0]
            D = self.lig_conv_layers[l].out_size
            intra, inter = ops.new_accumulators(n_out, D, x.device), ops.new_accumulators(n_out, D, x.device)
            self.lig_conv_layers[l].accumulate_group(x, g_ll, 0, n_out, ns, init=intra)
            self.rec_to_lig_conv_layers[l].accumulate_group(x, g_lr, 0, n_out, ns, init=inter)
            if not last:
                if l == 0 and shared:
                    self._shared_receptor_messages(x, c, n_lig, ea0, intra)
                else:
                    self.rec_conv_layers[l].accumulate_group(x, g_rr, 0, n_out, ns, init=intra)
                self.lig_to_rec_conv_layers[l].accumulate_group(x, g_rl, 0, n_out, ns, init=inter, swap_gathered=True)
            out = torch.empty((n_out, D), device=x.device)
            rows = [(slice(0, n_lig), self.lig_conv_layers[l], self.rec_to_lig_conv_layers[l])]
            if not last:
                rows.append((slice(n_lig, n_out), self.rec_conv_layers[l], self.lig_to_rec_conv_layers[l]))
            for sl, conv_a, conv_b in rows:      # pad(x) + BN_a(mean_a) + BN_b(mean_b)  (:281-290)
                part = ops.tpconv_finalize(intra[0][sl], intra[1][sl], True, *self._bn(conv_a), residual=x[sl])
                ops.tpconv_finalize(inter[0][sl], inter[1][sl], True, *self._bn(conv_b), residual=part, out=out[sl])
            x = out
        return x

    def _rec_edge_attr(self, sig, vec, row):
        """rec_edge_embedding(cat[sigma_emb of the edge's complex, rbf(|vec|)]) (:409-410, :222) with ``sig`` [rows, S] and
        ``row`` the sigma row of each edge; a receptor without contact edges (e.g. cropped to a few residues) has none."""
        if vec.shape[0] == 0:
            return vec.new_zeros((0, self.ns))
        return self._cross_edge_embedding(sig, vec, row, None, self.rec_edge_embedding, self.rec_distance_expansion)

    @staticmethod
    def _bn(layer):
        return layer.batch_norm.fold() if layer.batch_norm is not None else (None, None)

    def _shared_receptor_messages(self, x, c, n_lig, ea0, acc):
        """Layer-0 rec <- rec messages of a batch holding copies of the same receptors at ONE diffusion time
        (``data._uniform_t``): the residue features and contact edges (attributes ``ea0`` of copy 0) entering the first
        layer are the same in every copy, so the messages are computed once per distinct receptor, over the concatenated
        copy-0 graphs, and added to every copy's rows of ``acc``."""
        t0, s0, vec0, ew0 = c['rr0']
        tiles = c['tiles']
        n_u = tiles['nodes'].shape[0]
        sum0, cnt0 = self.rec_conv_layers[0].accumulate_group(x[n_lig + tiles['nodes']], (t0, s0, ea0, vec0, ew0, {}), 0,
                                                              n_u, self.ns)
        acc[0][n_lig:].add_(sum0[tiles['node_map']])
        acc[1][n_lig:].add_(cnt0[tiles['node_map']])

    def _forward_host_sized(self, data, tr_sigma):
        """Ligand node features after the interaction layers, with exactly-sized neighbour lists (one host read of each
        edge count) and every convolution through OldTensorProductConvLayer.forward: the confidence model, and the score
        model when a convolution shape is outside the fused kernel's templates."""
        lig, rec = data['ligand'], data['receptor']
        B, ns = data.num_graphs, self.ns
        rp = rec.pos.float()

        # ligand graph (:361-391): bonds + radius graph; row 0 = convolution target, row 1 = gathered node
        tgt, src, lig_ea, lig_vec, lig_ew, lig_x = ligand_graph(self, data, ops.segment_ptr(lig.batch, B))
        lig_ei = torch.stack([tgt, src])
        lig_node = self.lig_node_embedding(lig_x)
        lig_ea = self.lig_edge_embedding(lig_ea)

        # receptor graph (:393-414)
        rec.node_sigma_emb = self.timestep_emb_func(rec.node_t['tr'])
        rec_ei = data['receptor', 'receptor'].edge_index.long()
        rec_vec = rp[rec_ei[1]] - rp[rec_ei[0]]
        rec_ea = self.rec_edge_embedding(torch.cat([rec.node_sigma_emb[rec_ei[0]],
                                                    self.rec_distance_expansion(rec_vec.norm(dim=-1))], 1))
        rec_ew = self.get_edge_weight(rec_vec, self.rec_max_radius)
        rec_node = self.rec_node_embedding(torch.cat([rec.x.float(), rec.node_sigma_emb], 1))

        # cross graph (:439-461): row 0 = ligand atom, row 1 = receptor residue, vector receptor - ligand
        r, rpg = cross_cutoff(self, tr_sigma)
        li, ri, lr_ea, lr_vec, lr_ew = cross_graph(self, data, rp, ops.segment_ptr(rec.batch, B), r, rpg,
                                                   self.cross_distance_expansion, self.cross_edge_embedding)
        lr_ei, rl_ei = torch.stack([li, ri]), torch.stack([ri, li])

        L = len(self.lig_conv_layers)
        for l in range(L):
            ea_ = torch.cat([lig_ea, lig_node[lig_ei[0], :ns], lig_node[lig_ei[1], :ns]], -1)
            lig_intra = self.lig_conv_layers[l](lig_node, lig_ei, ea_, None, edge_weight=lig_ew, edge_vec=lig_vec)
            cross_ea_ = torch.cat([lr_ea, lig_node[li, :ns], rec_node[ri, :ns]], -1)
            lig_inter = self.rec_to_lig_conv_layers[l](rec_node, lr_ei, cross_ea_, None, out_nodes=lig_node.shape[0],
                                                       edge_weight=lr_ew, edge_vec=lr_vec, assume_sorted=True)
            if l != L - 1:
                ea_ = torch.cat([rec_ea, rec_node[rec_ei[0], :ns], rec_node[rec_ei[1], :ns]], -1)
                rec_intra = self.rec_conv_layers[l](rec_node, rec_ei, ea_, None, edge_weight=rec_ew, edge_vec=rec_vec)
                # ligand -> receptor messages reuse the ligand-centred attributes AND harmonics Y(receptor - ligand),
                # i.e. of the vector target - gathered (:275-276)
                rec_inter = self.lig_to_rec_conv_layers[l](lig_node, rl_ei, cross_ea_, None, out_nodes=rec_node.shape[0],
                                                           edge_weight=lr_ew, edge_vec=lr_vec)
            lig_node = F.pad(lig_node, (0, lig_intra.shape[-1] - lig_node.shape[-1])) + lig_intra + lig_inter
            if l != L - 1:
                rec_node = F.pad(rec_node, (0, rec_intra.shape[-1] - rec_node.shape[-1])) + rec_intra + rec_inter
        return lig_node
