"""Drop-in for the reference's confidence model ``models/old_cg_model.py:CGOldModel`` in confidence mode - the ranking
model ``utils/sampling.py:208-227`` calls once per batch of final poses (SURVEY.md section 8, row f2).

Same constructor keywords, ``forward(data) -> confidence [B]`` (``[B, 2]`` with affinity_prediction) and ``state_dict``
keys as the reference class for: confidence_mode=True, use_old_atom_encoder=True (the only encoder the reference class
can be built with - its new AtomEncoder rejects the ``lm_embedding_type`` keyword, models/old_cg_model.py:63-66), no
miscellaneous atoms, one noise schedule.  The convolutions are the same sm_90a kernels as the score model's: every
OldTensorProductConvLayer call goes through the fully fused wgmma kernel (csrc/fused_conv.cu) when its shapes allow,
neighbour lists come from ddb200_radius_*, spherical harmonics are evaluated in-kernel from the edge vectors.

CUDA only, inference only.  No CPU fallback.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F
from torch import nn

from . import ops
from .irreps import irreps_str, sh_irreps
from .layers import (GaussianSmearing, OldAtomEncoder, _mlp, check_forward, confidence_head, cross_cutoff, cross_graph,
                     edge_weight, ligand_graph)
from .synthetic import LIG_FEATURE_DIMS as lig_feature_dims, REC_RESIDUE_FEATURE_DIMS as rec_residue_feature_dims
from .tensor_layers import OldTensorProductConvLayer


class CGOldModel(nn.Module):
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
        if not confidence_mode:
            raise NotImplementedError("diffdock_b200.CGOldModel is built in confidence mode only (SURVEY.md row f2); "
                                      "the score model is diffdock_b200.cg_model.CGModel")
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
        bn = (lambda: nn.Identity()) if confidence_no_batchnorm else (lambda: nn.BatchNorm1d(ns))
        self.confidence_predictor = nn.Sequential(
            nn.Linear(2 * ns if num_conv_layers >= 3 else ns, ns), bn(), nn.ReLU(), nn.Dropout(confidence_dropout),
            nn.Linear(ns, ns), bn(), nn.ReLU(), nn.Dropout(confidence_dropout),
            nn.Linear(ns, 2 if affinity_prediction else 1))

    def load_state_dict(self, state_dict, strict=True, **kw):
        """Reference checkpoints carry e3nn's tensor-product buffers (``*.tp.*``): dropped, the kernels have their own tables."""
        sd = {k: v for k, v in state_dict.items() if '.tp.' not in k}
        return super().load_state_dict(sd, strict=strict, **kw)

    def get_edge_weight(self, edge_vec, max_norm):                      # models/old_cg_model.py:353-359
        return edge_weight(edge_vec, max_norm, self.smooth_edges)

    @torch.no_grad()
    def forward(self, data):                                            # models/old_cg_model.py:203-301
        check_forward(self, data)
        lig, rec = data['ligand'], data['receptor']
        B, ns = data.num_graphs, self.ns
        tr_sigma = data.complex_t['tr']                                 # confidence mode: times are used as they are
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
        return confidence_head(self, data, lig_node)
