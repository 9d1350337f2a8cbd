"""Oracle restatement of models/old_cg_model.py (CGOldModel) in SCORE MODE - the v1.0 score model that
``inference.py --old_score_model`` builds.  TEST INFRASTRUCTURE (CPU, plain PyTorch).

The graphs and the four convolutions per layer are those of the confidence-mode oracle (oracle/old_cg_model.py,
models/old_cg_model.py:203-294), which this class extends; the score heads (:303-351) are those of models/cg_model.py,
which oracle/cg_model.py restates.  Same constructor keywords and state_dict keys as the reference class in score mode (:156-201)."""
import torch
import torch.nn.functional as F
from torch import nn

from oracle import e3nn_lite as o3
from oracle.cg_model import CGModel
from oracle.layers import GaussianSmearing, OldAtomEncoder
from oracle.old_cg_model import LIG_FEATURE_DIMS, REC_RESIDUE_FEATURE_DIMS, CGOldModel, _mlp
from oracle.tensor_layers import OldTensorProductConvLayer


class CGOldScoreModel(CGOldModel):
    _dtype, _temb = CGModel._dtype, CGModel._temb
    build_center_conv_graph, build_bond_conv_graph, _heads = (CGModel.build_center_conv_graph, CGModel.build_bond_conv_graph,
                                                              CGModel._heads)

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
        # the modules of oracle/old_cg_model.py up to its confidence predictor, created in the reference's order (:63-201)
        # so that a seeded construction draws the reference's initial weights
        nn.Module.__init__(self)
        assert parallel == 1 and not confidence_mode, "score mode; the confidence mode is oracle.old_cg_model.CGOldModel"
        assert use_old_atom_encoder and not include_miscellaneous_atoms, "oracle subset"
        assert not (separate_noise_schedule or asyncronous_noise_schedule or use_second_order_repr), "oracle subset"
        self.t_to_sigma, self.device, self.timestep_emb_func = t_to_sigma, device, timestep_emb_func
        self.in_lig_edge_features, self.sigma_embed_dim = in_lig_edge_features, sigma_embed_dim
        self.lig_max_radius, self.rec_max_radius = lig_max_radius, rec_max_radius
        self.cross_max_distance, self.dynamic_max_cross = cross_max_distance, dynamic_max_cross
        self.sh_irreps = o3.Irreps.spherical_harmonics(lmax=sh_lmax)
        self.ns, self.nv, self.smooth_edges = ns, nv, smooth_edges
        self.confidence_mode, self.num_conv_layers = False, num_conv_layers
        self.no_aminoacid_identities = no_aminoacid_identities
        self.scale_by_sigma, self.no_torsion, self.odd_parity = scale_by_sigma, no_torsion, odd_parity
        self.fixed_center_conv = fixed_center_conv
        kw = dict(lm_embedding_dim=lm_embedding_dim) if lm_embedding_type is not None else {}
        self.lig_node_embedding = OldAtomEncoder(ns, LIG_FEATURE_DIMS, sigma_embed_dim)
        self.lig_edge_embedding = _mlp(in_lig_edge_features + sigma_embed_dim + distance_embed_dim, ns, ns, dropout)
        self.rec_node_embedding = OldAtomEncoder(ns, REC_RESIDUE_FEATURE_DIMS, sigma_embed_dim,
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
            lig.append(OldTensorProductConvLayer(**p))
            rec.append(OldTensorProductConvLayer(**p))
            l2r.append(OldTensorProductConvLayer(**p))
            r2l.append(OldTensorProductConvLayer(**p))
        self.lig_conv_layers, self.rec_conv_layers = nn.ModuleList(lig), nn.ModuleList(rec)
        self.lig_to_rec_conv_layers, self.rec_to_lig_conv_layers = nn.ModuleList(l2r), nn.ModuleList(r2l)
        S, D = sigma_embed_dim, distance_embed_dim                      # :156-201
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
            self.final_tp_tor = o3.FullTensorProduct(self.sh_irreps, "2e")
            self.tor_bond_conv = OldTensorProductConvLayer(in_irreps=self.lig_conv_layers[-1].out_irreps,
                                                           sh_irreps=self.final_tp_tor.irreps_out,
                                                           out_irreps=f'{ns}x0o + {ns}x0e' if not odd_parity else f'{ns}x0o',
                                                           n_edge_features=3 * ns, residual=False, dropout=dropout,
                                                           batch_norm=batch_norm)
            self.tor_final_layer = nn.Sequential(nn.Linear(2 * ns if not odd_parity else ns, ns, bias=False), nn.Tanh(),
                                                 nn.Dropout(dropout), nn.Linear(ns, 1, bias=False))

    def forward(self, data):                                            # :203-351
        if self.no_aminoacid_identities:
            data['receptor'].x = data['receptor'].x * 0
        tr_sigma, rot_sigma, tor_sigma = self.t_to_sigma(*[data.complex_t[k] for k in ('tr', 'rot', 'tor')])
        ns = self.ns
        lig_node, lig_ei, lig_ea, lig_sh, lig_ew = self.build_lig_conv_graph(data)
        lig_src, lig_dst = lig_ei
        lig_node, lig_ea = self.lig_node_embedding(lig_node), self.lig_edge_embedding(lig_ea)
        rec_node, rec_ei, rec_ea, rec_sh, rec_ew = self.build_rec_conv_graph(data)
        rec_src, rec_dst = rec_ei
        rec_node, rec_ea = self.rec_node_embedding(rec_node), self.rec_edge_embedding(rec_ea)
        cutoff = (tr_sigma * 3 + 20).unsqueeze(1) if self.dynamic_max_cross else self.cross_max_distance
        lr_ei, lr_ea, lr_sh, lr_ew = self.build_cross_conv_graph(data, cutoff)
        cross_lig, cross_rec = lr_ei
        lr_ea = self.cross_edge_embedding(lr_ea)
        L = len(self.lig_conv_layers)
        for l in range(L):
            ea_ = torch.cat([lig_ea, lig_node[lig_src, :ns], lig_node[lig_dst, :ns]], -1)
            lig_intra = self.lig_conv_layers[l](lig_node, lig_ei, ea_, lig_sh, edge_weight=lig_ew)
            ea_ = torch.cat([lr_ea, lig_node[cross_lig, :ns], rec_node[cross_rec, :ns]], -1)
            lig_inter = self.rec_to_lig_conv_layers[l](rec_node, lr_ei, ea_, lr_sh, out_nodes=lig_node.shape[0],
                                                       edge_weight=lr_ew)
            if l != L - 1:
                ea_ = torch.cat([rec_ea, rec_node[rec_src, :ns], rec_node[rec_dst, :ns]], -1)
                rec_intra = self.rec_conv_layers[l](rec_node, rec_ei, ea_, rec_sh, edge_weight=rec_ew)
                ea_ = torch.cat([lr_ea, lig_node[cross_lig, :ns], rec_node[cross_rec, :ns]], -1)
                rec_inter = self.lig_to_rec_conv_layers[l](lig_node, torch.flip(lr_ei, dims=[0]), ea_, lr_sh,
                                                           out_nodes=rec_node.shape[0], edge_weight=lr_ew)
            lig_node = F.pad(lig_node, (0, lig_intra.shape[-1] - lig_node.shape[-1])) + lig_intra + lig_inter
            if l != L - 1:
                rec_node = F.pad(rec_node, (0, rec_intra.shape[-1] - rec_node.shape[-1])) + rec_intra + rec_inter
        return self._heads(data, lig_node, tr_sigma, rot_sigma, tor_sigma)[:3]      # (tr, rot, tor)
