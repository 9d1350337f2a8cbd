"""Embedding layers with the reference's parameter names (models/layers.py) - plain PyTorch modules on the device
(small dense ops; the hot convolution lives in csrc/) - and the graph plumbing the four models share."""
import math

import numpy as np
import torch
from torch import nn

from . import ops
from .tensor_layers import FCBlock  # noqa: F401  (re-export: the reference keeps FCBlock in models/layers.py)


def _mlp(n_in, n_hidden, n_out, dropout):
    return nn.Sequential(nn.Linear(n_in, n_hidden), nn.ReLU(), nn.Dropout(dropout), nn.Linear(n_hidden, n_out))


def edge_weight(edge_vec, max_norm, smooth):
    """Smooth cosine cut-off of the edges (models/cg_model.py:459); the scalar 1 when edges are not smoothed."""
    if smooth:
        nrm = torch.clip(edge_vec.norm(dim=-1) * np.pi / max_norm, max=np.pi)
        return 0.5 * (torch.cos(nrm) + 1.0).unsqueeze(-1)
    return 1.0


def check_forward(model, data):
    """What every forward checks first: inference mode and CUDA inputs; ``no_aminoacid_identities`` zeroes the residue
    features in place as the reference does."""
    name = type(model).__name__
    if model.training:
        raise RuntimeError(f"diffdock_b200.{name} is inference-only: call .eval()")
    if not data['ligand'].pos.is_cuda:
        raise RuntimeError(f"diffdock_b200.{name} runs on CUDA tensors only (no CPU fallback): data.to('cuda')")
    if model.no_aminoacid_identities:
        data['receptor'].x = data['receptor'].x * 0


def cross_cutoff(model, tr_sigma):
    """``(r, r_per_graph)`` of the ligand-receptor radius search (models/cg_model.py:321-327): 3 sigma_tr + 20 A per complex
    with ``dynamic_max_cross``, else ``cross_max_distance``."""
    if model.dynamic_max_cross:
        return 1.0, (tr_sigma * 3 + 20).reshape(-1).float().contiguous()
    return float(model.cross_max_distance), None


def edge_cutoff(r, r_per_graph, batch, row):
    """The cut-off of each edge for the smooth edge weight; ``batch[row]`` is the graph of each edge."""
    return r_per_graph[batch[row]] if r_per_graph is not None else r


def ligand_graph(model, data, lig_ptr):
    """Bond edges + radius graph of the ligand (models/cg_model.py:467-497) in their original order: ``(target, source,
    edge attribute input, vector source - target, edge weight, node input)``; sets ``node_sigma_emb`` on the ligand."""
    lig, ll = data['ligand'], data['ligand', 'ligand']
    lig.node_sigma_emb = model.timestep_emb_func(lig.node_t['tr'])
    pos = lig.pos.float()
    centre, nbr, _ = ops.radius(pos, pos, lig_ptr, lig.batch, r=model.lig_max_radius, max_num_neighbors=33,
                                exclude_self=True)      # radius_graph: cap 32 (+ self)
    tgt = torch.cat([ll.edge_index[0].long(), nbr.long()])
    src = torch.cat([ll.edge_index[1].long(), centre.long()])
    vec = pos[src] - pos[tgt]
    bond_attr = torch.cat([ll.edge_attr.float(), pos.new_zeros(nbr.shape[0], model.in_lig_edge_features)], 0)
    attr = torch.cat([bond_attr, lig.node_sigma_emb[tgt], model.lig_distance_expansion(vec.norm(dim=-1))], 1)
    node = torch.cat([lig.x.float(), lig.node_sigma_emb], 1)
    return tgt, src, attr, vec, model.get_edge_weight(vec, model.lig_max_radius), node


def cross_graph(model, data, xpos, x_ptr, r, r_per_graph, expansion, mlp):
    """Ligand <- x edges within the cut-off (x: residues or receptor atoms at ``xpos`` with segment pointers ``x_ptr``,
    models/cg_model.py:539-562), grouped by ligand atom: ``(ligand index, x index, embedded edge attributes, vector x - ligand,
    edge weight)``.  Needs ``node_sigma_emb`` on the ligand."""
    lig = data['ligand']
    lp = lig.pos.float()
    li, xi, _ = ops.radius(xpos, lp, x_ptr, lig.batch, r=r, r_per_graph=r_per_graph, max_num_neighbors=10000)
    li, xi = li.long(), xi.long()
    vec = xpos[xi] - lp[li]
    ea = mlp(torch.cat([lig.node_sigma_emb[li], expansion(vec.norm(dim=-1))], 1))
    return li, xi, ea, vec, model.get_edge_weight(vec, edge_cutoff(r, r_per_graph, lig.batch, li))


def _mlp_dims(seq):
    """(in, hidden, out) of a confidence MLP: Linear, BN / Identity, ReLU, Dropout, Linear, BN / Identity, ReLU, Dropout,
    Linear (models/cg_model.py:198-208)."""
    return seq[0].in_features, seq[0].out_features, seq[8].out_features


def check_confidence_widths(model):
    """Rejects, at construction, confidence heads wider than ddb200_confidence_head takes (DDB200_CONF_MAX_*)."""
    heads = [model.confidence_predictor] + ([model.atom_confidence_predictor] if getattr(model, 'atom_confidence', False)
                                            else [])
    for seq in heads:
        n_in, h, n_out = _mlp_dims(seq)
        if seq is not model.confidence_predictor:
            n_out -= _mlp_dims(model.confidence_predictor)[0]        # the atom outputs; the rest is pooled
        if n_in > ops.CONF_MAX_IN or h > ops.CONF_MAX_HIDDEN or n_out > ops.CONF_MAX_OUT:
            raise NotImplementedError(f"confidence head of widths in={n_in} hidden={h} out={n_out}: the confidence kernel "
                                      f"takes in <= {ops.CONF_MAX_IN}, hidden <= {ops.CONF_MAX_HIDDEN}, "
                                      f"out <= {ops.CONF_MAX_OUT}")


def _pack_mlp(seq):
    """The packed float32 MLP of ddb200_confidence_head (include/diffdock_b200.h), BatchNorm folded into (scale, shift)."""
    parts = []
    for lin, norm in ((seq[0], seq[1]), (seq[4], seq[5]), (seq[8], None)):
        parts += [lin.weight.detach().float().reshape(-1), lin.bias.detach().float()]
        if norm is None:
            continue
        if isinstance(norm, nn.BatchNorm1d):
            scale = norm.weight.detach().float() / torch.sqrt(norm.running_var.float() + norm.eps)
            shift = norm.bias.detach().float() - norm.running_mean.float() * scale
        else:                                                          # confidence_no_batchnorm: nn.Identity
            scale, shift = torch.ones_like(lin.bias).float(), torch.zeros_like(lin.bias).float()
        parts += [scale, shift]
    return torch.cat(parts).contiguous()


def _packed_heads(model):
    """Packed confidence MLPs of ``model``, rebuilt only when a parameter or buffer changed (load_state_dict, .to())."""
    seqs = [model.confidence_predictor] + ([model.atom_confidence_predictor] if getattr(model, 'atom_confidence', False)
                                           else [])
    key = tuple((t.data_ptr(), t._version) for s in seqs for t in list(s.parameters()) + list(s.buffers()))
    cache = getattr(model, '_conf_pack', None)
    if cache is None or cache[0] != key:
        cache = (key, [_pack_mlp(s) for s in seqs])
        model._conf_pack = cache
    return cache[1]


def confidence_head(model, lig_node, lig_ptr):
    """``(confidence [B] or [B, k], atom_confidence [n_lig, k_atom] or zeros [n_lig])`` of the ligand node features in one
    ddb200_confidence_head launch (models/cg_model.py:354-366, models/old_cg_model.py:296-299): the first ``ns`` columns and
    the last ``model._conf_tail`` ones, the optional per-atom head, the mean per pose, ``confidence_predictor``."""
    packs = _packed_heads(model)
    n_tail = model._conf_tail
    dims = _mlp_dims(model.confidence_predictor)
    atom = getattr(model, 'atom_confidence', False)
    x = lig_node.float()
    if x.stride(1) != 1:
        x = x.contiguous()
    conf, atom_conf = ops.confidence_head(
        x, lig_ptr, model.ns, n_tail, packs[0], dims, atom_mlp=packs[1] if atom else None,
        atom_dims=(model.atom_confidence_predictor[0].out_features, model.atom_num_confidence_outputs) if atom else None)
    if atom_conf is None:
        atom_conf = torch.zeros((lig_node.shape[0],), device=lig_node.device)
    return conf.squeeze(dim=-1), atom_conf


def _sh_l2(vec):
    """Component-normalised l=2 real spherical harmonics of the normalised vectors (o3.spherical_harmonics("2e", ...),
    models/cg_model.py:411)."""
    v = torch.nn.functional.normalize(vec, dim=-1)
    x, y, z = v[:, 0], v[:, 1], v[:, 2]
    s5, s15 = math.sqrt(5.0), math.sqrt(15.0)
    return torch.stack([s15 * x * z, s15 * x * y, s5 * (y * y - 0.5 * (x * x + z * z)), s15 * y * z,
                        0.5 * s15 * (z * z - x * x)], dim=-1)


def _sh_full(vec, lmax):
    v = torch.nn.functional.normalize(vec, dim=-1)
    cols = [torch.ones_like(v[:, :1])]
    if lmax >= 1:
        cols.append(math.sqrt(3.0) * v)
    if lmax >= 2:
        cols.append(_sh_l2(vec))
    return torch.cat(cols, dim=-1)


def score_heads(model, data, c, lig_node, tr_sigma, rot_sigma, tor_sigma, sync_free):
    """The translation / rotation and torsion heads of the score models, ``(tr [B, 3], rot [B, 3], tor [n_bonds])``
    (models/cg_model.py:368-424 = models/aa_model.py:443-508 = models/old_cg_model.py:303-351): ``c`` holds the per-batch
    constants (bonds, segment pointers, capacities); ``sync_free`` selects the capacity-buffer bond graph."""
    lig = data['ligand']
    ns, B = model.ns, data.num_graphs
    n_lig = lig_node.shape[0]
    # -- translation / rotation head (:368-395) -----------------------------------------------------------------
    pos = lig.pos.float()
    arange = torch.arange(n_lig, device=pos.device)
    center = torch.zeros((B, 3), device=pos.device).index_add_(0, lig.batch, pos)
    center = center / c['lig_cnt_f']
    c_vec = pos - center[lig.batch]
    c_ea = torch.cat([model.center_distance_expansion(c_vec.norm(dim=-1)), lig.node_sigma_emb], 1)
    c_ea = model.center_edge_embedding(c_ea)
    # hazard C.6: the graph id indexes lig_node.  A packed batch (hetero.collate_packed) gives each pose the node it reads
    # when its complex is sampled alone
    centre_node = getattr(data, '_center_node', None)
    idx = arange if model.fixed_center_conv else (lig.batch if centre_node is None else centre_node[lig.batch])
    c_ea = torch.cat([c_ea, lig_node[idx, :ns]], -1)
    glob = model.final_conv(lig_node, torch.stack([lig.batch, arange]), c_ea, None, out_nodes=B, edge_vec=c_vec,
                            assume_sorted=True)
    tr_pred = glob[:, :3] + (glob[:, 6:9] if not model.odd_parity else 0)
    rot_pred = glob[:, 3:6] + (glob[:, 9:] if not model.odd_parity else 0)
    data.graph_sigma_emb = model.timestep_emb_func(data.complex_t['tr'])
    tr_norm = torch.linalg.vector_norm(tr_pred, dim=1).unsqueeze(1)
    tr_pred = tr_pred / tr_norm * model.tr_final_layer(torch.cat([tr_norm, data.graph_sigma_emb], dim=1))
    rot_norm = torch.linalg.vector_norm(rot_pred, dim=1).unsqueeze(1)
    rot_pred = rot_pred / rot_norm * model.rot_final_layer(torch.cat([rot_norm, data.graph_sigma_emb], dim=1))
    if model.scale_by_sigma:
        tr_pred = tr_pred / tr_sigma.unsqueeze(1)
        rot_pred = rot_pred * model._so3_score_norm(rot_sigma).unsqueeze(1)

    if model.no_torsion or c['n_bonds'] == 0:
        return tr_pred, rot_pred, torch.empty(0, device=model.device)

    # -- torsion head (:406-423) --------------------------------------------------------------------------------
    bonds = c['bonds']
    n_bonds = c['n_bonds']
    bond_pos = ((pos[bonds[0]] + pos[bonds[1]]) / 2).contiguous()
    if sync_free:
        # upper-bound buffer (32 atoms per bond, models/cg_model.py:630); slots beyond the live count point at an extra
        # dummy bond row (index n_bonds) that is dropped after the convolution
        pos_c = pos.contiguous()
        cnt = ops.radius_count(pos_c, bond_pos, c['lig_ptr'], c['bond_batch32'], r=model.lig_max_radius, max_num_neighbors=32)
        incl = torch.cumsum(cnt, 0, dtype=torch.int32)
        bi32, ai32, t_vec, _, _ = ops.graph_fill(pos_c, bond_pos, c['lig_ptr'], c['bond_batch32'], (incl - cnt).contiguous(),
                                                 c['cap_tor'], r=model.lig_max_radius, max_num_neighbors=32, fill_row=n_bonds)
        bi, ai = bi32.long(), ai32.long()
        bi_g = bi.clamp_max(n_bonds - 1)            # gathers of per-bond quantities for the dummy slots: any valid row
        n_out = n_bonds + 1
    else:
        bi, ai, _ = ops.radius(pos, bond_pos, c['lig_ptr'], c['bond_batch'], r=model.lig_max_radius, max_num_neighbors=32)
        bi, ai = bi.long(), ai.long()
        t_vec = pos[ai] - bond_pos[bi]
        bi_g, n_out = bi, n_bonds
    t_ea = model.final_edge_embedding(model.lig_distance_expansion(t_vec.norm(dim=-1)))
    bond_vec = pos[bonds[1]] - pos[bonds[0]]
    bond_attr = lig_node[bonds[0]] + lig_node[bonds[1]]
    t_sh = torch.einsum('ea,eb,abc->ec', _sh_full(t_vec, model.sh_lmax), _sh_l2(bond_vec)[bi_g], model._tor_tp)
    t_ea = torch.cat([t_ea, lig_node[ai, :ns], bond_attr[bi_g, :ns]], -1)
    tor_pred = model.tor_bond_conv(lig_node, torch.stack([bi, ai]), t_ea, t_sh, out_nodes=n_out, reduce='mean',
                                   edge_weight=model.get_edge_weight(t_vec, model.lig_max_radius), assume_sorted=True)
    tor_pred = model.tor_final_layer(tor_pred[:n_bonds]).squeeze(1)
    edge_sigma = tor_sigma[c['bond_lig_batch']]
    if model.scale_by_sigma:
        tor_pred = tor_pred * torch.sqrt(model._torus_score_norm(edge_sigma))
    return tr_pred, rot_pred, tor_pred


class GaussianSmearing(nn.Module):
    """Radial basis expansion exp(coeff * (d - mu_k)^2), mu = linspace(start, stop, K)  (models/layers.py:20-30)."""

    def __init__(self, start=0.0, stop=5.0, num_gaussians=50):
        super().__init__()
        mu = torch.linspace(start, stop, num_gaussians)
        self.coeff = -0.5 / (mu[1] - mu[0]).item() ** 2
        self.register_buffer('offset', mu)

    def forward(self, dist):
        diff = dist.reshape(-1, 1) - self.offset.reshape(1, -1)
        return torch.exp(self.coeff * diff * diff)


class AtomEncoder(nn.Module):
    """Sum of one embedding table per categorical column, then a Linear over [embedding | remaining float columns]
    (models/layers.py:33-67)."""

    def __init__(self, emb_dim, feature_dims, sigma_embed_dim, lm_embedding_dim=0):
        super().__init__()
        cat_dims, n_scalar = feature_dims
        self.num_categorical_features = len(cat_dims)
        self.additional_features_dim = n_scalar + sigma_embed_dim + lm_embedding_dim
        self.atom_embedding_list = nn.ModuleList()
        for d in cat_dims:
            table = nn.Embedding(d, emb_dim)
            nn.init.xavier_uniform_(table.weight.data)
            self.atom_embedding_list.append(table)
        if self.additional_features_dim > 0:
            self.additional_features_embedder = nn.Linear(self.additional_features_dim + emb_dim, emb_dim)

    def forward(self, x):
        nc = self.num_categorical_features
        assert x.shape[1] == nc + self.additional_features_dim
        idx = x[:, :nc].long()
        h = self.atom_embedding_list[0](idx[:, 0])
        for i in range(1, nc):
            h = h + self.atom_embedding_list[i](idx[:, i])
        if self.additional_features_dim > 0:
            h = self.additional_features_embedder(torch.cat([h, x[:, nc:].to(h.dtype)], dim=1))
        return h


class OldAtomEncoder(nn.Module):
    """models/layers.py:70-117: categorical embeddings + Linear(scalar features incl. sigma embedding), then an optional
    Linear([emb | LM columns]) - the encoder of the confidence model.  ``lm_embedding_dim`` (1280 in the reference,
    hard-wired for 'esm') is a keyword here so that small fixtures can be loaded."""

    def __init__(self, emb_dim, feature_dims, sigma_embed_dim, lm_embedding_type=None, lm_embedding_dim=1280):
        super().__init__()
        self.atom_embedding_list = nn.ModuleList()
        self.num_categorical_features = len(feature_dims[0])
        self.num_scalar_features = feature_dims[1] + sigma_embed_dim
        self.lm_embedding_type = lm_embedding_type
        for dim in feature_dims[0]:
            emb = nn.Embedding(dim, emb_dim)
            nn.init.xavier_uniform_(emb.weight.data)
            self.atom_embedding_list.append(emb)
        if self.num_scalar_features > 0:
            self.linear = nn.Linear(self.num_scalar_features, emb_dim)
        if lm_embedding_type is not None:
            if lm_embedding_type != 'esm':
                raise ValueError('LM Embedding type was not correctly determined. LM embedding type: ', lm_embedding_type)
            self.lm_embedding_dim = lm_embedding_dim
            self.lm_embedding_layer = nn.Linear(self.lm_embedding_dim + emb_dim, emb_dim)

    def forward(self, x):
        nc, nsf = self.num_categorical_features, self.num_scalar_features
        assert x.shape[1] == nc + nsf + (self.lm_embedding_dim if self.lm_embedding_type is not None else 0)
        out = 0
        for i in range(nc):
            out = out + self.atom_embedding_list[i](x[:, i].long())
        if nsf > 0:
            out = out + self.linear(x[:, nc:nc + nsf].float())
        if self.lm_embedding_type is not None:
            out = self.lm_embedding_layer(torch.cat([out, x[:, -self.lm_embedding_dim:].float()], 1))
        return out
