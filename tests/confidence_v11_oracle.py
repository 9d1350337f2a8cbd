"""Oracle restatement of the v1.1 models in CONFIDENCE MODE - ``CGModel`` / ``AAModel`` built with ``confidence_mode=True``,
what the reference's confidence trainer builds (confidence/confidence_train.py:284 -> utils/utils.py:221-224).  TEST
INFRASTRUCTURE (CPU, plain PyTorch).

The embeddings, graphs and interaction stack are those of the score-mode oracle (oracle/cg_model.py, oracle/aa_model.py);
confidence mode changes two things (models/cg_model.py:181-208,312-366 = models/aa_model.py:177-225,380-455): the diffusion
times are used as the sigmas (no ``t_to_sigma``, so ``dynamic_max_cross`` gives 3 t + 20), and the score heads are replaced by
``confidence_predictor`` (and ``atom_confidence_predictor``) over the mean of the selected ligand scalars.  Same constructor
keywords and state_dict keys as the reference classes in confidence mode."""
import torch
from torch import nn

from oracle.aa_model import AAModel
from oracle.cg_model import CGModel

_SCORE_HEADS = ('center_distance_expansion', 'center_edge_embedding', 'final_conv', 'tr_final_layer', 'rot_final_layer',
                'final_edge_embedding', 'final_tp_tor', 'tor_bond_conv', 'tor_final_layer')


def _head(n_in, ns, n_out, dropout, no_batchnorm):
    bn = (lambda: nn.Identity()) if no_batchnorm else (lambda: nn.BatchNorm1d(ns))
    return nn.Sequential(nn.Linear(n_in, ns), bn(), nn.ReLU(), nn.Dropout(dropout), nn.Linear(ns, ns), bn(), nn.ReLU(),
                         nn.Dropout(dropout), nn.Linear(ns, n_out))


class _Confidence:
    def _to_confidence(self, ns, nv, num_conv_layers, num_prot_emb_layers, reduce_pseudoscalars, affinity_prediction,
                       num_confidence_outputs, atom_confidence, atom_num_confidence_outputs, confidence_dropout,
                       confidence_no_batchnorm):
        for name in _SCORE_HEADS:
            if hasattr(self, name):
                delattr(self, name)
        self.t_to_sigma = lambda tr, rot, tor: (tr, rot, tor)          # the times are the sigmas (:312-315)
        self.confidence_mode = True
        self.tail = (nv if reduce_pseudoscalars else ns) if num_conv_layers + num_prot_emb_layers >= 3 else 0
        n_in = ns + self.tail
        self.atom_confidence, self.atom_num_confidence_outputs = atom_confidence, atom_num_confidence_outputs
        if atom_confidence:
            self.atom_confidence_predictor = _head(n_in, ns, atom_num_confidence_outputs + ns, confidence_dropout,
                                                   confidence_no_batchnorm)
            n_in = ns
        self.confidence_predictor = _head(n_in, ns, num_confidence_outputs + (1 if affinity_prediction else 0),
                                          confidence_dropout, confidence_no_batchnorm)

    def _dtype(self):
        return self.confidence_predictor[0].weight.dtype

    def _heads(self, data, lig_node, *sigmas):                         # :354-366
        ns = self.ns
        scal = torch.cat([lig_node[:, :ns], lig_node[:, -self.tail:]], 1) if self.tail else lig_node[:, :ns]
        if self.atom_confidence:
            scal = self.atom_confidence_predictor(scal)
            atom_conf = scal[:, :self.atom_num_confidence_outputs]
            scal = scal[:, self.atom_num_confidence_outputs:]
        else:
            atom_conf = torch.zeros((len(lig_node),), dtype=lig_node.dtype)
        batch, B = data['ligand'].batch, data.num_graphs
        pooled = torch.zeros((B, scal.shape[1]), dtype=scal.dtype).index_add_(0, batch, scal)
        pooled = pooled / torch.bincount(batch, minlength=B).clamp(min=1).unsqueeze(1).to(scal.dtype)   # scatter_mean
        return self.confidence_predictor(pooled).squeeze(dim=-1), atom_conf


def _confidence_kw(kw):
    keys = dict(affinity_prediction=False, num_confidence_outputs=1, atom_confidence=False, atom_num_confidence_outputs=1,
                confidence_dropout=0, confidence_no_batchnorm=False)
    out = {k: kw.pop(k, v) for k, v in keys.items()}
    kw.pop('confidence_mode', None)
    return out


class CGConfidenceModel(_Confidence, CGModel):
    def __init__(self, t_to_sigma, device, timestep_emb_func, **kw):
        conf = _confidence_kw(kw)
        CGModel.__init__(self, t_to_sigma, device, timestep_emb_func, **kw)
        self._to_confidence(kw.get('ns', 16), kw.get('nv', 4), kw.get('num_conv_layers', 2), kw.get('num_prot_emb_layers', 0),
                            kw.get('reduce_pseudoscalars', False), **conf)


class AAConfidenceModel(_Confidence, AAModel):
    def __init__(self, t_to_sigma, device, timestep_emb_func, **kw):
        conf = _confidence_kw(kw)
        AAModel.__init__(self, t_to_sigma, device, timestep_emb_func, **kw)
        self._to_confidence(kw.get('ns', 16), kw.get('nv', 4), kw.get('num_conv_layers', 2), kw.get('num_prot_emb_layers', 0),
                            kw.get('reduce_pseudoscalars', False), **conf)
