"""Model factory: drop-in for ``utils/utils.py:get_model`` (the call inference.py:201-211 / evaluate.py use to build the score
and confidence models from a ``model_parameters.yml`` namespace).  Same signature, same mapping from the training flags to
constructor keywords - including the flags older checkpoints' yml files do not contain, which fall back to the reference's
defaults - but the classes are the H100-native ones:

    old=False : diffdock_b200.cg_model.CGModel       / diffdock_b200.aa_model.AAModel        (``all_atoms``)
    old=True  : diffdock_b200.old_cg_model.CGOldModel / diffdock_b200.old_aa_model.AAOldModel

The mapping is written as two tables (flag, keyword, default, transform) rather than as the reference's call expression;
tests/test_get_model_cpu.py holds it to the keywords the UNMODIFIED reference function passes to its model classes
(tests/golden/ref_get_model.pt).  ``torch_geometric``'s DataParallel wrapper of the reference (utils/utils.py:279-280) is not
reproduced: one process drives one GPU here (diffdock_b200.distributed shards over GPUs), so ``no_parallel=False`` raises."""
from __future__ import annotations

from .diffusion_utils import get_timestep_embedding

_NOT = lambda v: not v
_LEN1 = lambda v: len(v) + 1

# (constructor keyword, args attribute, default when the attribute is absent [REQUIRED = must be present], transform)
REQUIRED = object()
_COMMON = [
    ('no_torsion', 'no_torsion', REQUIRED, None),
    ('num_conv_layers', 'num_conv_layers', REQUIRED, None),
    ('lig_max_radius', 'max_radius', REQUIRED, None),
    ('scale_by_sigma', 'scale_by_sigma', REQUIRED, None),
    ('sigma_embed_dim', 'sigma_embed_dim', REQUIRED, None),
    ('norm_by_sigma', 'norm_by_sigma', False, None),
    ('ns', 'ns', REQUIRED, None),
    ('nv', 'nv', REQUIRED, None),
    ('distance_embed_dim', 'distance_embed_dim', REQUIRED, None),
    ('cross_distance_embed_dim', 'cross_distance_embed_dim', REQUIRED, None),
    ('batch_norm', 'no_batch_norm', REQUIRED, _NOT),
    ('dropout', 'dropout', REQUIRED, None),
    ('use_second_order_repr', 'use_second_order_repr', REQUIRED, None),
    ('cross_max_distance', 'cross_max_distance', REQUIRED, None),
    ('dynamic_max_cross', 'dynamic_max_cross', REQUIRED, None),
    ('smooth_edges', 'smooth_edges', False, None),
    ('odd_parity', 'odd_parity', False, None),
    ('affinity_prediction', 'affinity_prediction', False, None),
    ('parallel', 'parallel', 1, None),
    ('parallel_aggregators', 'parallel_aggregators', '', None),
    ('fixed_center_conv', 'not_fixed_center_conv', False, _NOT),
    ('no_aminoacid_identities', 'no_aminoacid_identities', False, None),
    ('include_miscellaneous_atoms', 'include_miscellaneous_atoms', False, None),
]
_OLD_ONLY = [('use_old_atom_encoder', 'use_old_atom_encoder', True, None)]
_NEW_ONLY = [
    ('sh_lmax', 'sh_lmax', 2, None),
    ('differentiate_convolutions', 'no_differentiate_convolutions', True, _NOT),
    ('tp_weights_layers', 'tp_weights_layers', 2, None),
    ('num_prot_emb_layers', 'num_prot_emb_layers', 0, None),
    ('reduce_pseudoscalars', 'reduce_pseudoscalars', False, None),
    ('embed_also_ligand', 'embed_also_ligand', False, None),
    ('depthwise_convolution', 'depthwise_convolution', False, None),
]
_ESM_PATH_FLAGS = ('moad_esm_embeddings_path', 'pdbbind_esm_embeddings_path', 'pdbsidechain_esm_embeddings_path',
                   'esm_embeddings_path')


def _has(args, name):
    return name in args if hasattr(args, '__contains__') else hasattr(args, name)


def _from_table(args, table):
    kw = {}
    for key, attr, default, fn in table:
        if _has(args, attr):
            v = getattr(args, attr)
            kw[key] = fn(v) if fn else v
        elif default is REQUIRED:
            raise AttributeError(f"model arguments lack '{attr}'")
        else:
            kw[key] = default
    return kw


def _n_outputs(args, flag):
    v = getattr(args, flag) if _has(args, flag) else None
    return len(v) + 1 if isinstance(v, list) else 1


def model_kwargs(args, confidence_mode=False, old=False):
    """(model class name, constructor keywords without ``t_to_sigma`` / ``device`` / ``timestep_emb_func``) that
    utils/utils.py:172-276 derives from ``args``."""
    all_atoms = _has(args, 'all_atoms') and bool(args.all_atoms)
    kw = _from_table(args, _COMMON)
    kw['confidence_mode'] = confidence_mode
    kw['num_confidence_outputs'] = _n_outputs(args, 'rmsd_classification_cutoff')
    if old:
        kw.update(_from_table(args, _OLD_ONLY))
        kw['lm_embedding_type'] = 'esm' if args.esm_embeddings_path is not None else None       # :185-186
        return ('AAOldModel' if all_atoms else 'CGOldModel'), kw
    kw.update(_from_table(args, _NEW_ONLY))
    lm = 'precomputed' if any(_has(args, f) and getattr(args, f) is not None for f in _ESM_PATH_FLAGS) else None
    if _has(args, 'esm_embeddings_model') and args.esm_embeddings_model is not None:
        lm = args.esm_embeddings_model
    kw['lm_embedding_type'] = lm
    kw['atom_num_confidence_outputs'] = _n_outputs(args, 'atom_rmsd_classification_cutoff')
    kw['atom_confidence'] = args.atom_confidence_loss_weight > 0.0 if _has(args, 'atom_confidence_loss_weight') else False
    kw['sidechain_pred'] = (_has(args, 'sidechain_loss_weight') and args.sidechain_loss_weight > 0) or \
                           (_has(args, 'backbone_loss_weight') and args.backbone_loss_weight > 0)
    return ('AAModel' if all_atoms else 'CGModel'), kw


def _model_class(name):
    if name == 'CGModel':
        from .cg_model import CGModel as cls
    elif name == 'AAModel':
        from .aa_model import AAModel as cls
    elif name == 'CGOldModel':
        from .old_cg_model import CGOldModel as cls
    else:
        from .old_aa_model import AAOldModel as cls
    return cls


def get_model(args, device, t_to_sigma, no_parallel=False, confidence_mode=False, old=False):
    """utils/utils.py:172-281.  Returns the model on ``device`` (call ``load_state_dict`` / ``eval`` as inference.py does)."""
    import torch
    device = torch.device(device)
    if device.type == 'cuda' and not no_parallel and (not _has(args, 'dataset') or args.dataset != 'torsional'):
        raise NotImplementedError("torch_geometric DataParallel is not reproduced: pass no_parallel=True (as inference.py does) "
                                  "and shard over GPUs with diffdock_b200.distributed")
    emb = get_timestep_embedding(embedding_type=args.embedding_type if _has(args, 'embedding_type') else 'sinusoidal',
                                 embedding_dim=args.sigma_embed_dim,
                                 embedding_scale=args.embedding_scale if _has(args, 'embedding_type') else 10000)
    name, kw = model_kwargs(args, confidence_mode=confidence_mode, old=old)
    model = _model_class(name)(t_to_sigma=t_to_sigma, device=device, timestep_emb_func=emb, **kw)
    return model.to(device)
