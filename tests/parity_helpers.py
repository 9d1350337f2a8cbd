"""Shared helpers of the parity tests: seeded random layers/graphs evaluated by the oracle (CPU) and the product (CUDA)."""
import functools

import torch


def rand_bn_(bn, gen):
    """Non-trivial eval-mode statistics (SURVEY.md section 8(d))."""
    with torch.no_grad():
        bn.running_mean.copy_(0.1 * torch.randn(bn.running_mean.shape, generator=gen))
        bn.running_var.copy_(0.5 + torch.rand(bn.running_var.shape, generator=gen))
        bn.weight.copy_(1.0 + 0.2 * torch.randn(bn.weight.shape, generator=gen))
        bn.bias.copy_(0.1 * torch.randn(bn.bias.shape, generator=gen))


def make_layer_pair(in_irreps, sh_irreps, out_irreps, n_edge_features, seed=0, **kw):
    """(oracle layer on CPU, product layer with identical parameters)."""
    from oracle.tensor_layers import TensorProductConvLayer as OLayer
    from diffdock_b200.tensor_layers import TensorProductConvLayer as PLayer
    torch.manual_seed(seed)
    o = OLayer(in_irreps, sh_irreps, out_irreps, n_edge_features, **kw).eval()
    gen = torch.Generator().manual_seed(seed + 1)
    if o.batch_norm is not None:
        rand_bn_(o.batch_norm, gen)
    p = PLayer(in_irreps, sh_irreps, out_irreps, n_edge_features, **kw).eval()
    sd = {k: v for k, v in o.state_dict().items() if not k.startswith('tp.')}
    missing, unexpected = p.load_state_dict(sd, strict=False)
    assert not missing and not unexpected, (missing, unexpected)
    return o, p


def rel_err(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


# Cases of the fused convolution shared by the plan emulation (CPU) and the kernel tests (GPU).
# Consumer kinds: (ns, nv) = (48, 10) has the (48, 1) / (10, 3) kinds, (16, 4) the (16, 1) / (4, 3) kinds; every stage of the
# irreps sequence, with spherical harmonics up to l = 2, up to l = 1, and the closed-form l <= 1 product ('faster').
KIND_GRID = [((ns, nv), stage, lmax, faster) for ns, nv in ((48, 10), (16, 4)) for stage in range(4)
             for lmax, faster in ((2, False), (1, False), (1, True))]
# (ne, ns, H) of the radial MLP: production shapes, then the element-wise A0 path (ne, ns not multiples of 8; neither
# K1 = 30 nor H a multiple of 16), K1 > H, K1 < H and H < 64
SHAPE_GRID = [(48, 48, 144), (16, 16, 48), (144, 0, 144), (48, 0, 48),
              (20, 5, 100), (48, 48, 48), (16, 16, 144), (48, 0, 40)]


def fused_table(ns, nv, stage, lmax, faster):
    from diffdock_b200.tensor_layers import get_irrep_seq
    from diffdock_b200.tp_table import build_table
    seq = get_irrep_seq(ns, nv, False, False)
    shs = '1x0e + 1x1o' if lmax == 1 else '1x0e + 1x1o + 1x2e'
    return build_table(seq[min(stage, 3)], shs, seq[min(stage + 1, 3)], 'faster' if faster else 'fctp')


def fused_weights(table, H, K1, gen):
    """Radial MLP parameters (W1 [H, K1], b1, W2 [weight_numel, H] in reference row order, b2) at a trained model's scale."""
    r = lambda *s: torch.randn(*s, generator=gen)
    return r(H, K1) / K1 ** 0.5, 0.1 * r(H), r(table.weight_numel, H) / H ** 0.5, 0.1 * r(table.weight_numel)


def irreps_str(irreps):
    """[(mul, l, parity)] of a TpTable -> an irreps string the oracle parses."""
    return ' + '.join(f'{m}x{l}{"e" if p == 1 else "o"}' for m, l, p in irreps)


def _reference_tp(table, dev):
    """The oracle's tensor product of a TpTable (FullyConnectedTensorProduct or FasterTensorProduct) on ``dev``."""
    from oracle import e3nn_lite as o3
    from oracle.tensor_layers import FasterTensorProduct
    ins, shs, outs = irreps_str(table.in_irreps), irreps_str(table.sh_irreps), irreps_str(table.out_irreps)
    tp = FasterTensorProduct(ins, shs, outs) if table.kind == 'faster' else o3.FullyConnectedTensorProduct(ins, shs, outs)
    assert tp.weight_numel == table.weight_numel
    return tp.to(dev)


def tp_scatter_reference(table, x, src, tgt, geo, w_ref, n_out, ew=None, device=None, chunk=2048, tp=None, out=None):
    """float64 restatement of the streaming convolution (include/diffdock_b200.h:ddb200_tpconv_accumulate):
        sum[tgt[e]] += TP(x[src[e]], Y_e, w_ref[e]) * ew[e],   cnt[tgt[e]] += 1
    Y_e is the oracle's spherical harmonics of geo[e] (normalize=True, component normalisation) when the table evaluates
    them from edge vectors (table.sh_lmax >= 0), otherwise geo[e] itself (given SH).  ``w_ref`` [E, weight_numel] is in the
    reference's weight order.  Built only from plain torch and the oracle, evaluated chunk by chunk over the edges.
    ``out``: a float64 [n_out, d_out] accumulator to add into.  Returns (sum, cnt) in float64 on ``device`` (default: x's)."""
    from oracle import e3nn_lite as o3
    dev = torch.device(device) if device is not None else x.device
    tp = tp if tp is not None else _reference_tp(table, dev)
    assert w_ref.shape[1] == table.weight_numel
    x = x.to(dev, torch.float64)
    tgt, src = tgt.to(dev).long(), src.to(dev).long()
    E = tgt.shape[0]
    shs = o3.Irreps(irreps_str(table.sh_irreps))
    if out is None:
        out = torch.zeros(n_out, table.d_out, dtype=torch.float64, device=dev)
    for c0 in range(0, E, chunk):
        c1 = min(E, c0 + chunk)
        g = geo[c0:c1].to(dev, torch.float64)
        sh = o3.spherical_harmonics(shs, g, normalize=True, normalization='component') if table.sh_lmax >= 0 else g
        m = tp(x[src[c0:c1]], sh, w_ref[c0:c1].to(dev, torch.float64))
        if ew is not None:
            m = m * ew.reshape(-1)[c0:c1].to(dev, torch.float64)[:, None]
        out.index_add_(0, tgt[c0:c1], m)
    return out, torch.bincount(tgt, minlength=n_out).double()


def kernel_weights(table, w_ref, stride=None, fill=float('nan')):
    """Per-edge weight rows [E, stride] in the kernel's layout (table.w_perm) from reference-order rows [E, weight_numel].
    Padding columns (w_perm == -1) and the columns past weight_numel_padded hold ``fill``: with NaN, a read of anything but
    a weight shows up as NaN in the output."""
    stride = stride or table.weight_numel_padded
    assert stride >= table.weight_numel_padded
    out = torch.full((w_ref.shape[0], stride), fill, dtype=w_ref.dtype, device=w_ref.device)
    perm = torch.as_tensor(table.w_perm, device=w_ref.device)
    cols = torch.nonzero(perm >= 0).reshape(-1)
    out[:, cols] = w_ref[:, perm[cols]]
    return out


def fused_conv_reference(table, w1, b1, w2, b2, ea, node, ns, tgt, src, x, vec, n_out, ew=None, edge_perm=None,
                         vec_sign=1.0, ea_add=None, ea_add_idx=None, device=None, chunk=2048):
    """float64 restatement of the fused convolution of one edge group (include/diffdock_b200.h:ddb200_fused_conv):
        r = edge_perm[e] (default e),  a = [ea[r, :ne] (+ ea_add[ea_add_idx[e]]) | node[tgt[e], :ns] | node[src[e], :ns]]
        sum[tgt[e]] += TP(x[src[e]], Y(vec_sign * vec[r]), (relu(a W1^T + b1) W2^T + b2) * ew[r]),   cnt[tgt[e]] += 1
    w2 / b2 are in the reference weight-row order.  The radial MLP is evaluated chunk by chunk over the edges, so that the
    per-edge weight tensor never exists whole, and each chunk goes through tp_scatter_reference.  Returns
    (sum [n_out, d_out], cnt [n_out]) in float64 on ``device`` (default: ea's)."""
    dev = torch.device(device) if device is not None else ea.device
    tp = _reference_tp(table, dev)
    assert w2.shape[0] == table.weight_numel
    d = lambda t: t.to(dev, torch.float64)
    w1, b1, w2, b2, x = d(w1), d(b1), d(w2), d(b2), d(x)
    ne = w1.shape[1] - 2 * ns
    tgt, src = tgt.to(dev).long(), src.to(dev).long()
    E = tgt.shape[0]
    ea, vec = d(ea[:, :ne]), d(vec)
    node = d(node[:, :ns]) if ns else None
    ew = d(ew.reshape(-1)) if ew is not None else None
    ea_add = d(ea_add) if ea_add is not None else None
    out = torch.zeros(n_out, table.d_out, dtype=torch.float64, device=dev)
    for c0 in range(0, E, chunk):
        c1 = min(E, c0 + chunk)
        r = edge_perm[c0:c1].to(dev).long() if edge_perm is not None else torch.arange(c0, c1, device=dev)
        t, s = tgt[c0:c1], src[c0:c1]
        a = ea[r]
        if ea_add is not None:
            a = a + ea_add[ea_add_idx[c0:c1].to(dev).long()]
        if ns:
            a = torch.cat([a, node[t], node[s]], 1)
        w = torch.relu(a @ w1.T + b1) @ w2.T + b2
        tp_scatter_reference(table, x, s, t, vec_sign * vec[r], w, n_out, ew=ew[r] if ew is not None else None,
                             device=dev, chunk=c1 - c0, tp=tp, out=out)
    return out, torch.bincount(tgt, minlength=n_out).double()


def tp_table_grid():
    """{name: TpTable} of the streaming kernel's table features (tile kinds, z kinds, column tiles, remainder rows, TMA
    chunking, padding, given SH, D_in > 256), built with tp_table.build_table:
      final / final_odd    the score model's final_conv (seq[3] -> 2x1o + 2x1e, lmax 2; -> 1x1o + 1x1e, lmax 1)
      tor / tor_odd        tor_bond_conv with given SH (FullTensorProduct(sh, 2e): 45 / 20 columns)
      ladder_*             every stage of the irreps ladder at four (ns, nv), fctp lmax 2 / lmax 1 / faster
      second_*             second-order representations (generic tile kind, 2l+1 = 5, the default z kind)
      wide                 D_in = 512, a 160x0e output split over two column tiles, three lanes-per-row values
      small_stages         seq[3] -> seq[3] with 100-float TMA chunks: many chunks, pieces split with remainder rows"""
    return _tp_table_grid()


@functools.lru_cache(maxsize=None)
def _tp_table_grid():
    from diffdock_b200.irreps import irreps_str as ir_str
    from diffdock_b200.tensor_layers import get_irrep_seq
    from diffdock_b200.tp_table import build_table, full_tensor_product
    sh1, sh2 = '1x0e+1x1o', '1x0e+1x1o+1x2e'
    seq = get_irrep_seq(48, 10, False, False)
    g = {'final': build_table(seq[3], sh2, '2x1o + 2x1e'),
         'final_odd': build_table(seq[3], sh1, '1x1o + 1x1e'),
         'tor': build_table(seq[3], ir_str(full_tensor_product(sh2, '1x2e')[1]), '48x0o + 48x0e', sh_from_vector=False),
         'tor_odd': build_table(seq[3], ir_str(full_tensor_product(sh1, '1x2e')[1]), '48x0o', sh_from_vector=False)}
    for ns, nv in ((48, 10), (16, 4), (6, 3), (24, 6)):
        s = get_irrep_seq(ns, nv, False, False)
        for stage in range(4):
            for name, shs, kind in (('l2', sh2, 'fctp'), ('l1', sh1, 'fctp'), ('faster', sh1, 'faster')):
                g[f'ladder_{ns}_{nv}_s{stage}_{name}'] = build_table(s[stage], shs, s[min(stage + 1, 3)], kind)
    for ns, nv, red in ((48, 10, False), (5, 3, True)):
        s = get_irrep_seq(ns, nv, True, red)
        g[f'second_{ns}_{nv}'] = build_table(s[3], sh2, s[3])
    g['wide'] = build_table('96x0e + 20x1o + 20x2e + 20x1e + 20x2o + 96x0o', sh2, '160x0e + 8x1o')
    g['small_stages'] = build_table(seq[3], sh2, seq[3], stage_floats=100)
    return g


def table_sections(table):
    """(paths [n, 8], tiles [n, 16], chunks [n, 4], ment [n, 3]) of a compiled table's int blob."""
    ib = table.iblob
    sec = lambda i, n, w: ib[ib[15 + i]:ib[15 + i] + w * n].reshape(-1, w)
    return sec(0, ib[1], 8), sec(1, ib[2], 16), sec(2, ib[3], 4), sec(3, ib[4], 3)


def block_errors(got, ref, out_irreps):
    """Per output irrep block: max |got - ref| over the block / max |ref| over the block, the denominator floored at 1e-2 of
    the global max |ref| (a near-zero block would otherwise turn rounding noise into a large ratio).  ``out_irreps`` is a
    TpTable's [(mul, l, parity)].  Returns {'<mul>x<l><p>@<offset>': error}."""
    got, ref = got.double(), ref.double().to(got.device)
    floor = 1e-2 * float(ref.abs().max().clamp_min(1e-30))
    errs, off = {}, 0
    for m, l, p in out_irreps:
        n = m * (2 * l + 1)
        g, r = got[:, off:off + n], ref[:, off:off + n]
        errs[f'{m}x{l}{"e" if p == 1 else "o"}@{off}'] = float((g - r).abs().max()) / max(float(r.abs().max()), floor)
        off += n
    return errs


def max_block_err(got, ref, out_irreps):
    return max(block_errors(got, ref, out_irreps).values())


def layer_parity_case(seed=0, n_nodes=64, n_edges=700, ns=48, nv=10, lmax=2, stage=3, groups=1, faster=False,
                      device='cuda:0', reduce='mean', use_vec=True, edge_weight_tensor=False, out_nodes=None,
                      residual=True):
    from oracle import e3nn_lite as o3
    from oracle.tensor_layers import get_irrep_seq
    seq = get_irrep_seq(ns, nv, False, False)
    sh_irreps = str(o3.Irreps.spherical_harmonics(lmax))
    o, p = make_layer_pair(seq[min(stage, 3)], sh_irreps, seq[min(stage + 1, 3)], 3 * ns, seed=seed,
                           hidden_features=3 * ns, edge_groups=groups, faster=faster, residual=residual)
    g = torch.Generator().manual_seed(seed + 2)
    x = torch.randn(n_nodes, o3.Irreps(seq[min(stage, 3)]).dim, generator=g)
    n_tgt = out_nodes or n_nodes
    ei = torch.stack([torch.randint(0, n_tgt, (n_edges,), generator=g), torch.randint(0, n_nodes, (n_edges,), generator=g)])
    vec = torch.randn(n_edges, 3, generator=g)
    ea = torch.randn(n_edges, 3 * ns, generator=g)
    sh = o3.spherical_harmonics(o3.Irreps(sh_irreps), vec, normalize=True, normalization='component')
    ew = torch.rand(n_edges, 1, generator=g) if edge_weight_tensor else 1.0
    if groups > 1:
        cuts = sorted(torch.randint(0, n_edges, (groups - 1,), generator=g).tolist())
        b = [0] + cuts + [n_edges]
        ea_o = [ea[b[i]:b[i + 1]] for i in range(groups)]
    else:
        ea_o = ea
    with torch.no_grad():
        ref = o(x, ei, ea_o, sh, out_nodes=out_nodes, reduce=reduce, edge_weight=ew)
    p = p.to(device)
    dev = lambda t: t.to(device) if torch.is_tensor(t) else t
    ea_p = [dev(a) for a in ea_o] if groups > 1 else dev(ea)
    got = p(dev(x), dev(ei), ea_p, dev(sh), out_nodes=out_nodes, reduce=reduce, edge_weight=dev(ew),
            edge_vec=dev(vec) if use_vec else None)
    torch.cuda.synchronize()
    return rel_err(got, ref)


def make_model_pair(args, seed=0, lm=True, product=True):
    """(oracle CGModel on CPU, product CGModel) sharing one random state_dict (BatchNorm statistics randomised)."""
    from functools import partial
    from oracle.cg_model import CGModel as OModel
    from oracle.layers import get_timestep_embedding as o_emb
    from oracle.diffusion import t_to_sigma as o_t2s
    from diffdock_b200.cg_model import CGModel as PModel
    from diffdock_b200.diffusion_utils import get_timestep_embedding as p_emb, t_to_sigma as p_t2s
    kw = dict(sigma_embed_dim=args.sigma_embed_dim, sh_lmax=args.sh_lmax, ns=args.ns, nv=args.nv,
              num_conv_layers=args.num_conv_layers, lig_max_radius=args.max_radius, rec_max_radius=args.rec_max_radius,
              cross_max_distance=args.cross_max_distance, center_max_distance=args.center_max_distance,
              distance_embed_dim=args.distance_embed_dim, cross_distance_embed_dim=args.cross_distance_embed_dim,
              dynamic_max_cross=args.dynamic_max_cross, lm_embedding_type='precomputed' if lm else None,
              embed_also_ligand=True, num_prot_emb_layers=args.num_prot_emb_layers,
              use_second_order_repr=args.use_second_order_repr, no_torsion=args.no_torsion,
              smooth_edges=args.smooth_edges, fixed_center_conv=args.fixed_center_conv,
              reduce_pseudoscalars=args.reduce_pseudoscalars,
              differentiate_convolutions=args.differentiate_convolutions)
    torch.manual_seed(seed)
    o = OModel(partial(o_t2s, args=args), 'cpu', o_emb('sinusoidal', args.sigma_embed_dim, args.embedding_scale), **kw).eval()
    gen = torch.Generator().manual_seed(seed + 1)
    for m in o.modules():
        if m.__class__.__name__ == 'BatchNorm':
            rand_bn_(m, gen)
    if not product:
        return o, None
    p = PModel(partial(p_t2s, args=args), torch.device('cuda:0'),
               p_emb('sinusoidal', args.sigma_embed_dim, args.embedding_scale), **kw).eval()
    p.load_state_dict(o.state_dict(), strict=True)     # includes e3nn-style tp.* buffers, which must be accepted
    return o, p.to('cuda:0')


def model_parity_case(seed=0, lmax=2, ns=16, nv=4, n_layers=3, emb=16, n_res=60, n_atoms=12, n_poses=3, t=0.5,
                      far_poses=(), run_product=True, **over):
    from diffdock_b200.synthetic import default_model_args, make_pose_list
    from diffdock_b200.hetero import collate
    from oracle.diffusion import set_time
    args = default_model_args(ns=ns, nv=nv, sh_lmax=lmax, num_conv_layers=n_layers, distance_embed_dim=emb,
                              cross_distance_embed_dim=emb, sigma_embed_dim=emb, **over)
    o, p = make_model_pair(args, seed, product=run_product)
    poses = make_pose_list(n_poses, n_res=n_res, n_atoms=n_atoms, seed=seed + 3, tr_sigma_max=args.tr_sigma_max * t)
    for i in far_poses:       # ligand moved out of every cross cut-off: that complex has no ligand-receptor edges
        # (80 A: beyond receptor radius + cut-off for the sizes used, yet small enough that the fp32 centroid sum - whose
        # order differs between CPU and GPU atomics - keeps the 1e-4 tolerance; at 500 A it is borderline)
        poses[i]['ligand'].pos = poses[i]['ligand'].pos + 80.0
    g_cpu = collate(poses)
    set_time(g_cpu, t, t, t, n_poses, 'cpu')
    if not run_product:
        with torch.no_grad():
            return o(g_cpu)
    g_gpu = collate(poses).to('cuda:0')
    set_time(g_gpu, t, t, t, n_poses, 'cuda:0')
    with torch.no_grad():
        ref = o(g_cpu)
    got = p(g_gpu)
    torch.cuda.synchronize()
    errs = {'tr': rel_err(got[0], ref[0]), 'rot': rel_err(got[1], ref[1]), 'tor_numel': int(ref[2].numel())}
    assert got[2].numel() == ref[2].numel()
    if ref[2].numel():
        errs['tor'] = rel_err(got[2], ref[2])
    errs = {k: v for k, v in errs.items()}
    if errs['tor_numel'] > 0:
        errs.pop('tor_numel')
    return errs


# ---------------------------------------------------------------------------------------------- golden fixtures
import os as _os

GOLDEN = _os.path.join(_os.path.dirname(_os.path.abspath(__file__)), 'golden')


def load_golden(name):
    return torch.load(_os.path.join(GOLDEN, name), weights_only=False)


def golden_model(case, which, all_atoms=False):
    """Model ('oracle' on CPU | 'product' on cuda:0) + pose list rebuilt from a ref_cg_model.pt case (``all_atoms``: a
    ref_aa_model.pt case, models/aa_model.py)."""
    from argparse import Namespace
    from functools import partial
    from diffdock_b200.hetero import graph_from_dict
    a = Namespace(**case['args'])
    if which == 'oracle':
        if all_atoms:
            from oracle.aa_model import AAModel as CGModel
        else:
            from oracle.cg_model import CGModel
        from oracle.layers import get_timestep_embedding
        from oracle.diffusion import t_to_sigma
        dev = 'cpu'
    else:
        if all_atoms:
            from diffdock_b200.aa_model import AAModel as CGModel
        else:
            from diffdock_b200.cg_model import CGModel
        from diffdock_b200.diffusion_utils import get_timestep_embedding, t_to_sigma
        dev = torch.device('cuda:0')
    m = CGModel(partial(t_to_sigma, args=a), dev, get_timestep_embedding('sinusoidal', 8, a.embedding_scale),
                **case['kw']).eval()
    if case['lm_dim']:   # the fixture shrinks the 1280-wide LM embedding to 16 columns (see make_golden.py)
        m.rec_node_embedding.additional_features_dim = case['lm_dim']
        m.rec_node_embedding.additional_features_embedder = torch.nn.Linear(case['lm_dim'] + 6, 6)
    m.load_state_dict(case['state'], strict=True)
    poses = [graph_from_dict(d) for d in case['poses']]
    return m.to(dev), poses, a


def golden_confidence_model(case, which, all_atoms=False):
    """Confidence model ('oracle' on CPU | 'product' on cuda:0) + pose list rebuilt from a ref_confidence.pt case
    (``all_atoms``: a ref_confidence_aa.pt case, models/old_aa_model.py)."""
    from functools import partial
    from diffdock_b200.hetero import graph_from_dict
    from diffdock_b200.synthetic import default_model_args
    a = default_model_args()
    if which == 'oracle':
        if all_atoms:
            from oracle.old_aa_model import AAOldModel as CGOldModel
        else:
            from oracle.old_cg_model import CGOldModel
        from oracle.layers import get_timestep_embedding
        from oracle.diffusion import t_to_sigma
        dev = 'cpu'
    else:
        if all_atoms:
            from diffdock_b200.old_aa_model import AAOldModel as CGOldModel
        else:
            from diffdock_b200.old_cg_model import CGOldModel
        from diffdock_b200.diffusion_utils import get_timestep_embedding, t_to_sigma
        dev = torch.device('cuda:0')
    kw = dict(case['kw'])
    if case['lm_dim']:
        kw['lm_embedding_dim'] = case['lm_dim']     # the fixture shrinks the 1280-wide LM embedding to 16 columns
    m = CGOldModel(partial(t_to_sigma, args=a), dev, get_timestep_embedding('sinusoidal', 8, a.embedding_scale), **kw).eval()
    m.load_state_dict(case['state'], strict=True)
    return m.to(dev), [graph_from_dict(d) for d in case['poses']]


def canonical_contact_edges(edge_index, coords):
    """Contact-graph edge list [2, E] (rows [neighbour, centre], centre by centre) with TIES made canonical: where a centre's
    neighbours are listed by distance (more hits than max_neighbors: np.argsort order, datasets/process_mols.py:184), runs of
    exactly equal fp32 distance are re-ordered by index.  np.argsort's default sort is not stable and its tie order depends on
    the numpy build (AVX-512 quicksort vs introsort), so that is the strongest order a restatement can reproduce."""
    import numpy as np
    from oracle.inputs import cdist_sq_f32
    ei = np.asarray(edge_index)
    sq = cdist_sq_f32(np.asarray(coords, dtype=np.float32))
    out = ei.copy()
    start = 0
    E = ei.shape[1]
    while start < E:
        end = start
        while end < E and ei[1, end] == ei[1, start]:
            end += 1
        nb = ei[0, start:end]
        if not np.all(np.diff(nb) > 0):            # listed by distance
            i = ei[1, start]
            order = sorted(range(end - start), key=lambda q: (sq[i, nb[q]], nb[q]))
            out[0, start:end] = nb[order]
        start = end
    return out


CONTACT_CAP = 1024        # hits contact_kernel (csrc/inputs.cu) keeps per centre in shared memory


class ContactRule:
    """The contact graph's documented rule (diffdock_b200.inputs.contact_graph), vectorised so that it runs at the
    3000-residue limit: the distances of oracle.inputs.cdist_f32 (torch.cdist's fp32 arithmetic, direct form up to 25
    points), one stable argsort per row - every exact distance tie broken by index - and the centre excluded by index, not
    by distance (a duplicate of the centre, d = 0 with j != i, is an ordinary neighbour).  Per centre, with
    hits = #{j != i : d_ij < cutoff}:
        knn_only     the min(K, n - 1) nearest by (distance, index)
        hits == 0    the nearest other point (none when n == 1)
        hits <= K    the hits in index order
        hits >  K    the K nearest by (distance, index)
    K = max_neighbors or 1000.  Distances and order depend on the points only, so one instance serves every cut-off and K."""

    def __init__(self, coords):
        from oracle.inputs import cdist_f32
        self.d = cdist_f32(coords)
        self.n = self.d.shape[0]
        self._order = None

    @property
    def order(self):
        """[n, n - 1]: every centre's other points by (distance, index)."""
        if self._order is None:
            import numpy as np
            o = np.argsort(self.d, axis=1, kind='stable')
            self._order = o[o != np.arange(self.n)[:, None]].reshape(self.n, self.n - 1)
        return self._order

    def graph(self, cutoff, max_neighbors=None, knn_only=False):
        """(edge_index [2, E] int64, rows [neighbour, centre], listed centre by centre; hits [n] as contact_kernel counts
        them: the points within the cut-off, or all n - 1 others when ``knn_only``)."""
        import numpy as np
        n, k = self.n, (max_neighbors if max_neighbors else 1000)
        hit = self.d < np.float32(cutoff)
        np.fill_diagonal(hit, False)
        hits = np.full(n, n - 1) if knn_only else hit.sum(1)
        rows = []
        for i in range(n):
            if knn_only:
                rows.append(self.order[i, :min(k, n - 1)])
            elif hits[i] == 0:
                rows.append(self.order[i, :1])
            elif hits[i] <= k:
                rows.append(np.flatnonzero(hit[i]))
            else:
                rows.append(self.order[i, :k])
        nbr = np.concatenate(rows) if rows else np.zeros(0, np.int64)
        ctr = np.repeat(np.arange(n), [len(r) for r in rows])
        return np.stack([nbr, ctr]).astype(np.int64).reshape(2, -1), hits


def contact_paths(hits, max_neighbors=None, knn_only=False):
    """Per centre, the branch of contact_kernel that writes its row, from the rule's hit counts (knn_only: hits = n - 1):
        'list_index'     0 < hits <= K, hits <= CAP     the shared-memory hit list, index order
        'rescan_index'   CAP < hits <= K                a second scan of all points, index order
        'list_select'    hits > K, hits <= CAP          K selection rounds over the list
        'rescan_select'  hits > K, hits > CAP           K selection rounds, each rescanning all points with the cut-off
        'nearest'        hits == 0                      nearest other point, by a full rescan
        'knn_list'       knn_only, n - 1 <= CAP         selection over the list
        'knn_rescan'     knn_only, n - 1 > CAP          selection by full rescans"""
    import numpy as np
    hits = np.asarray(hits)
    k = max_neighbors if max_neighbors else 1000
    if knn_only:
        return np.where(hits <= CONTACT_CAP, 'knn_list', 'knn_rescan')
    small = hits <= CONTACT_CAP
    return np.select([hits == 0, (hits <= k) & small, hits <= k, small],
                     ['nearest', 'list_index', 'rescan_index', 'list_select'], 'rescan_select')
