"""GPU: ranking packed complexes in one confidence forward per pack - ``sampling._rank_packed`` against ``_rank_batch`` per
complex for the four rankers (``AAOldModel``, ``CGOldModel``, ``CGModel`` / ``AAModel`` in confidence mode) at two widths,
``AAOldModel`` on the block layout of ``collate_packed`` against ``collate_shared_receptor``, the plain collate, the oracle
and the pinned reference confidences, the receptor work done once per distinct receptor, no host read after the per-batch
constants, ``sample_packed`` end to end, and two mutations the comparisons catch."""
import copy
from argparse import Namespace
from functools import partial

import numpy as np
import pytest
import torch

from tests.confidence_v10_fused_helpers import batch_of, fixture, pair
from tests.parity_helpers import golden_confidence_model, load_golden, rand_bn_

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')
RANKERS = ['AAOldModel', 'CGOldModel', 'CGModel', 'AAModel']
WIDTHS = {False: dict(ns=16, nv=4), True: dict(ns=48, nv=10)}


def _close(got, ref, tol):
    got, ref = got.float().cpu(), ref.float().cpu()
    return got.shape == ref.shape and float((got - ref).abs().max()) <= tol * max(1.0, float(ref.abs().max()))


def _all_atoms(cls_name):
    return cls_name in ('AAOldModel', 'AAModel')


def _ranker(cls_name, full, seed=7):
    """A seeded product ranker on cuda:0 (random BatchNorm statistics) and its ``confidence_model_args``."""
    args = Namespace(all_atoms=_all_atoms(cls_name), crop_beyond=None)
    if cls_name in ('AAOldModel', 'CGOldModel'):
        return pair(cls_name, seed, **WIDTHS[full])[1], args
    from diffdock_b200.aa_model import AAModel
    from diffdock_b200.cg_model import CGModel
    from diffdock_b200.diffusion_utils import get_timestep_embedding
    torch.manual_seed(seed)
    cls = AAModel if cls_name == 'AAModel' else CGModel
    m = cls(None, DEV, get_timestep_embedding('sinusoidal', 16, 1000), sigma_embed_dim=16, sh_lmax=2, num_conv_layers=3,
            distance_embed_dim=16, cross_distance_embed_dim=16, cross_max_distance=30.0, dynamic_max_cross=True,
            embed_also_ligand=True, confidence_mode=True, **WIDTHS[full]).eval()
    g = torch.Generator().manual_seed(seed + 1)
    for mod in m.modules():
        if mod.__class__.__name__ in ('BatchNorm', 'BatchNorm1d'):
            rand_bn_(mod, g)
    return m.to(DEV), args


def _share(dst, src):
    """The poses of ``dst`` take the receptor side of ``src`` (same stores)."""
    for d in dst:
        for k in [k for k in d._nodes if k != 'ligand']:
            d._nodes[k] = src[0]._nodes[k]
        for k in [k for k in d._edges if 'ligand' not in k]:
            d._edges[k] = src[0]._edges[k]


def _complexes(all_atoms, big=2):
    """Six complexes: receptor A for 0, 2 and 3 (interleaved with B, then consecutive), B for 1, a receptor without
    contact edges for 4, and for 5 (``big`` x 3 poses) ligands more than 5 A away from every receptor atom (empty
    ligand<-atom groups).  Ligand sizes differ between complexes."""
    from diffdock_b200.synthetic import make_pose_list
    mk = lambda n, n_res, n_lig, seed: make_pose_list(n, n_res=n_res, n_atoms=n_lig, seed=seed, tr_sigma_max=2.0, lm_dim=0,
                                                      all_atoms=all_atoms)
    cx = [mk(3, 40, 12, 1), mk(2, 48, 20, 2), mk(2, 40, 9, 3), mk(2, 40, 15, 4), mk(2, 30, 10, 5), mk(3 * big, 44, 11, 6)]
    _share(cx[2], cx[0])
    _share(cx[3], cx[0])
    for d in cx[4]:
        rr = d['receptor', 'receptor']
        rr.edge_index = rr.edge_index[:, :0]
    far = cx[5][0]['atom'].pos if all_atoms else cx[5][0]['receptor'].pos
    for d in cx[5]:
        lig = d['ligand']
        lig.pos = lig.pos + (far.max(0).values - lig.pos.min(0).values + 8.0)
        assert float(torch.cdist(lig.pos, far).min()) > 5.0
    return cx


def _finals(cx):
    """Final ligand coordinates per complex on the device: each pose's own prior coordinates."""
    return [torch.cat([d['ligand'].pos for d in p]).float().to(DEV) for p in cx]


def _count_forwards(model):
    calls = []
    real = model.forward
    model.forward = lambda data: (calls.append(data.num_graphs), real(data))[1]
    return calls


def _packed_vs_alone(model, args, cx, max_pairs):
    from diffdock_b200.sampling import _rank_batch, _rank_packed, pack_cost, pack_plan
    finals = _finals(cx)
    calls = _count_forwards(model)
    try:
        packed = _rank_packed(model, args, cx, finals, max_pairs, DEV)
        n_fwd = len(calls)
    finally:
        del model.forward
    alone = [torch.nan_to_num(_rank_batch(model, args, p, None, f, len(p), DEV), nan=-1000) for p, f in zip(cx, finals)]
    packs = pack_plan([pack_cost(p, args.all_atoms) for p in cx], max_pairs)
    assert n_fwd == len(packs)                          # one confidence forward per ranking pack
    return packed, alone, packs


# ---------------------------------------------------------------------------------------------------------------------
# 1. packed ranking against per-complex ranking
@pytest.mark.parametrize('full', [False, True])
@pytest.mark.parametrize('cls_name', RANKERS)
def test_packed_ranking_matches_ranking_complex_by_complex(built_lib, cls_name, full):
    from diffdock_b200.sampling import pack_cost
    model, args = _ranker(cls_name, full)
    assert model.sync_free_capable()
    cx = _complexes(args.all_atoms, big=4)
    costs = [pack_cost(p, args.all_atoms) for p in cx]
    budget = sum(costs[:3])                             # A, B, A in one pack; complex 5 is larger than the budget
    assert costs[5] > budget
    for max_pairs in (sum(costs), budget):
        packed, alone, packs = _packed_vs_alone(model, args, cx, max_pairs)
        if max_pairs == budget:
            assert packs[0] == [0, 1, 2] and [5] in packs
        else:
            assert packs == [list(range(6))]
        for k, (a, b) in enumerate(zip(packed, alone)):
            assert torch.isfinite(a).all() and _close(a, b, 1e-5), (cls_name, k, a, b)


# ---------------------------------------------------------------------------------------------------------------------
# 2. AAOldModel on one layout
def _timed(b, t=0.0, uniform=True):
    from diffdock_b200.diffusion_utils import set_time
    set_time(b, 0, t, t, t, b.num_graphs, True, DEV)
    if uniform:
        b._uniform_t = True
    return b


def _conf(m, b):
    with torch.no_grad():
        return m(b).float().cpu()


@pytest.mark.parametrize('full', [False, True])
def test_aaold_shared_and_packed_batches_agree_with_the_oracle(built_lib, full):
    from diffdock_b200.hetero import collate, collate_packed, collate_shared_receptor
    from diffdock_b200.synthetic import make_pose_list
    o, p = pair('AAOldModel', 61, **WIDTHS[full])
    poses = make_pose_list(4, n_res=50, n_atoms=12, seed=8, tr_sigma_max=2.0, lm_dim=0, all_atoms=True)
    sh = _conf(p, _timed(collate_shared_receptor([d.clone() for d in poses], DEV)))
    g = _timed(collate_packed([[d.clone() for d in poses]], DEV))
    pk = _conf(p, g)
    assert 'shared' in p._static(g)                     # one block: the layer-0 groups were shared
    ref = _conf(o, batch_of(poses, [0.0] * 4, 'cpu', all_atoms=True))
    assert _close(sh, pk, 1e-5) and _close(sh, ref, 1e-4) and _close(pk, ref, 1e-4), (sh, pk, ref)
    # several complexes: the packed batch against the plain collate (no layout, every copy computed) and the oracle
    cx = _complexes(True)
    flat = [d for q in cx for d in q]
    pk = _conf(p, _timed(collate_packed([[d.clone() for d in q] for q in cx], DEV)))
    plain = _conf(p, _timed(collate([d.clone() for d in flat]).to(DEV), uniform=False))
    ref = _conf(o, batch_of(flat, [0.0] * len(flat), 'cpu', all_atoms=True))
    assert _close(pk, plain, 1e-5) and _close(pk, ref, 1e-4), (pk, plain, ref)


@pytest.mark.parametrize('i', [2, 3])
def test_aaold_packed_batch_matches_the_reference_fixtures(built_lib, i):
    """The unmodified reference's confidences: ref_confidence_v10_fused.pt (fused widths, one time per pose: embeddings
    once per receptor, attributes per edge) and ref_confidence_aa.pt (ns=6: the host-sized forward)."""
    from diffdock_b200.hetero import collate_packed
    from tests.confidence_v10_fused_helpers import build
    from tests.old_score_helpers import set_times
    case = fixture()['cases'][i]
    m, poses = build(case, 'product')
    g = collate_packed([poses], DEV)
    set_times(g, case['times'], DEV)
    t = torch.as_tensor(case['times'], dtype=torch.float32, device=DEV)
    g['atom'].node_t = {k: t[g['atom'].batch] for k in ('tr', 'rot', 'tor')}
    assert _close(_conf(m, g), case['confidence'], 1e-4)
    case = load_golden('ref_confidence_aa.pt')[i - 2]
    m, poses = golden_confidence_model(case, 'product', all_atoms=True)
    assert not m.sync_free_capable()
    assert _close(_conf(m, _timed(collate_packed([poses], DEV))), case['confidence'], 1e-4)


# ---------------------------------------------------------------------------------------------------------------------
# 3. receptor work once per distinct receptor
def test_layer0_groups_and_embeddings_run_over_the_distinct_receptors(built_lib, monkeypatch):
    from diffdock_b200.hetero import collate_packed
    from diffdock_b200.tensor_layers import OldTensorProductConvLayer
    p, _ = _ranker('AAOldModel', False)
    cx = _complexes(True)
    distinct = list({id(q[0]['receptor']): q[0] for q in cx}.values())
    assert len(distinct) == 4
    n_res = sum(d['receptor'].num_nodes for d in distinct)
    n_atom = sum(d['atom'].num_nodes for d in distinct)
    e = {k: sum(d[k].num_edges for d in distinct) for k in (('receptor', 'receptor'), ('atom', 'atom'), ('atom', 'receptor'))}
    seen, rows = [], {'rec': [], 'atom': []}
    real = OldTensorProductConvLayer.accumulate_group

    def spy(self, x, group, *a, **kw):
        seen.append((self, int(group[0].shape[0]), int(a[1]), int(x.shape[0])))
        return real(self, x, group, *a, **kw)
    monkeypatch.setattr(OldTensorProductConvLayer, 'accumulate_group', spy)
    for key, enc in (('rec', p.rec_node_embedding), ('atom', p.atom_node_embedding)):
        real_f = enc.forward
        monkeypatch.setattr(enc, 'forward', (lambda k, f: lambda x: (rows[k].append(x.shape[0]), f(x))[1])(key, real_f))
    g = _timed(collate_packed(cx, DEV))
    _conf(p, g)
    assert rows == {'rec': [n_res], 'atom': [n_atom]}
    by_conv = {}
    for conv, n_e, n_out, n_x in seen:
        by_conv.setdefault(id(conv), []).append((n_e, n_out, n_x))
    C = p.conv_layers
    n_u = n_res + n_atom
    want = {6: e['receptor', 'receptor'], 8: e['atom', 'receptor'], 3: e['atom', 'atom'], 5: e['atom', 'receptor']}
    for k, n_e in want.items():
        assert by_conv[id(C[k])] == [(n_e, n_u, n_u)], (k, by_conv[id(C[k])])
    # layer 1 runs the same groups over the whole batch
    assert by_conv[id(C[9 + 6])][0][0] == g['receptor', 'receptor'].num_edges


# ---------------------------------------------------------------------------------------------------------------------
# 4. no host read after the per-batch constants
@pytest.mark.parametrize('uniform', [True, False])
def test_packed_aaold_forward_is_sync_free(built_lib, uniform):
    from diffdock_b200.hetero import collate_packed
    p, _ = _ranker('AAOldModel', True)
    b = _timed(collate_packed(_complexes(True), DEV), uniform=uniform)
    with torch.no_grad():
        first = p(b).clone()               # builds the per-batch constants (host reads of the node counts)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            again = p(b)
        finally:
            torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert _close(again, first, 1e-5)      # the same forward up to the order of float atomics


# ---------------------------------------------------------------------------------------------------------------------
# 5. sample_packed end to end
def _sample_both(conf, cargs, cx, conf_data, steps=4):
    from diffdock_b200.diffusion_utils import get_t_schedule, t_to_sigma
    from diffdock_b200.sampling import sample_packed, sampling
    from tests.test_packed_aa_gpu import _aa_model
    model, args = _aa_model(False)
    sched = get_t_schedule('expbeta', steps)
    t2s = partial(t_to_sigma, args=args)
    ids = [5, 9, 2]
    calls = _count_forwards(conf)
    try:
        packed = sample_packed([[d.clone() for d in p] for p in cx], model, steps, sched, sched, sched, DEV, t2s, args,
                               seed=11, complex_ids=ids, no_final_step_noise=True, confidence_model=conf,
                               confidence_data=conf_data, confidence_model_args=cargs)
        n_fwd = len(calls)
    finally:
        del conf.forward
    alone = [sampling([d.clone() for d in p], model, steps, sched, sched, sched, DEV, t2s, args, batch_size=len(p),
                      no_final_step_noise=True, rng='philox', seed=11, pose_keys=(cid << 32) + torch.arange(len(p)),
                      confidence_model=conf, confidence_model_args=cargs,
                      confidence_data_list=conf_data[k] if conf_data is not None else None)
             for k, (cid, p) in enumerate(zip(ids, cx))]
    torch.cuda.synchronize()
    pos = max(float((torch.stack([x['ligand'].pos for x in pl]) - torch.stack([x['ligand'].pos for x in al])).abs().max())
              for (pl, _), (al, _) in zip(packed, alone))
    return [c for _, c in packed], [c for _, c in alone], n_fwd, pos


def test_sample_packed_ranks_in_one_forward_per_ranking_pack(built_lib):
    from diffdock_b200.sampling import PACK_MAX_PAIRS, pack_cost, pack_plan
    from tests.test_packed_aa_gpu import _complexes as score_complexes
    conf, cargs = _ranker('AAOldModel', False)
    cx = score_complexes()
    conf_data = [[d.clone() for d in p] for p in cx]
    before = copy.deepcopy(conf_data)
    packed, alone, n_fwd, pos = _sample_both(conf, cargs, cx, conf_data)
    assert pos < 2e-3
    assert n_fwd == len(pack_plan([pack_cost(p, True) for p in conf_data], PACK_MAX_PAIRS)) == 1
    for a, b in zip(packed, alone):
        assert torch.isfinite(a).all() and _close(a, b, 2.5e-5), (a, b)
    for p, q in zip(conf_data, before):               # the caller's confidence graphs are not written to
        for d, e in zip(p, q):
            assert torch.equal(d['ligand'].pos, e['ligand'].pos)


def test_sample_packed_without_confidence_graphs_ranks_the_score_packs(built_lib):
    from tests.test_packed_aa_gpu import _complexes as score_complexes
    conf, cargs = _ranker('AAOldModel', False)
    packed, alone, n_fwd, pos = _sample_both(conf, cargs, score_complexes(), None)
    assert pos < 2e-3 and n_fwd == 1                   # one score pack
    for a, b in zip(packed, alone):
        assert a.shape == b.shape and torch.isfinite(a).all() and _close(a, b, 1e-4), (a, b)


def test_sample_packed_with_confidence_crop_ranks_complex_by_complex(built_lib):
    from tests.test_packed_aa_gpu import _complexes as score_complexes
    conf, _ = _ranker('CGOldModel', False)
    # the route is what is tested: a crop wide enough that every complex keeps residues around its drifted ligands
    cargs = Namespace(all_atoms=False, crop_beyond=1000.0)
    cx = score_complexes()
    conf_data = [[d.clone() for d in p] for p in cx]
    packed, alone, n_fwd, pos = _sample_both(conf, cargs, cx, conf_data)
    assert pos < 2e-3 and n_fwd == len(cx)
    for a, b in zip(packed, alone):
        assert torch.isfinite(a).all() and _close(a, b, 1e-4), (a, b)


# ---------------------------------------------------------------------------------------------------------------------
# 6. mutations
def _packed_vs_plain(p):
    from diffdock_b200.hetero import collate, collate_packed
    cx = _complexes(True)
    pk = _conf(p, _timed(collate_packed([[d.clone() for d in q] for q in cx], DEV)))
    plain = _conf(p, _timed(collate([d.clone() for q in cx for d in q]).to(DEV), uniform=False))
    return float((pk - plain).abs().max()) / max(1.0, float(plain.abs().max()))


def test_mutation_wrong_node_map_is_caught(built_lib, monkeypatch):
    from diffdock_b200.old_aa_model import AAOldModel
    p, _ = _ranker('AAOldModel', False)
    assert _packed_vs_plain(p) < 1e-5
    real = AAOldModel._receptor_tiles

    def wrong(data, B, *a):
        t = real(data, B, *a)
        if t is not None:
            t['rec']['node_map'] = t['rec']['node_map'].roll(1)
        return t
    monkeypatch.setattr(AAOldModel, '_receptor_tiles', staticmethod(wrong))
    assert _packed_vs_plain(p) > 1e-4


def test_mutation_shared_message_left_out_is_caught(built_lib, monkeypatch):
    from diffdock_b200.old_aa_model import AAOldModel
    p, _ = _ranker('AAOldModel', False)
    real = AAOldModel._shared_static_messages

    def drop(self, *a):
        acc = real(self, *a)
        acc[8][0].zero_()                  # residue <- atom messages never reach the residues
        return acc
    monkeypatch.setattr(AAOldModel, '_shared_static_messages', drop)
    assert _packed_vs_plain(p) > 1e-4
