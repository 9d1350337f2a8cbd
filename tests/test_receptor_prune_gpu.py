"""GPU: the sync-free forward drops the receptor <- receptor messages that cannot reach a ligand atom
(CGModel._pruned_contact_groups).  The need sets (ddb200_receptor_need) are compared bit for bit with a breadth-first
search on the host, the need-filtered edge selection (ddb200_crop_select_edges) exactly with boolean-mask indexing, and the
pruned forward / captured sampler with the same model running every contact edge (``_prune_receptor = False``)."""
import copy
from functools import partial

import numpy as np
import pytest
import torch

from tests.parity_helpers import rel_err

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
TOL = 1e-4          # the sync-free against host-sized tolerance; two unpruned runs differ by a few 1e-5 (atomics order)


# ---------------------------------------------------------------------------------------------------------------------
# need sets and edge selection
def _bfs(cross_tgt, n_live, offset, tgt, src, n_rec, n_levels, keep=None):
    """R_1 .. R_n_levels on the host: the live reverse cross targets, then one contact hop back per level."""
    need = np.zeros((n_levels, n_rec), dtype=np.uint8)
    need[0, np.asarray(cross_tgt[:n_live]) - offset] = 1
    ok = np.ones(len(tgt), dtype=bool) if keep is None else keep[tgt] & keep[src]
    for k in range(1, n_levels):
        need[k] = need[k - 1]
        need[k, src[ok & (need[k - 1][tgt] == 1)]] = 1
    return need


def _contact_lists(sizes, k, seed):
    """A kNN-like contact list (k sources per target, CSR by target) over complexes of ``sizes`` residues laid out one after
    the other: ``(tgt, src, gid)`` int numpy arrays."""
    rng = np.random.default_rng(seed)
    tgt, src, gid, off = [], [], [], 0
    for b, n in enumerate(sizes):
        pos = rng.normal(size=(n, 3)) * n ** (1 / 3) * 2.0
        d = np.linalg.norm(pos[:, None] - pos[None], axis=-1)
        np.fill_diagonal(d, np.inf)
        nb = np.argsort(d, axis=1)[:, :k]
        tgt.append(np.repeat(np.arange(n), k) + off)
        src.append(nb.reshape(-1) + off)
        gid.append(np.full(n * k, b))
        off += n
    return np.concatenate(tgt), np.concatenate(src), np.concatenate(gid)


def _i32(a):
    return torch.as_tensor(np.asarray(a), dtype=torch.int32, device=DEV).contiguous()


@pytest.mark.parametrize("case", ['local', 'empty', 'whole', 'cropped'])
def test_need_sets_match_host_bfs_bit_for_bit(built_lib, case):
    from diffdock_b200 import ops
    sizes, n_lig, n_levels = (300, 170), 57, 5
    tgt, src, _ = _contact_lists(sizes, 6, seed=3)
    n_rec = sum(sizes)
    rng = np.random.default_rng(11)
    if case == 'empty':
        live = np.zeros(0, dtype=np.int64)                        # a pose without any cross edge: R_1 empty
    elif case == 'whole':
        live = rng.permutation(np.repeat(np.arange(n_rec), 2))    # every residue is a cross target
    else:                                                         # a few residues of each complex
        live = np.concatenate([rng.choice(300, 7, replace=False), 300 + rng.choice(170, 4, replace=False)])
    live = np.sort(live) + n_lig
    # capacity rows past the live count hold other residues: they must not enter R_1
    cap = np.concatenate([live, n_lig + rng.integers(0, n_rec, size=400)])
    keep = None
    if case == 'cropped':
        keep = rng.uniform(size=n_rec) < 0.6
        keep[live - n_lig] = True                                 # cross targets are never cropped away
    got = ops.receptor_need(_i32(cap), _i32([len(live)]), n_lig, _i32(tgt), _i32(src), n_rec, n_levels,
                            keep=torch.as_tensor(keep, device=DEV) if keep is not None else None)
    want = _bfs(cap, len(live), n_lig, tgt, src, n_rec, n_levels, keep)
    assert np.array_equal(got.cpu().numpy(), want)
    if case == 'local':
        assert 0 < want[0].sum() < want[-1].sum() < n_rec        # the sets grow and stay proper
    if case == 'empty':
        assert want.sum() == 0
    if case == 'whole':
        assert want.all()
    # the second complex's residues enter only through its own cross targets
    if case in ('local', 'cropped'):
        assert want[:, 300:].any() and want[:, :300].any()


@pytest.mark.parametrize("with_keep", [False, True])
def test_need_filtered_selection_matches_boolean_mask(built_lib, with_keep):
    from diffdock_b200 import ops
    tgt, src, gid = _contact_lists((250, 130), 8, seed=5)
    n_rec, off = 380, 23
    rng = np.random.default_rng(2)
    need = rng.uniform(size=n_rec) < 0.3
    keep = rng.uniform(size=n_rec) < 0.7 if with_keep else None
    # a buffer set reused from an earlier, larger selection: stale rows must not leak into the result
    out = ops.select_edges_buffers(len(tgt), torch.device(DEV))
    ops.crop_select_edges(_i32(tgt), _i32(src), None, _i32(gid), offset=off, out=out)
    t, s, perm, g, n_dev = ops.crop_select_edges(_i32(tgt), _i32(src),
                                                 torch.as_tensor(keep, device=DEV) if keep is not None else None,
                                                 _i32(gid), offset=off, need=torch.as_tensor(need, device=DEV), out=out)
    sel = need[tgt] & (keep[tgt] & keep[src] if keep is not None else True)
    idx = np.nonzero(sel)[0]                                      # CSR order kept
    n = int(n_dev.item())
    assert n == len(idx) and 0 < n < len(tgt)
    assert np.array_equal(perm[:n].cpu().numpy(), idx)
    assert np.array_equal(t[:n].cpu().numpy(), tgt[idx] + off)
    assert np.array_equal(s[:n].cpu().numpy(), src[idx] + off)
    assert np.array_equal(g[:n].cpu().numpy(), gid[idx])


# ---------------------------------------------------------------------------------------------------------------------
# forward: pruned against every contact edge
def _model(over=None, confidence=False, seed=0):
    from bench import model_kwargs, randomise_bn
    from diffdock_b200.cg_model import CGModel
    from diffdock_b200.diffusion_utils import get_timestep_embedding, t_to_sigma
    from diffdock_b200.synthetic import default_model_args
    a = default_model_args(**(over or {}))
    kw = model_kwargs(a)
    kw.update(reduce_pseudoscalars=a.reduce_pseudoscalars, smooth_edges=a.smooth_edges, odd_parity=a.odd_parity)
    if confidence:
        kw.update(confidence_mode=True)
    torch.manual_seed(seed)
    m = CGModel(partial(t_to_sigma, args=a), torch.device(DEV),
                get_timestep_embedding('sinusoidal', a.sigma_embed_dim, a.embedding_scale), **kw).eval()
    randomise_bn(m, seed + 1)
    m = m.to(DEV)
    assert m.sync_free_capable()
    return m, a


def _batch(a, poses, t, shared, crop_beyond=None):
    from diffdock_b200.diffusion_utils import set_time, t_to_sigma
    from diffdock_b200.hetero import collate, collate_shared_receptor
    from diffdock_b200.sampling import crop_cutoff2
    n = len(poses)
    g = collate_shared_receptor(copy.deepcopy(poses), DEV) if shared else collate(copy.deepcopy(poses)).to(DEV)
    set_time(g, None, t, t, t, n, False, DEV)
    g._uniform_t = True
    if crop_beyond is not None:
        t2s = partial(t_to_sigma, args=a)
        g._crop = (torch.tensor([crop_cutoff2(t2s, t, t, t, crop_beyond)], dtype=torch.float32, device=DEV),
                   torch.zeros(1, dtype=torch.int32, device=DEV))
    return g


def _run(m, g, prune):
    m._prune_receptor = prune
    try:
        out = m(g)
        torch.cuda.synchronize()
        return [o.clone() if torch.is_tensor(o) else o for o in out]
    finally:
        m._prune_receptor = True


def _compare(m, a, poses, t, shared, crop_beyond=None):
    """max relative error of the pruned outputs against the unpruned ones, and the live fraction of the R_1 set."""
    g = _batch(a, poses, t, shared, crop_beyond)
    got, ref = _run(m, g, True), _run(m, g, False)
    errs = [rel_err(x, y) for x, y in zip(got, ref) if torch.is_tensor(x) and x.numel()]
    assert errs and all(np.isfinite(errs))
    c = m._static(g)
    need = [v[0] for k, v in c.items() if isinstance(k, tuple) and k[0] == 'prune']
    frac = float(need[0][0].float().mean()) if need else None
    return max(errs), frac


@pytest.fixture(scope='module')
def full_case():
    from diffdock_b200.synthetic import make_pose_list
    m, a = _model()
    return m, a, make_pose_list(40, n_res=1500, n_atoms=40, seed=100, tr_sigma_max=a.tr_sigma_max)


@pytest.mark.parametrize("t", [1.0, 0.5, 0.05])
@pytest.mark.parametrize("shared", [True, False])
def test_full_size_pruned_forward_matches_unpruned(built_lib, full_case, t, shared):
    from diffdock_b200.synthetic import make_pose_list
    m, a, _ = full_case
    poses = make_pose_list(40, n_res=1500, n_atoms=40, seed=100, tr_sigma_max=a.tr_sigma_max * t)
    err, frac = _compare(m, a, poses, t, shared)
    assert err < TOL, err
    if t < 1.0:
        assert frac < 0.9                       # R_1 is a proper subset: the comparison covers dropped edges


def test_full_size_cropped_pruned_forward_matches_unpruned(built_lib, full_case):
    from diffdock_b200.synthetic import make_pose_list
    m, a, _ = full_case
    poses = make_pose_list(40, n_res=1500, n_atoms=40, seed=100, tr_sigma_max=a.tr_sigma_max * 0.5)
    err, _ = _compare(m, a, poses, 0.5, True, crop_beyond=20.0)
    assert err < TOL, err


def test_pruning_one_hop_short_changes_the_scores(built_lib, full_case, monkeypatch):
    """R_k instead of R_{k+1} at every pruned layer (R_0: no residue): the comparison above must notice."""
    from diffdock_b200 import ops
    from diffdock_b200.synthetic import make_pose_list
    m, a, _ = full_case
    exact = ops.receptor_need

    def short(*args, **kw):
        need = exact(*args, **kw)
        need[1:] = need[:-1].clone()
        need[0] = 0
        return need
    monkeypatch.setattr(ops, 'receptor_need', short)
    poses = make_pose_list(40, n_res=1500, n_atoms=40, seed=100, tr_sigma_max=a.tr_sigma_max * 0.5)
    err, _ = _compare(m, a, poses, 0.5, True)
    assert err > 10 * TOL, err


@pytest.mark.parametrize("name,over,confidence", [
    ('sh_lmax1', dict(sh_lmax=1), False),
    ('diffdock_l', dict(sh_lmax=1, num_prot_emb_layers=3, reduce_pseudoscalars=True, smooth_edges=True, odd_parity=True),
     False),
    ('layers2', dict(num_conv_layers=2), False),
    ('layers3', dict(num_conv_layers=3), False),
    ('confidence', dict(num_conv_layers=4), True),
])
@pytest.mark.parametrize("shared", [True, False])
def test_model_variants_pruned_forward_matches_unpruned(built_lib, name, over, confidence, shared):
    from diffdock_b200.synthetic import make_pose_list
    m, a = _model(over, confidence=confidence, seed=4)
    t = 0.2
    poses = make_pose_list(6, n_res=1200, n_atoms=20, seed=8, tr_sigma_max=a.tr_sigma_max * t)
    err, frac = _compare(m, a, poses, t, shared)
    assert err < TOL, (name, err)
    if not (over.get('num_conv_layers') == 2 and shared):      # 2 layers with shared layer-0 messages: nothing to prune
        assert frac is not None and frac < 0.9


def test_sample_packed_two_receptors_pruned_matches_unpruned(built_lib):
    from diffdock_b200.diffusion_utils import get_t_schedule, t_to_sigma
    from diffdock_b200.sampling import sample_packed
    from diffdock_b200.synthetic import make_pose_list
    m, a = _model(seed=6)
    cx = [make_pose_list(3, n_res=500, n_atoms=14, seed=21, tr_sigma_max=5.0),
          make_pose_list(4, n_res=350, n_atoms=22, seed=22, tr_sigma_max=5.0)]
    sched = get_t_schedule('expbeta', 6)
    t2s = partial(t_to_sigma, args=a)
    out = {}
    for prune in (True, False):
        m._prune_receptor = prune
        res = sample_packed([[d.clone() for d in p] for p in cx], m, 6, sched, sched, sched, DEV, t2s, a, seed=11,
                            complex_ids=[1, 2], no_final_step_noise=True, cuda_graph=True)
        out[prune] = [torch.stack([x['ligand'].pos for x in pl]).cpu() for pl, _ in res]
    m._prune_receptor = True
    d = max(float((x - y).abs().max()) for x, y in zip(out[True], out[False]))
    assert d < 1e-2, d


# ---------------------------------------------------------------------------------------------------------------------
# captured sampler: 20 steps, Philox noise
def test_graphed_20_steps_pruned_within_unpruned_spread_and_sync_free(built_lib, full_case):
    from bench import N_SCHED, TEMPS
    from diffdock_b200.diffusion_utils import get_t_schedule, t_to_sigma
    from diffdock_b200.hetero import collate_shared_receptor
    from diffdock_b200.sampling import GraphedSteps, step_coefficients
    m, a, poses = full_case
    n = len(poses)
    t2s = partial(t_to_sigma, args=a)
    sched = get_t_schedule('expbeta', N_SCHED)
    coef = []
    for i in range(N_SCHED):
        c = step_coefficients(i, N_SCHED, sched, sched, sched, t2s, a, False, **TEMPS)
        if i == N_SCHED - 1:
            c[1] = c[3] = c[5] = 0.0
        coef.append(c)
    lig0 = poses[0]['ligand']
    rb = poses[0]['ligand', 'ligand'].edge_index.T[lig0.edge_mask]
    bu, bv = rb[:, 0].int().contiguous().to(DEV), rb[:, 1].int().contiguous().to(DEV)
    mask = torch.from_numpy(lig0.mask_rotate[0].astype(np.uint8)).to(DEV)
    keys = torch.arange(n, device=DEV)

    def run(prune, sync_check=False):
        m._prune_receptor = prune
        try:
            g = collate_shared_receptor(copy.deepcopy(poses), DEV)
            s = GraphedSteps(m, g, n, coef, [[float(t)] * 3 for t in sched], bu, bv, mask, True, DEV, draw_noise=True,
                             philox=(1234, keys))
            torch.cuda.synchronize()
            if sync_check:
                torch.cuda.set_sync_debug_mode("error")
            try:
                s.run(N_SCHED)
                if sync_check:
                    s.step.fill_(N_SCHED // 2)
                    m(g)                   # the pruned forward launched op by op
            finally:
                torch.cuda.set_sync_debug_mode(0)
            torch.cuda.synchronize()
            pos = s.pos.clone().cpu()
            del s, g
            torch.cuda.empty_cache()
            return pos
        finally:
            m._prune_receptor = True

    ref_a, ref_b, got = run(False), run(False), run(True, sync_check=True)
    assert torch.isfinite(got).all()
    spread = float((ref_a - ref_b).abs().max())
    d = (got - ref_a).abs()
    assert float(d.max()) < 1e-2, (float(d.max()), spread)
    assert float(d.median()) < 1e-3, float(d.median())
