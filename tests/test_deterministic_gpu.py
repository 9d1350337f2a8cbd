"""GPU: bit-reproducible forwards and sampling under ``torch.use_deterministic_algorithms(True)``.

Under the flag the convolutions scatter 64-bit fixed-point values (``ddb200_fused_conv_fixed`` / ``_so_fixed``,
``ddb200_tpconv_accumulate_fixed``, ``ddb200_tpconv_finalize_fixed``; arithmetic restated in
tests/test_deterministic_cpu.py).  Checked here, all with the flag on and ``CUBLAS_WORKSPACE_CONFIG`` set:
  1. every fused tile kind, the second-order and the deep-MLP instantiation and the streaming kernel against float64 at
     the tolerances of the per-launch tests, and the int64 sums against the restated sum of each edge's rounded message;
  2. the int64 sums bit for bit under shuffled edges, prepended foreign edges and a list split over several launches;
  3. two forwards of real models give equal outputs, within 1e-4 of the flag-off outputs (and the oracle for CGModel);
  4. two calls of ``sampling`` (graphed, eager, crop_beyond, visualization_list), ``sample_packed`` with an AAOldModel
     ranker and the per-rank shares of ``sample_packed_sharded`` give equal poses and confidences;
  5. the captured step replays without a host synchronisation;
  6. a value outside the fixed-point range sets the error word and ``sampling`` raises;
  7. with the flag off no fixed-point entry point is called."""
import copy
from functools import partial

import numpy as np
import pytest
import torch

from tests.parity_helpers import block_errors, fused_table, make_model_pair, rel_err
from tests.test_deterministic_cpu import restated_fixed_sum
from tests.test_fused_conv_cta128_gpu import _runs, _sms
from tests.test_fused_conv_fp64_gpu import TOL, Case
from tests.test_second_order_cpu import so_tables
from tests.test_tp_weights_layers_gpu import DeepCase

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
FIXED_NAMES = ('ddb200_fused_conv_fixed', 'ddb200_fused_conv_so_fixed', 'ddb200_tpconv_accumulate_fixed',
               'ddb200_tpconv_finalize_fixed')


@pytest.fixture
def det(monkeypatch):
    monkeypatch.setenv('CUBLAS_WORKSPACE_CONFIG', ':4096:8')
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev)


def _flag_off(fn):
    torch.use_deterministic_algorithms(False)
    try:
        return fn()
    finally:
        torch.use_deterministic_algorithms(True)


# ------------------------------------------------------------------------------------------------ 1. kernels vs float64
def _fused_fixed(c, tgt=None, n_out=None, sl=None, acc=None, **over):
    """int64 sums and counts of one fused launch of case ``c`` (edges ``sl`` of its list), into ``acc`` if given."""
    from diffdock_b200 import fused, ops
    n_out = n_out or c.n_out
    s, n = acc if acc is not None else ops.new_accumulators(n_out, c.table.d_out, DEV)
    assert s.dtype == torch.int64
    a = dict(ea=c.ea, node=c.node, x=c.x, vec=c.vec, tgt=c.tgt if tgt is None else tgt, src=c.src)
    a.update(over)
    sl = sl or slice(0, a['tgt'].shape[0])
    fused.fused_conv(c.plan, a['ea'][sl], a['node'], c.ns, a['tgt'][sl].contiguous(), a['src'][sl].contiguous(), a['x'],
                     a['vec'][sl].contiguous(), s, n)
    torch.cuda.synchronize()
    return s, n


def _per_edge_messages(c):
    """Each edge's fp32 message: the float kernel with every edge on its own row (one reduction onto zero)."""
    from diffdock_b200 import fused
    E = c.tgt.shape[0]
    out = torch.zeros(E, c.table.d_out, device=DEV)
    cnt = torch.zeros(E, device=DEV)
    fused.fused_conv(c.plan, c.ea, c.node, c.ns, torch.arange(E, dtype=torch.int32, device=DEV), c.src, c.x, c.vec, out,
                     cnt)
    torch.cuda.synchronize()
    return out


def _finalized(s, n):
    from diffdock_b200 import ops
    return ops.tpconv_finalize(s, n, False)


N_NODES = 1200          # more than the target rows of _runs over these edge counts: the radial MLP gathers node[tgt]
# (table, ne, gathered node scalars, H, edges, seed); gather=False drops the node scalars, so that an edge's message does not
# depend on its target row
_SPECS = {
    'ns16_nv4_lmax2': (lambda: fused_table(16, 4, 3, 2, False), 16, 16, 48, 3, 501),
    'ns16_nv4_lmax1': (lambda: fused_table(16, 4, 1, 1, False), 16, 16, 48, 3, 502),
    'ns48_nv10_lmax2': (lambda: fused_table(48, 10, 3, 2, False), 48, 48, 144, 2, 503),
    'ns48_nv10_lmax1': (lambda: fused_table(48, 10, 2, 1, False), 48, 48, 144, 2, 504),
    'second_order': (lambda: so_tables(48, 10, 2)[3], 48, 48, 144, 2, 505),
    'tp_weights_layers_3': (lambda: fused_table(16, 4, 3, 2, False), 16, 16, 48, 2, 506),
}


def _fused_case(name, gather=True):
    table, ne, ns, H, tiles, seed = _SPECS[name]
    E = tiles * _sms() * 128 + 17
    ns = ns if gather else 0
    if name == 'tp_weights_layers_3':
        return DeepCase(table(), ne, ns, H, E, seed=seed, layers=3, n_nodes=N_NODES)
    return Case(table(), ne, ns, H, E, seed=seed, n_nodes=N_NODES)


def _with_runs(c, seed):
    """CSR targets of runs that cross tile boundaries (tests/test_fused_conv_cta128_gpu.py:_runs)."""
    tgt, n_out = _runs(c.E, torch.Generator().manual_seed(seed))
    c.tgt, c.n_out = tgt.cuda(), max(n_out, int(tgt.max()) + 1)
    assert c.n_out < N_NODES
    return c


FUSED_CASES = list(_SPECS)


@pytest.mark.parametrize('name', FUSED_CASES)
def test_fused_fixed_matches_fp64_and_the_restated_sum(built_lib, det, name):
    c = _with_runs(_fused_case(name), 7)
    s, n = _fused_fixed(c)
    ref, rcnt = c.reference()
    assert torch.equal(n.double(), rcnt)
    errs = block_errors(_finalized(s, n), ref, c.table.out_irreps)
    print(f"\n[fixed fused] {name}: max block err {max(errs.values()):.2e}")
    assert max(errs.values()) < TOL, errs
    if not c.plan.second_order:          # second order: a (10, 5) block is converted once per tile, not once per edge
        c = _with_runs(_fused_case(name, gather=False), 8)
        s, _ = _fused_fixed(c)
        m = _per_edge_messages(c)
        want = restated_fixed_sum(m.cpu().numpy(), c.tgt.cpu().numpy(), c.n_out)
        diff = np.abs(s.cpu().numpy() - want)
        per_row = np.bincount(c.tgt.cpu().numpy(), minlength=c.n_out)[:, None]
        print(f"[fixed fused] {name}: restated-sum difference max {diff.max()} units")
        assert (diff <= per_row).all()


def _tpconv_case(pattern='csr', E=20000, seed=601):
    from tests.test_tpconv_fp64_gpu import Case as TpCase, _table
    return TpCase(_table('ladder_48_10_s3_l2'), E, seed, pattern=pattern)


def _tpconv_fixed(c, h, sl=slice(None), acc=None, tgt=None):
    from diffdock_b200 import ops
    s, n = acc if acc is not None else ops.new_accumulators(c.n_out, c.table.d_out, DEV)
    t = c.tgt if tgt is None else tgt
    ops.tpconv_accumulate(h, c.x, c.src[sl].contiguous(), t[sl].contiguous(), c.geo[sl].contiguous(), c.w[sl], s, n,
                          edge_weight=c.ew[sl] if c.ew is not None else None)
    torch.cuda.synchronize()
    return s, n


def test_streaming_fixed_matches_fp64_and_the_restated_sum(built_lib, det):
    from diffdock_b200 import ops
    from tests.test_tpconv_fp64_gpu import TOL as TP_TOL
    c = _tpconv_case()
    h = ops.TpHandle(c.table)
    s, n = _tpconv_fixed(c, h)
    ref, rcnt = c.reference()
    assert torch.equal(n.double(), rcnt)
    errs = block_errors(_finalized(s, n), ref, c.table.out_irreps)
    print(f"\n[fixed tpconv] max block err {max(errs.values()):.2e}")
    assert max(errs.values()) < TP_TOL, errs
    m = torch.zeros(c.E, c.table.d_out, device=DEV)           # every edge's message on its own row, fp32 kernel
    ops.tpconv_accumulate(h, c.x, c.src, torch.arange(c.E, dtype=torch.int32, device=DEV), c.geo, c.w, m, None,
                          edge_weight=c.ew)
    want = restated_fixed_sum(m.cpu().numpy(), c.tgt.cpu().numpy(), c.n_out)
    per_row = np.bincount(c.tgt.cpu().numpy(), minlength=c.n_out)[:, None]
    assert (np.abs(s.cpu().numpy() - want) <= per_row).all()


def test_fixed_finalize_restated(built_lib, det):
    from diffdock_b200 import ops
    from tests.test_deterministic_cpu import restated_finalize
    g = torch.Generator().manual_seed(3)
    s = (torch.randn(97, 40, generator=g, dtype=torch.float64) * 2.0 ** 36).long()
    n = torch.randint(0, 9, (97,), generator=g).float()
    sc, sh = torch.rand(40, generator=g) + 0.5, torch.randn(40, generator=g)
    res = torch.randn(97, 24, generator=g)
    got = ops.tpconv_finalize(s.cuda(), n.cuda(), True, sc.cuda(), sh.cuda(), res.cuda()).cpu()
    want = restated_finalize(s.numpy(), n.numpy(), True, sc.numpy(), sh.numpy(), res.numpy())
    assert np.array_equal(got.numpy(), want)
    got = ops.tpconv_finalize(s.cuda(), n.cuda(), False).cpu()
    assert np.array_equal(got.numpy(), restated_finalize(s.numpy(), n.numpy(), False, None, None, None))


# ------------------------------------------------------------------------------------------- 2. order independence
@pytest.mark.parametrize('name', ['ns16_nv4_lmax2', 'ns48_nv10_lmax2', 'second_order', 'tp_weights_layers_3'])
def test_fused_fixed_sums_do_not_depend_on_edge_placement(built_lib, det, name):
    c = _with_runs(_fused_case(name), 11)
    base, bcnt = _fused_fixed(c)
    g = torch.Generator().manual_seed(12)
    # shuffled within and across runs
    perm = torch.randperm(c.E, generator=g).cuda()
    s, _ = _fused_fixed(c, tgt=c.tgt[perm], src=c.src[perm], ea=c.ea[perm], vec=c.vec[perm])
    assert torch.equal(s, base), 'shuffled edges'
    # foreign edges in front: every run crosses other tile boundaries
    for k in (1, 37, 64, 101):
        pre = torch.full((k,), c.n_out, dtype=torch.int32, device=DEV)
        s, _ = _fused_fixed(c, tgt=torch.cat([pre, c.tgt]), n_out=c.n_out + 1, src=torch.cat([c.src[:k], c.src]),
                            ea=torch.cat([c.ea[:k], c.ea]), vec=torch.cat([c.vec[:k], c.vec]))
        assert torch.equal(s[:c.n_out], base), f'{k} foreign edges in front'
    # the list split over several launches into one buffer
    cuts = [0, 1000, 1001, 5555, c.E]
    acc = None
    for a, b in zip(cuts[:-1], cuts[1:]):
        acc = _fused_fixed(c, sl=slice(a, b), acc=acc)
    assert torch.equal(acc[0], base) and torch.equal(acc[1], bcnt), 'split launches'


def test_streaming_fixed_sums_do_not_depend_on_edge_placement(built_lib, det):
    from diffdock_b200 import ops
    c = _tpconv_case(seed=602)
    h = ops.TpHandle(c.table)
    base, _ = _tpconv_fixed(c, h)
    perm = torch.randperm(c.E, generator=torch.Generator().manual_seed(5)).cuda()
    c2 = copy.copy(c)
    c2.src, c2.tgt, c2.geo, c2.w = c.src[perm], c.tgt[perm], c.geo[perm], c.w[perm]
    c2.ew = c.ew[perm] if c.ew is not None else None
    s, _ = _tpconv_fixed(c2, h)
    assert torch.equal(s, base), 'shuffled edges'
    acc = None
    for a, b in ((0, 31), (31, 7000), (7000, c.E)):
        acc = _tpconv_fixed(c, h, sl=slice(a, b), acc=acc)
    assert torch.equal(acc[0], base), 'split launches'


# ---------------------------------------------------------------------------------------- 3. repeatable forwards
def _cg_args(**over):
    from diffdock_b200.synthetic import default_model_args
    kw = dict(ns=16, nv=4, sh_lmax=2, num_conv_layers=3, distance_embed_dim=16, cross_distance_embed_dim=16,
              sigma_embed_dim=16)
    kw.update(over)
    return default_model_args(**kw)


def _score_batch(poses, t, all_atoms=False):
    from diffdock_b200.diffusion_utils import set_time
    from diffdock_b200.hetero import collate
    g = collate([d.clone() for d in poses]).to(DEV)
    set_time(g, None, t, t, t, len(poses), all_atoms, DEV)
    return g


def _outputs(out):
    out = out if isinstance(out, (tuple, list)) else (out,)
    return [o.clone() for o in out if torch.is_tensor(o)]


def _repeatable(fn):
    """Two flag-on calls equal bit for bit; returns their outputs and the flag-off ones."""
    a, b = _outputs(fn()), _outputs(fn())
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    off = _outputs(_flag_off(fn))
    for x, y in zip(a, off):
        if y.numel():
            assert rel_err(x, y) < 1e-4
    return a


@pytest.mark.parametrize('path', ['sync_free', 'host_sized'])
def test_cg_model_forward_is_repeatable(built_lib, det, path):
    from diffdock_b200.synthetic import make_pose_list
    from diffdock_b200.hetero import collate
    from oracle.diffusion import set_time as o_set_time
    args = _cg_args() if path == 'sync_free' else _cg_args(ns=24, nv=6)
    o, p = make_model_pair(args, seed=3)
    poses = make_pose_list(3, n_res=60, n_atoms=12, seed=11, tr_sigma_max=args.tr_sigma_max * 0.5)
    calls = {'sync_free': 0, 'host_sized': 0}
    for k in calls:
        real = getattr(p, f'_forward_{k}')
        setattr(p, f'_forward_{k}', (lambda r, k: lambda *a: (calls.__setitem__(k, calls[k] + 1), r(*a))[1])(real, k))
    got = _repeatable(lambda: p(_score_batch(poses, 0.5)))
    assert calls[path] > 0 and calls['host_sized' if path == 'sync_free' else 'sync_free'] == 0, calls
    g_cpu = collate(poses)
    o_set_time(g_cpu, 0.5, 0.5, 0.5, 3, 'cpu')
    with torch.no_grad():
        ref = o(g_cpu)
    for a, b in zip(got[:3], ref[:3]):
        if b.numel():
            assert rel_err(a, b) < 1e-4


def test_score_models_aa_and_v10_forwards_are_repeatable(built_lib, det):
    from diffdock_b200.synthetic import make_pose_list
    from tests.old_score_helpers import model_pair
    from tests.test_packed_aa_gpu import _aa_model
    aa, _ = _aa_model(False)
    aa_poses = make_pose_list(3, n_res=40, n_atoms=12, seed=5, tr_sigma_max=5.0, lm_dim=0, all_atoms=True)
    _repeatable(lambda: aa(_score_batch(aa_poses, 0.4, all_atoms=True)))
    _, old, _ = model_pair(seed=2, ns=16, nv=4, num_conv_layers=3, sigma_embed_dim=16, distance_embed_dim=16)
    old_poses = make_pose_list(3, n_res=50, n_atoms=12, seed=6, tr_sigma_max=5.0)
    _repeatable(lambda: old(_score_batch(old_poses, 0.4)))


@pytest.mark.parametrize('cls_name', ['CGOldModel', 'AAOldModel', 'CGModel'])
def test_confidence_forwards_are_repeatable(built_lib, det, cls_name):
    from diffdock_b200.sampling import _rank_batch
    from tests.test_packed_rank_gpu import _complexes, _finals, _ranker
    model, args = _ranker(cls_name, False)
    cx = _complexes(args.all_atoms)[:2]
    finals = _finals(cx)
    for p, f in zip(cx, finals):
        _repeatable(lambda: _rank_batch(model, args, p, None, f, len(p), DEV))


# --------------------------------------------------------------------------------------- 4. repeatable sampling
class _Frames:
    def __init__(self):
        self.seen = []

    def add(self, coords, part=0, order=1, repeat=1):
        self.seen.append((part, order, coords.clone()))


def _sample(p, args, poses, steps=6, **kw):
    from diffdock_b200.diffusion_utils import get_t_schedule, t_to_sigma
    from diffdock_b200.sampling import sampling
    sched = get_t_schedule('expbeta', steps)
    out, conf = sampling([q.clone() for q in poses], p, steps, sched, sched, sched, DEV, partial(t_to_sigma, args=args),
                         args, batch_size=len(poses), no_final_step_noise=True, **kw)
    torch.cuda.synchronize()
    return torch.stack([d['ligand'].pos for d in out]).cpu(), conf


def _cg_old_ranker():
    """A seeded v1.0 ranker that reads the score graphs' language-model features (as tests/test_packed_sharded_gpu.py)."""
    from types import SimpleNamespace
    from diffdock_b200.diffusion_utils import get_timestep_embedding
    from diffdock_b200.old_cg_model import CGOldModel
    torch.manual_seed(4)
    conf = CGOldModel(None, torch.device(DEV), get_timestep_embedding('sinusoidal', 16, 1000), ns=16, nv=4,
                      num_conv_layers=2, sigma_embed_dim=16, distance_embed_dim=16, cross_distance_embed_dim=16,
                      confidence_mode=True, use_old_atom_encoder=True, lm_embedding_type='esm', lm_embedding_dim=1280,
                      dynamic_max_cross=True, cross_max_distance=80.0).eval().to(DEV)
    return conf, SimpleNamespace(crop_beyond=None, all_atoms=False)


@pytest.mark.parametrize('mode', ['graphed', 'eager', 'crop', 'frames'])
def test_sampling_is_repeatable(built_lib, det, mode):
    from diffdock_b200.synthetic import make_pose_list
    args = _cg_args(crop_beyond=20.0) if mode == 'crop' else _cg_args()
    _, p = make_model_pair(args, seed=9)
    conf, cargs = _cg_old_ranker()
    poses = make_pose_list(4, n_res=60, n_atoms=12, seed=41, tr_sigma_max=args.tr_sigma_max)
    for i, q in enumerate(poses):
        q.original_center = torch.tensor([[2.0 * i, 1.5, -1.0]])
    kw = dict(rng='philox', seed=123, cuda_graph=mode != 'eager', confidence_model=conf, confidence_model_args=cargs)
    runs = []
    for _ in range(2):
        vis = [_Frames() for _ in poses] if mode == 'frames' else None
        pos, c = _sample(p, args, poses, visualization_list=vis, **kw)
        runs.append((pos, c.cpu(), vis))
    (p0, c0, v0), (p1, c1, v1) = runs
    assert torch.isfinite(p0).all() and torch.equal(p0, p1) and torch.equal(c0, c1)
    if v0 is not None:
        for a, b in zip(v0, v1):
            assert len(a.seen) == len(b.seen) and all(torch.equal(x[2], y[2]) for x, y in zip(a.seen, b.seen))
    off, _ = _flag_off(lambda: _sample(p, args, poses, **kw))
    print(f"\n[fixed sampling] {mode}: largest |dpos| against the flag-off run {float((off - p0).abs().max()):.2e} A")


def test_sample_packed_and_sharded_shares_are_repeatable(built_lib, det):
    from tests.test_packed_sharded_gpu import _emulated, _one_call, _setup
    model, args, kw, load, costs, shapes = _setup('aa')
    a, b = _one_call(model, args, kw, load, len(costs)), _one_call(model, args, kw, load, len(costs))
    for (p, c), (q, e) in zip(a, b):
        assert torch.equal(p, q) and torch.equal(c, e)
    model, args, kw, load, costs, shapes = _setup('cg_crop')
    one = _one_call(model, args, kw, load, len(costs))
    x, y = (_emulated(model, args, kw, load, costs, shapes, 2) for _ in range(2))
    d = 0.0
    for (p, c), (q, e), (r, _) in zip(x, y, one):
        assert torch.equal(p, q) and torch.equal(c, e)
        d = max(d, float((p.cpu() - r.cpu()).abs().max()))
    print(f"\n[fixed sharded] world 2 against one call: largest |dpos| {d:.2e} A (not asserted: cuBLAS batch sizes)")


# -------------------------------------------------------------------------------------------------- 5. no host sync
def test_captured_step_replays_without_host_sync(built_lib, det):
    from diffdock_b200.diffusion_utils import get_t_schedule, t_to_sigma
    from diffdock_b200.hetero import collate_shared_receptor
    from diffdock_b200.sampling import GraphedSteps, crop_cutoff2, step_coefficients
    from diffdock_b200.synthetic import make_pose_list
    args = _cg_args(crop_beyond=20.0)
    _, p = make_model_pair(args, seed=31)
    n = 4
    poses = make_pose_list(n, n_res=120, n_atoms=12, seed=71, tr_sigma_max=args.tr_sigma_max)
    g = collate_shared_receptor(poses, DEV)
    sched = get_t_schedule('expbeta', 6)
    t2s = partial(t_to_sigma, args=args)
    coef = [step_coefficients(i, 6, sched, sched, sched, t2s, args, False, 1.0, 0.0, 0.5) for i in range(6)]
    lig0 = poses[0]['ligand']
    rb = poses[0]['ligand', 'ligand'].edge_index.T[lig0.edge_mask]
    bu, bv = rb[:, 0].int().contiguous().to(DEV), rb[:, 1].int().contiguous().to(DEV)
    mask = torch.from_numpy(lig0.mask_rotate[0].astype(np.uint8)).to(DEV)
    steps = GraphedSteps(p, g, n, coef, [[float(t)] * 3 for t in sched], bu, bv, mask, True, DEV, draw_noise=True,
                         philox=(3, torch.arange(n, device=DEV)),
                         crop_rows=[crop_cutoff2(t2s, t, t, t, 20.0) for t in sched])
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        steps.run(6)
        done = steps.step.clone()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert int(done.item()) == 6 and torch.isfinite(steps.pos).all()


# ------------------------------------------------------------------------------------------------------ 6. saturation
def test_saturation_sets_the_error_word_and_sampling_raises(built_lib, det):
    from diffdock_b200 import ops
    from diffdock_b200.synthetic import make_pose_list
    c = _fused_case('ns16_nv4_lmax2')
    ops.check_fixed_error()                          # clear
    c.x = c.x * 1e12                                 # messages of order 1e12 > 2^31
    _fused_fixed(c)
    assert int(ops.fixed_error_word(DEV).item()) & 1
    with pytest.raises(RuntimeError, match='fixed-point range'):
        ops.check_fixed_error(DEV)
    assert int(ops.fixed_error_word(DEV).item()) == 0
    args = _cg_args()
    _, p = make_model_pair(args, seed=9)
    with torch.no_grad():                            # layer 0's radial MLP output bias: messages of order 1e12
        fc = p.conv_layers[0].fc
        for f in (fc if isinstance(fc, torch.nn.ModuleList) else [fc]):
            f[-1].bias.mul_(1e12)
    poses = make_pose_list(2, n_res=60, n_atoms=12, seed=41, tr_sigma_max=args.tr_sigma_max)
    with pytest.raises(RuntimeError, match='fixed-point range'):
        _sample(p, args, poses, steps=2, rng='philox', seed=1, cuda_graph=False)
    assert int(ops.fixed_error_word(DEV).item()) == 0


# ------------------------------------------------------------------------------------------------ 7. default untouched
def test_flag_off_calls_no_fixed_point_entry_point(built_lib):
    from diffdock_b200 import _lib
    from diffdock_b200.synthetic import make_pose_list
    assert not torch.are_deterministic_algorithms_enabled()
    L = _lib.lib()
    called = []
    saved = {n: getattr(L, n) for n in FIXED_NAMES}
    for n in FIXED_NAMES:
        setattr(L, n, (lambda n: lambda *a: called.append(n) or saved[n](*a))(n))
    try:
        args = _cg_args(crop_beyond=20.0)
        _, p = make_model_pair(args, seed=9)
        poses = make_pose_list(3, n_res=60, n_atoms=12, seed=41, tr_sigma_max=args.tr_sigma_max)
        _sample(p, args, poses, steps=3, rng='philox', seed=1)
        _, wide = make_model_pair(_cg_args(ns=24, nv=6), seed=3)         # host-sized forward
        wide(_score_batch(poses, 0.5))
        c = _fused_case('ns16_nv4_lmax2')
        c.run()
    finally:
        for n, f in saved.items():
            setattr(L, n, f)
    assert called == []
