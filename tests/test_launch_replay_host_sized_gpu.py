"""GPU: every kernel launch of host-sized forwards (``_forward_host_sized`` of CGModel, AAModel, CGOldModel and AAOldModel,
and the confidence models) replayed one launch at a time against the float64 or oracle reference of that kernel: the recorder,
per-launch checks and tolerances of test_launch_replay_gpu.

The host-sized forward reads each neighbour-list size back to the host and runs every edge group over an exactly sized list.
Users reach it with any complex of more than 10 000 residues or receptor atoms (the cross graphs' radius cap could bind), and
with convolution widths outside the fused kernel's templates (only ns / nv 48 / 10 and 16 / 4 are fused).  Its kernel uses
differ from the sync-free forward's: the streaming ``tpconv_accumulate`` / ``tpconv_finalize`` for every layer of a non-fused
width, two-layer radial MLPs on ``radial_mlp`` and deeper ones as torch Linears followed by ``radial_gemm``, the merged
single-group radial MLP of ``differentiate_convolutions=False``, the reference-signature ``TensorProductConvLayer.forward``
of the embedding stacks (second-order layers on the streaming kernel there), ``ops.radius`` with its cap of 10 000 for the
cross graphs, and the cross graph's reverse direction from ``torch.sort``.  Past 10 000 residues the CG forward builds its
cross graph with ``layers.cross_graph``: the slot-less branch of ``CGModel._cross_graph_sync_free`` is reached by no model
forward (only the sync-free forward calls it, and only up to 10 000 residues), so the test asserts it is not called.

Every workload wraps ``_forward_host_sized`` and ``_forward_sync_free`` of its model classes with call counters and asserts
that only the host-sized forward ran; every ``ddb200_*`` call is made inside a recorded wrapper (EXEMPT entry points aside).

Largest errors of the replay per launch kind over the unmutated workloads, measured in one run on an NVIDIA H100 80GB HBM3
(700 W power limit); 771 launches (17 workloads and the unmutated runs of the mutation tests), the whole file in 48 s:
  fused_conv 8.77e-6 (30 launches, the workloads past 10 000 residues or atoms), radial_mlp 1.02e-5 (213),
  radial_gemm 6.03e-6 (20), tpconv_accumulate 1.09e-6 (246), tpconv_finalize 1.07e-7, confidence_head 5.46e-7,
  pose_update 8.85e-6 (host coefficients, torch noise), pose_update_dev 9.54e-6; the 78 radius launches exact, including the
  capped cross graph of the 10 200-residue complex (every ligand atom has all 10 200 residues inside the cut-off).
Mutations: a device Clebsch-Gordan table scaled by 1 + 3e-4 in one layer is flagged on that layer's 4 tpconv_accumulate
launches while the scores move by 1.7e-5 of their maxima; two exchanged output columns of one radial MLP are flagged on
that launch while the scores move by 2.7e-4 (radial_mlp) and 8.4e-5 (radial_gemm); a cross-graph cap of 9 999 fails the
radius launch while the scores move by 5.3e-5.  A model-level 1e-4 check notices only the radial_mlp one.
The sampler run with crop_beyond found a fault: a step whose crop keeps no residue of the batch (with crop_beyond 5 the
steps kept 600, 0 and 0 of 600 residues) gave ``ddb200_radius_count`` a null x, which it rejects with DDB200_EINVAL, so
the host-sized forward raised where the reference runs on empty graphs.  ``ops.radius`` now returns no pair for an empty x
(test_host_sized_forward_of_a_receptor_cropped_to_no_residue).
Run with -s for the table of every workload and launch kind."""
import copy
from collections import Counter, defaultdict
from functools import partial

import numpy as np
import pytest
import torch
from torch import nn

from tests.parity_helpers import rel_err, table_sections
from tests.test_launch_replay_gpu import (DEV, EXEMPT, Recorder, _batch_of_ptr, _count, _failed, _oracle, _run, _shared_batch,
                                          _small_args, assert_clean, replay)

pytestmark = pytest.mark.gpu
CAP = 10000                     # max_num_neighbors of the cross graphs' radius search (models/cg_model.py:546)

TABLE = defaultdict(lambda: [0.0, 0])          # (workload, kind) -> [largest error, launches]
PATHS = {}                                     # workload -> (host-sized calls, sync-free calls, escaped, exempt calls)


class PathCount:
    """Call counters on ``_forward_host_sized`` / ``_forward_sync_free`` of the given model classes (and on
    ``CGModel._cross_graph_sync_free``, the capacity-buffer cross graph only the sync-free forward builds)."""

    def __init__(self, mp, *classes):
        from diffdock_b200.cg_model import CGModel
        self.host, self.free, self.cross_sync_free = Counter(), Counter(), 0
        for cls in set(classes):
            for name, counter in (('_forward_host_sized', self.host), ('_forward_sync_free', self.free)):
                mp.setattr(cls, name, self._counted(getattr(cls, name), counter))
        real = CGModel._cross_graph_sync_free

        def cross(model, *a, **kw):
            self.cross_sync_free += 1
            return real(model, *a, **kw)
        mp.setattr(CGModel, '_cross_graph_sync_free', cross)

    @staticmethod
    def _counted(f, counter):
        def g(model, *a, **kw):
            counter[type(model).__name__] += 1
            return f(model, *a, **kw)
        return g


def _replay(rec, paths, name):
    """Replays the workload's launches; asserts that only the host-sized forward ran and that no launch is past its
    tolerance (replay itself asserts that no ddb200 call escaped the recorder)."""
    host, free = sum(paths.host.values()), sum(paths.free.values())
    is_exempt = lambda k: k in EXEMPT or k.split(':')[0] in EXEMPT
    escaped = sum(v for k, v in rec.escaped.items() if not is_exempt(k))
    PATHS[name] = (host, free, escaped, sum(v for k, v in rec.escaped.items() if is_exempt(k)))
    out = replay(rec, name, table=TABLE)
    assert host > 0 and free == 0, f"{name}: host-sized forwards {dict(paths.host)}, sync-free {dict(paths.free)}"
    assert paths.cross_sync_free == 0
    assert_clean(out, name)
    return out


@pytest.fixture(scope='module', autouse=True)
def _print_table():
    yield
    if not TABLE:
        return
    print(f"\n[host-sized replay] {torch.cuda.get_device_name(0)}; forwards per workload:")
    for w, (host, free, esc, exempt) in sorted(PATHS.items()):
        print(f"  {w:<34s} host-sized {host:3d}  sync-free {free}  escaped {esc}  (exempt calls {exempt})")
    print("[host-sized replay] largest error per launch kind (relative per block / column / pose extent; 0 = exact):")
    kinds = defaultdict(lambda: [0.0, 0])
    for (w, k), (e, n) in sorted(TABLE.items()):
        print(f"  {w:<34s} {k:<22s} {n:6d} launches  max {e:.3e}")
        if not w.startswith('mutation'):
            kinds[k][0], kinds[k][1] = max(kinds[k][0], e), kinds[k][1] + n
    print("[host-sized replay] over the unmutated workloads:")
    for k, (e, n) in sorted(kinds.items()):
        print(f"  {k:<22s} {n:6d} launches  max {e:.3e}")
    print(f"  total {sum(n for _, n in kinds.values())} launches checked")


def _scores_moved(got, ref):
    """Largest relative change of the model outputs, as the model-level parity tests measure it (1e-4 of the maximum)."""
    got, ref = (got, ref) if isinstance(ref, tuple) else ((got,), (ref,))
    return max(rel_err(x, y) for x, y in zip(got, ref) if torch.is_tensor(y) and y.numel())


def _report(what, n_flagged, moved):
    print(f"\n[host-sized replay] {what}: replay flags {n_flagged} launches; the outputs move by {moved:.2e} of their "
          f"maxima, which a model-level 1e-4 check {'notices' if moved >= 1e-4 else 'misses'}")


# ---------------------------------------------------------------------------------------------------------------------
# workloads
def _cg24(seed, **over):
    """CGModel at ns 24 / nv 6 (outside the fused kernel's templates), three interaction layers, 16-wide embeddings."""
    from tests.parity_helpers import make_model_pair
    a = _small_args(ns=24, nv=6, num_conv_layers=3, **over)
    return make_model_pair(a, seed=seed, lm=False)[1], a


def _cg_poses(seed, n=3):
    from diffdock_b200.synthetic import make_pose_list
    return make_pose_list(n, n_res=200, n_atoms=25, seed=seed, tr_sigma_max=4.0, lm_dim=0)


@pytest.mark.parametrize('lmax', [2, 1])
@pytest.mark.parametrize('diff', [True, False], ids=['groups', 'merged'])
def test_cg_non_fused_width(built_lib, monkeypatch, lmax, diff):
    """ns 24 / nv 6: every convolution on the streaming kernel with ``radial_mlp``; ``differentiate_convolutions=False``
    runs the four edge types of a layer as one concatenated group through one radial MLP."""
    from diffdock_b200.cg_model import CGModel
    p, a = _cg24(31 + lmax, sh_lmax=lmax, differentiate_convolutions=diff)
    assert not p.sync_free_capable()
    paths = PathCount(monkeypatch, CGModel)
    rec = Recorder(monkeypatch)
    _run(rec, p, _shared_batch(_cg_poses(41 + lmax), 0.5))
    name = f"cg 24/6 lmax {lmax} {'groups' if diff else 'merged'}"
    out = _replay(rec, paths, name)
    L = len(p.conv_layers)
    # one launch per edge group of every interaction layer (4, and 2 in the last; 1 when merged) + final_conv + tor_bond_conv
    assert _count(out, 'tpconv_accumulate') == (4 * (L - 1) + 2 if diff else L) + 2, sorted(out.items())
    assert _count(out, 'radial_mlp') >= L and _count(out, 'tpconv_finalize') == L + 2
    assert _count(out, 'fused_conv') == 0 and _count(out, 'radius') >= 3


def _flag_model(flag):
    if flag == 'reduce_pseudoscalars':
        from tests.test_reduce_pseudoscalars_gpu import l_pair
        a = _small_args(ns=24, nv=6, num_conv_layers=3, reduce_pseudoscalars=True, sh_lmax=1, smooth_edges=True,
                        odd_parity=True, differentiate_convolutions=False, num_prot_emb_layers=2)
        return l_pair(a, seed=51, lm=False)[1], a
    if flag == 'second_order':
        return _cg24(52, use_second_order_repr=True, num_prot_emb_layers=2)
    from tests.test_tp_weights_layers_gpu import tw_pair
    a = _small_args(ns=24, nv=6, num_conv_layers=3, tp_weights_layers=3, embed_also_ligand=True)
    return tw_pair(a, seed=53)[1], a


@pytest.mark.parametrize('flag', ['reduce_pseudoscalars', 'second_order', 'tp_weights_layers'])
def test_cg_flag_models_non_fused_width(built_lib, monkeypatch, flag):
    """The DiffDock-L flag set (smooth edge weights, odd parity, merged groups, two receptor embedding layers through the
    reference-signature forward), second-order irreps (l = 2 blocks on the streaming kernel, also in the embedding
    stacks) and a three-layer radial MLP (torch Linears, then ``radial_gemm``) at ns 24 / nv 6."""
    from diffdock_b200.cg_model import CGModel
    p, a = _flag_model(flag)
    paths = PathCount(monkeypatch, CGModel)
    rec = Recorder(monkeypatch)
    _run(rec, p, _shared_batch(_cg_poses(61), 0.4))
    out = _replay(rec, paths, f"cg 24/6 {flag}")
    kind = 'radial_gemm' if flag == 'tp_weights_layers' else 'tpconv_accumulate'
    assert _count(out, kind) >= len(p.conv_layers), sorted(out)
    assert _count(out, 'fused_conv') == 0


@pytest.fixture(scope='module')
def cg_past_cap(built_lib):
    """CGModel at ns 48 / nv 10 (two interaction layers) and 2 poses of a 10 200-residue complex, the ligands near the
    receptor's centre: at t = 1 the cut-off 3 sigma_tr + 20 A = 77 A covers the whole receptor (radius 69 A)."""
    from diffdock_b200.synthetic import make_pose_list
    from tests.parity_helpers import make_model_pair
    a = _small_args(ns=48, nv=10, num_conv_layers=2)
    _, p = make_model_pair(a, seed=71, lm=False)
    poses = make_pose_list(2, n_res=10200, n_atoms=12, seed=72, tr_sigma_max=2.0, lm_dim=0, max_neighbors=10)
    assert p.sync_free_capable()              # a fused width: only the residue count sends it to the host-sized forward
    return p, a, poses


def _cross_radius(records):
    """The recorded cross-graph radius launches (cap 10 000) and the oracle's uncapped neighbour count of each ligand atom."""
    found = []
    for path, a, ret, _, _ in records:
        if path == 'ops.radius' and a['max_num_neighbors'] == CAP:
            row, _ = _oracle(a['x'], a['y'], _batch_of_ptr(a['x_ptr']), a['y_batch'].long().cpu(), a['r'], a['r_per_graph'],
                             1 << 30)
            found.append((ret, torch.bincount(row, minlength=a['y'].shape[0])))
    return found


def test_cg_radius_cap_binds_past_10000_residues(cg_past_cap, monkeypatch):
    """A complex of 10 200 residues at t = 1: the cross graph's radius cap binds in a real forward (some ligand atom has
    more than 10 000 residues inside the cut-off, per the oracle's uncapped search), and the radius launches equal the
    oracle exactly with the cap the call passed; the fused kernel runs over the exactly sized lists."""
    from diffdock_b200.cg_model import CGModel
    p, a, poses = cg_past_cap
    paths = PathCount(monkeypatch, CGModel)
    rec = Recorder(monkeypatch)
    g = _shared_batch(poses, 1.0, a)
    assert int(g['receptor'].pos.shape[0]) == 2 * 10200
    _run(rec, p, g)
    cross = _cross_radius(rec.records)
    assert len(cross) == 1, "one cross-graph radius search per forward"
    (row, _, cnt), uncapped = cross[0]
    assert int(uncapped.max()) > CAP, f"the cap does not bind: at most {int(uncapped.max())} residues in the cut-off"
    assert int(cnt.max()) == CAP and int((uncapped > CAP).sum()) > 0
    print(f"\n[host-sized replay] 10 200 residues at t = 1: up to {int(uncapped.max())} residues within the cut-off of a "
          f"ligand atom, {int((uncapped > CAP).sum())} of {uncapped.shape[0]} ligand atoms capped at {CAP}")
    out = _replay(rec, paths, "cg 48/10 10200 residues t=1")
    assert _count(out, 'radius') >= 3 and _count(out, 'fused_conv') >= 4, sorted(out)     # rr, lr, rl; lr of the last layer


def test_all_atom_models_past_10000_atoms(built_lib, monkeypatch):
    """AAModel (score, ns 16 / nv 4) and AAOldModel (v1.0 ranker with an LM embedding, ns 48 / nv 10) on a receptor of
    more than 10 000 atoms: fused widths, sent to the host-sized forward by the atom count alone."""
    from diffdock_b200.aa_model import AAModel
    from diffdock_b200.diffusion_utils import set_time
    from diffdock_b200.hetero import collate
    from diffdock_b200.old_aa_model import AAOldModel
    from diffdock_b200.synthetic import make_pose_list
    from tests.confidence_v10_fused_helpers import batch_of as v10_batch, pair as v10_pair
    from tests.test_tp_weights_layers_gpu import tw_pair
    poses = make_pose_list(2, n_res=2100, n_atoms=15, seed=81, tr_sigma_max=3.0, lm_dim=32, all_atoms=True)
    n_atoms = int(poses[0]['atom'].pos.shape[0])
    assert n_atoms > CAP, f"{n_atoms} receptor atoms"
    print(f"\n[host-sized replay] all-atom receptor: 2100 residues, {n_atoms} atoms")

    a = _small_args(num_conv_layers=2, tp_weights_layers=2, embed_also_ligand=True)
    p = tw_pair(a, seed=82, model='aa')[1]
    assert p.sync_free_capable()
    paths = PathCount(monkeypatch, AAModel)
    rec = Recorder(monkeypatch)
    g = collate([q.clone() for q in poses]).to(DEV)
    g['receptor'].x = g['receptor'].x[:, :1]             # the score model reads no LM embedding
    set_time(g, None, 0.3, 0.3, 0.3, 2, True, DEV)
    _run(rec, p, g)
    out = _replay(rec, paths, f"aa score 16/4 {n_atoms} atoms")
    assert _count(out, 'fused_conv') >= 9, sorted(out)
    monkeypatch.undo()

    _, m = v10_pair('AAOldModel', 83, num_conv_layers=2, lm_embedding_type='esm', lm_embedding_dim=32)
    assert m.sync_free_capable()
    paths = PathCount(monkeypatch, AAOldModel)
    rec = Recorder(monkeypatch, conf_model=m)
    _run(rec, m, v10_batch(poses, [0.2, 0.2], DEV, all_atoms=True, shared=True))
    out = _replay(rec, paths, f"aa v1.0 ranker 48/10 {n_atoms} atoms")
    assert _count(out, 'confidence_head') == 1 and _count(out, 'fused_conv') >= 9, sorted(out)


@pytest.mark.parametrize('which', ['v1.0 score', 'v1.0 confidence', 'v1.1 confidence', 'v1.0 aa confidence'])
def test_confidence_and_v10_models_non_fused_width(built_lib, monkeypatch, which):
    """ns 24 / nv 6: CGOldModel in score and confidence mode (the v1.0 wiring, every convolution through the
    reference-signature forward), CGModel(confidence_mode=True) with the atom head, and AAOldModel on a small complex."""
    from diffdock_b200.hetero import collate
    from diffdock_b200.synthetic import make_pose_list
    aa = which == 'v1.0 aa confidence'
    poses = make_pose_list(2, n_res=150 if aa else 200, n_atoms=20, seed=91, tr_sigma_max=3.0, lm_dim=32 if aa else 0,
                           all_atoms=aa)
    if which == 'v1.0 score':
        from tests.old_score_helpers import model_pair, set_times
        _, m, _ = model_pair(seed=92, ns=24, nv=6, num_conv_layers=3, sigma_embed_dim=16, distance_embed_dim=16, lm_dim=0)
        g = collate([q.clone() for q in poses]).to(DEV)
        set_times(g, [0.3, 0.6], DEV)
    elif which == 'v1.1 confidence':
        from tests.confidence_v11_helpers import batch_of
        from tests.test_confidence_v11_gpu import _pair
        _, m = _pair('CGModel', 93, ns=24, nv=6)
        g = batch_of(poses, [0.0, 0.4], DEV)
    else:
        from tests.confidence_v10_fused_helpers import batch_of as v10_batch, pair as v10_pair
        kw = dict(lm_embedding_type='esm', lm_embedding_dim=32) if aa else {}
        _, m = v10_pair('AAOldModel' if aa else 'CGOldModel', 94, ns=24, nv=6, **kw)
        g = v10_batch(poses, [0.2, 0.2], DEV, all_atoms=aa, shared=True)
    assert not m.sync_free_capable()
    paths = PathCount(monkeypatch, type(m))
    rec = Recorder(monkeypatch, conf_model=m if 'confidence' in which else None)
    _run(rec, m, g)
    out = _replay(rec, paths, f"{which} 24/6")
    assert _count(out, 'tpconv_accumulate') >= 2 * m.num_conv_layers and _count(out, 'fused_conv') == 0, sorted(out)
    assert _count(out, 'confidence_head') == (1 if 'confidence' in which else 0)


@pytest.mark.parametrize('mode', ['torch noise, crop_beyond', 'philox'])
def test_sampling_host_sized(built_lib, monkeypatch, mode):
    """sampling() for 3 steps with the ns 24 / nv 6 CGModel and a ns 24 / nv 6 ranker (CGOldModel, CGModel confidence):
    the eager step loop.  With torch noise and ``crop_beyond`` every step crops the receptor (``crop_receptor``, one
    radius search of cap 1) and moves the poses with ``ddb200_pose_update`` on host coefficients and torch.normal noise;
    with ``rng='philox'`` through ``ddb200_pose_update_dev``."""
    from diffdock_b200.cg_model import CGModel
    from diffdock_b200.diffusion_utils import get_t_schedule, t_to_sigma
    from diffdock_b200.old_cg_model import CGOldModel
    from diffdock_b200.sampling import sampling
    from diffdock_b200.synthetic import default_model_args, make_pose_list
    crop = mode != 'philox'
    p, a = _cg24(101, crop_beyond=25.0 if crop else None)
    if crop:
        from tests.confidence_v10_fused_helpers import pair as v10_pair
        ranker = v10_pair('CGOldModel', 102, ns=24, nv=6)[1]
    else:
        from tests.test_confidence_v11_gpu import _pair
        ranker = _pair('CGModel', 103, ns=24, nv=6)[1]
    poses = make_pose_list(3, n_res=200, n_atoms=22, seed=104, tr_sigma_max=a.tr_sigma_max, lm_dim=0)
    conf_poses = [q.clone() for q in poses]
    sched = get_t_schedule('expbeta', 3)
    paths = PathCount(monkeypatch, CGModel, CGOldModel)
    rec = Recorder(monkeypatch, conf_model=ranker)
    torch.manual_seed(105)
    rec.start()
    _, conf = sampling(poses, p, 3, sched, sched, sched, DEV, partial(t_to_sigma, args=a), a, batch_size=3,
                       no_final_step_noise=True, confidence_model=ranker, confidence_data_list=conf_poses,
                       confidence_model_args=default_model_args(), rng=None if crop else 'philox', seed=21)
    rec.stop()
    assert conf.shape[0] == 3 and bool(torch.isfinite(conf).all())
    if crop:        # residues of the batch each step's crop keeps (the crop's search has cap 1)
        kept = [int((r[2][2] > 0).sum()) for r in rec.records if r[0] == 'ops.radius' and r[1]['max_num_neighbors'] == 1]
        assert len(kept) == 3
        print(f"\n[host-sized replay] crop_beyond 25: residues kept per step {kept} of {3 * 200}")
    out = _replay(rec, paths, f"sampling 3 steps, {mode}")
    assert paths.host['CGModel'] == 3 + (0 if crop else 1) and paths.host['CGOldModel'] == (1 if crop else 0)
    assert _count(out, 'pose_update' if crop else 'pose_update_dev') == 3 and _count(out, 'confidence_head') == 1
    if crop:        # the crop searches: cap 1, ligand atoms as the searched points
        assert _count(out, 'radius') >= 3 * 4 + 1, sorted(out.items())


def test_host_sized_forward_of_a_receptor_cropped_to_no_residue(built_lib, monkeypatch):
    """``crop_beyond`` can leave a batch without any residue: every ligand farther than the cut-off from its receptor, as
    after a large early step of the sampler.  The reference runs such a batch with empty contact and cross graphs.  The
    cross graph's ``ops.radius`` over no residue used to fail with DDB200_EINVAL (the entry points take no null x); it now
    returns no pair and the host-sized forward runs."""
    from diffdock_b200.cg_model import CGModel
    from diffdock_b200.diffusion_utils import set_time
    from diffdock_b200.hetero import collate_shared_receptor
    from diffdock_b200.sampling import crop_receptor
    p, a = _cg24(131)
    g = crop_receptor(collate_shared_receptor([q.clone() for q in _cg_poses(132)], DEV), 1e-3)
    assert g['receptor'].pos.shape[0] == 0 and g['receptor', 'receptor'].edge_index.shape[1] == 0
    set_time(g, None, 0.5, 0.5, 0.5, 3, False, DEV)
    paths = PathCount(monkeypatch, CGModel)
    rec = Recorder(monkeypatch)
    tr, rot, tor, _ = _run(rec, p, g)
    assert all(bool(torch.isfinite(t).all()) for t in (tr, rot, tor))
    out = _replay(rec, paths, "cg 24/6 cropped to no residue")
    assert _count(out, 'radius') == 3 and _count(out, 'tpconv_accumulate') == len(p.conv_layers) + 2, sorted(out)


# ---------------------------------------------------------------------------------------------------------------------
# mutations the replay must catch
def _scaled_device_table(handle, factor):
    """A handle whose DEVICE table has the Clebsch-Gordan terms of its widest l_out = 1 path scaled by ``factor``, while
    ``handle.table`` (what the replay's reference reads) stays the true table."""
    from diffdock_b200.ops import TpHandle
    t = handle.table
    paths = sorted(t.paths, key=lambda q: (q.i_out, q.w_ref_off))          # the kernel's path order (tp_table._compile)
    pi = max((i for i, q in enumerate(paths) if q.l_out == 1), key=lambda i: paths[i].mul_in)
    psec, _, _, ment = table_sections(t)
    m0, n_m = int(psec[pi][5]), int(psec[pi][2] * psec[pi][3])
    fb = t.fblob.copy()
    hit = 0
    for mi, tb, tc in ment:
        if m0 <= mi < m0 + n_m:
            fb[tb:tb + tc] *= np.float32(factor)
            hit += 1
    assert hit
    mt = copy.copy(t)
    mt.fblob = fb
    h = TpHandle(mt)
    h.table = t
    return h


def _run_pair(rec, p, poses, name, mutate):
    """The workload unmutated (replayed clean), then with ``mutate()`` applied; returns (replay of the mutated run, how far
    the outputs moved)."""
    ref = _run(rec, p, _shared_batch(poses, 0.5))
    assert_clean(replay(rec, f"{name} (unmutated)", table=TABLE), name)
    mutate()
    got = _run(rec, p, _shared_batch(poses, 0.5))
    return replay(rec, f"mutation {name}", table=TABLE), _scores_moved(got, ref)


def test_mutation_tp_table_of_one_host_sized_layer(built_lib, monkeypatch):
    """One interaction layer's TpHandle with the device Clebsch-Gordan terms of its widest l_out = 1 path scaled by
    1 + 3e-4: the replay flags that layer's tpconv_accumulate launches and no other launch."""
    p, a = _cg24(111)
    layer = p.conv_layers[1]

    def mutate():
        layer.tp._handles[True] = _scaled_device_table(layer.tp.handle(True), 1 + 3e-4)
    rec = Recorder(monkeypatch)
    out, moved = _run_pair(rec, p, _cg_poses(112), "tp table x (1 + 3e-4)", mutate)
    bad = _failed(out, 'tpconv_accumulate')
    assert bad, "the replay missed a device Clebsch-Gordan table scaled by 1 + 3e-4"
    assert len(bad) == len(layer.fc), "only the mutated layer's launches are wrong"
    assert not [b for k, v in out.items() if k != 'tpconv_accumulate' for b in v[3]]
    _report("tp table x (1 + 3e-4) in one layer", len(bad), moved)


@pytest.mark.parametrize('kind', ['radial_mlp', 'radial_gemm'])
def test_mutation_radial_output_columns_exchanged(built_lib, monkeypatch, kind):
    """One radial MLP whose output-layer image has two weight columns of ``table.w_perm`` exchanged: the per-edge weights of
    that group land in each other's slots.  ``radial_mlp`` (two-layer MLP) or ``radial_gemm`` (three layers) is flagged;
    the tensor-product launches, which take those weights as inputs, still pass."""
    from diffdock_b200.tensor_layers import TensorProductConvLayer
    if kind == 'radial_gemm':
        from tests.test_tp_weights_layers_gpu import tw_pair
        p = tw_pair(_small_args(ns=24, nv=6, num_conv_layers=3, tp_weights_layers=3, embed_also_ligand=True), seed=121)[1]
    else:
        p, _ = _cg24(121)
    layer = p.conv_layers[1]
    target = layer.fc[0] if isinstance(layer.fc, nn.ModuleList) else layer.fc
    orig = TensorProductConvLayer._last_linear

    def exchanged(self, fc, table):
        W, b = orig(self, fc, table)
        if fc is not target:
            return W, b
        i, j = np.nonzero(np.asarray(table.w_perm) >= 0)[0][[0, -1]]
        W, b = W.detach().clone(), b.detach().clone()
        W[[i, j]], b[[i, j]] = W[[j, i]], b[[j, i]]
        return W, b

    def mutate():
        monkeypatch.setattr(TensorProductConvLayer, '_last_linear', exchanged)
        for cache in (layer._wcache, layer._fcache, layer._gcache):
            cache.clear()
    rec = Recorder(monkeypatch)
    out, moved = _run_pair(rec, p, _cg_poses(122), f"{kind} columns exchanged", mutate)
    bad = _failed(out, kind)
    assert bad, f"the replay missed {kind} writing two weight columns exchanged"
    assert not _failed(out, 'tpconv'), "the weights are the tensor product's inputs: its launches stay right"
    _report(f"{kind} with two w_perm columns exchanged", len(bad), moved)


def test_mutation_cross_radius_cap_9999(cg_past_cap, monkeypatch):
    """The 10 200-residue workload with the cross graph's radius launches given max_num_neighbors = 9 999 instead of the
    10 000 the call passed: the replay of the radius launch fails its exact comparison with the oracle."""
    p, a, poses = cg_past_cap
    rec = Recorder(monkeypatch)
    ref = _run(rec, p, _shared_batch(poses, 1.0, a))
    cap = lambda args: args[:7] + (CAP - 1 if args[7] == CAP else args[7],) + args[8:]
    rec.call_mutation.update({'ddb200_radius_count': cap, 'ddb200_radius_fill': cap})
    got = _run(rec, p, _shared_batch(poses, 1.0, a))
    with pytest.raises(AssertionError, match='^radius'):
        replay(rec, "mutation cap 9999", table=TABLE)
    path, args = rec._replaying[rec._cur][:2]
    assert path == 'ops.radius' and args['max_num_neighbors'] == CAP, (path, args.get('max_num_neighbors'))
    _report("cross-graph radius cap 9 999 (call passed 10 000)", 1, _scores_moved(got, ref))
