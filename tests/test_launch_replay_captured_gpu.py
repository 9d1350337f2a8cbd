"""GPU: every kernel launch of the captured reverse-diffusion step, replay by replay, and of packed sampling and ranking,
against the float64 or oracle reference of that kernel: the per-launch checks and tolerances of test_launch_replay_gpu.

``sampling(cuda_graph=True)`` and ``sample_packed`` capture one step as a CUDA graph (``sampling.GraphedSteps``) and replay it
once per step; the captured and eager final coordinates are compared elsewhere at 2e-3 after 6 chained steps, which a
per-launch error of 1e-4 cannot show through.  The recorder of test_launch_replay_gpu clones each launch's inputs and
outputs.  A clone taken while the step is being captured is itself part of the graph (allocated in its pool, copied between
the product's kernels), so every replay refreshes it with that replay's values.  Here ``GraphedSteps.run`` replays one step
at a time, synchronises and checks that step's launches; the eager warm-up step, which the sampler keeps as step 0, is
checked like any eager launch (so each workload uses a model that has not met its batch shape).  On every replay k, beyond
the per-launch references:
  - every recorded ``step_dev`` snapshot is k: each launch check reads its table row through that snapshot, so a stale step
    counter would otherwise pass as consistent;
  - the captured step makes the same sequence of launches as the eager warm-up step of the same batch;
  - no ddb200 entry point is called outside a recorded wrapper during the capture;
  - with ``rng=None`` (torch.normal inside the graph) the tr / rot / tor noise differs between every two steps, and the
    pooled draws have the mean and variance of N(0, 1) within NOISE_SE standard errors;
  - a launch with no live edge leaves its accumulator bit-identical (block_errors fails any change over an all-zero
    reference); such launches are counted in the table.
The mutation tests make one argument a legal but wrong value: the crop kernel and the packed pose update reading table row 0
at every step (``step_dev`` NULL), and in-graph noise replaced by one tensor drawn before the capture.  Run with -s for the
largest error per (workload, launch kind) at every step of the schedule.

Largest errors per launch kind over the unmutated workloads, measured in one run on an NVIDIA H100 80GB HBM3 (700 W power
limit); 5333 launches, the whole file in 58 s:
  fused_conv 1.77e-5 (2009 launches), swapped 1.01e-5 (14), radial_mlp 1.09e-5, tpconv_accumulate 3.05e-6,
  tpconv_finalize 1.23e-7, edge_embed 6.05e-7, confidence_head 2.10e-7 (one launch per ranking pack), pose_update_dev
  6.63e-6, pose_update_packed 6.69e-6; graph, crop and need kernels exact at every step.
The errors do not grow along the schedule: the fused convolution's largest error per step stays between 6e-6 and 1.8e-5
from step 0 to step 19, including the steps where the 1 A crop keeps no residue (53 convolution launches with no live edge
in that workload, every accumulator unchanged).  The noise drawn in the graph: 1380 draws over 20 steps, mean +0.051 (bound
0.135), variance 0.977 (bound 1 +- 0.190), no two steps alike.  With the crop reading row 0 the replay flags crop_flags from
step 3 on, while the final coordinates move by 8.3e-4 from the eager sampler's, which the 2e-3 comparison misses."""
import math
from collections import Counter, defaultdict
from functools import partial

import pytest
import torch

from tests.test_launch_replay_gpu import DEV, EXEMPT, Recorder, _small_args, replay

pytestmark = pytest.mark.gpu
NOISE_SE = 5.0       # bound on the pooled noise mean and variance, in standard errors (|mean| < 5 / sqrt(n), ...)

STEP_TABLE = defaultdict(lambda: [0.0, 0])     # (workload, step, kind) -> [largest error, launches]
KIND_TABLE = defaultdict(lambda: [0.0, 0])     # (workload, kind) -> [largest error, launches]
ZERO_LIVE = Counter()                          # (workload, wrapper) -> launches whose device live count was 0
LIVE_COUNTED = ('fused.fused_conv', 'ops.edge_embed')


def _escaped(counts):
    return {k: v for k, v in counts.items() if k not in EXEMPT and k.split(':')[0] not in EXEMPT}


def _first_diff(a, b):
    i = next((i for i, (x, y) in enumerate(zip(a, b)) if x != y), min(len(a), len(b)))
    return f"{len(a)} eager / {len(b)} captured launches, first difference at {i}: {a[i:i + 2]} / {b[i:i + 2]}"


class CapturedReplay:
    """Patches ``GraphedSteps`` so that each replay of a step graph is followed by the check of that step's launches."""

    def __init__(self, mp, rec, name, model):
        from diffdock_b200 import sampling as smod
        self.rec, self.name = rec, name
        self.failures = []          # (step, what, detail)
        self.per_step = {}          # step -> Counter {kind: launches checked}
        self.noise = {}             # step -> host copy of the step's tr / rot / tor noise
        self.kept = {}              # step -> (residues kept by the crop, residues)
        self.batches, self.mark = [], None
        real_static = model._static

        def static(data):           # the first call of a GraphedSteps: what follows it is the eager warm-up step
            c = real_static(data)
            if self.mark is None:
                self.mark = len(rec.records)
            return c
        mp.setattr(model, '_static', static)
        real_init = smod.GraphedSteps.__init__

        def init(gs, *a, **kw):
            self.mark = None
            rec.captured.clear()          # the records of an earlier batch's graph
            real_init(gs, *a, **kw)
        mp.setattr(smod.GraphedSteps, '__init__', init)
        mp.setattr(smod.GraphedSteps, 'run', lambda gs, n: self._run(gs, n))

    def _run(self, gs, n_steps):
        rec = self.rec
        self.batches.append(gs.g)
        assert gs.steps_done == 1 and self.mark is not None, \
            f"{self.name}: no eager warm-up step (the model had met this batch shape): its kernels were not loaded"
        warm = rec.records[self.mark:]
        if [r[0] for r in warm] != [r[0] for r in rec.captured]:
            self.failures.append((0, 'launch sequence', _first_diff([r[0] for r in warm], [r[0] for r in rec.captured])))
        esc = _escaped(rec.cap_escaped)
        assert not esc and sum(rec.cap_matched.values()), f"{self.name}: ddb200 calls outside the recorder in the capture: {esc}"
        self._check(0, rec.records, warm, clear=True)
        for k in range(gs.steps_done, n_steps):
            gs.graph.replay()
            torch.cuda.synchronize()
            self._check(k, rec.captured, rec.captured, clear=False)
        gs.steps_done = n_steps
        return gs.pos

    def _check(self, k, records, step_records, clear):
        rec = self.rec
        rec.active = False            # nothing the references call is recorded
        try:
            for path, a, ret, post, ctx in step_records:
                s = a.get('step_dev')
                if torch.is_tensor(s) and int(s.reshape(-1)[0]) != k:
                    self.failures.append((k, 'step', f"{path} read step {int(s.reshape(-1)[0])}"))
                n_dev = a.get('n_edges_dev')
                if path in LIVE_COUNTED and n_dev is not None and int(n_dev.reshape(-1)[0]) == 0:
                    ZERO_LIVE[(self.name, path)] += 1
                if path == 'ops.crop_flags':
                    self.kept[k] = (int(ret[0].sum()), int(ret[0].numel()))
                if path == 'ops.pose_update_dev' and a['tr_z'] is not None:
                    self.noise[k] = torch.cat([a[z].reshape(-1).cpu() for z in ('tr_z', 'rot_z', 'tor_z') if a[z] is not None])
            rec._cur = None
            try:
                out = replay(rec, self.name, records, clear=clear, table=KIND_TABLE)
            except AssertionError as e:        # an exact kernel (graph, crop) differs from its reference, or a call escaped
                what = records[rec._cur][0] if rec._cur is not None else 'replay'
                self.failures.append((k, what, str(e).splitlines()[0]))
                if clear:
                    records.clear()
                return
        finally:
            rec.active = True
        for kind, (e, tol, n, bad) in out.items():
            cell = STEP_TABLE[(self.name, k, kind)]
            cell[0], cell[1] = max(cell[0], e), cell[1] + n
            if bad:
                self.failures.append((k, kind, bad[:3]))
        self.per_step.setdefault(k, Counter()).update({kind: v[2] for kind, v in out.items()})

    def flagged(self, what):
        return sorted({k for k, w, _ in self.failures if what in w})

    def summary(self, steps, pose_kind, crop=False):
        """Asserts that every replay (steps 1 .. steps - 1 of each captured batch) was checked with at least one
        convolution, one pose update and, with cropping, one crop launch; prints the counts."""
        replays = sorted(k for k in self.per_step if k > 0)
        assert self.batches and replays == list(range(1, steps)), (self.name, replays)
        for k in range(steps):
            c = self.per_step[k]
            assert sum(n for kind, n in c.items() if kind.startswith('fused_conv')) >= len(self.batches), (k, c)
            assert c[pose_kind] == len(self.batches), (k, c)
            if crop:
                assert c['crop_flags'] >= len(self.batches), (k, c)
        total = sum(sum(c.values()) for c in self.per_step.values())
        kinds = Counter()
        for c in self.per_step.values():
            kinds.update(c)
        print(f"\n[captured replay] {self.name}: {len(self.batches)} step graph(s), {len(replays)} replays + the eager "
              f"warm-up step, {total} launches checked ({', '.join(f'{k} {n}' for k, n in sorted(kinds.items()))})")
        if self.kept:
            print(f"  crop kept {[self.kept[k][0] for k in sorted(self.kept)]} of {self.kept[0][1]} residues by step")
        return total


def noise_failures(noise):
    """What is wrong with the noise of the steps ``noise`` {step: draws}: two steps with identical draws, or pooled draws
    whose mean or variance is more than NOISE_SE standard errors from N(0, 1)'s."""
    steps = sorted(noise)
    same = [(i, j) for x, i in enumerate(steps) for j in steps[x + 1:] if torch.equal(noise[i], noise[j])]
    z = torch.cat([noise[k] for k in steps]).double()
    n, mean, var = z.numel(), float(z.mean()), float(z.var())
    bad = [f"identical noise at steps {same[:6]}"] if same else []
    if abs(mean) > NOISE_SE / math.sqrt(n):
        bad.append(f"pooled mean {mean:.4f} of {n} draws")
    if abs(var - 1.0) > NOISE_SE * math.sqrt(2.0 / n):
        bad.append(f"pooled variance {var:.4f} of {n} draws")
    print(f"  noise: {len(steps)} steps, {n} draws, mean {mean:+.4f} (bound {NOISE_SE / math.sqrt(n):.4f}), variance "
          f"{var:.4f} (bound 1 +- {NOISE_SE * math.sqrt(2.0 / n):.4f}), {len(same)} pairs of steps identical")
    return bad


@pytest.fixture(scope='module', autouse=True)
def _print_table():
    yield
    if not STEP_TABLE:
        return
    print(f"\n[captured replay] {torch.cuda.get_device_name(0)}; largest error per launch kind at each step (relative per "
          f"block / column / pose extent; 0 = exact comparison passed; - = no launch):")
    for w in sorted({w for w, _, _ in STEP_TABLE}):
        steps = sorted({k for ww, k, _ in STEP_TABLE if ww == w})
        print(f"  {w}   steps {steps[0]} .. {steps[-1]}")
        for kind in sorted({kd for ww, _, kd in STEP_TABLE if ww == w}):
            row = [STEP_TABLE.get((w, k, kind)) for k in steps]
            cells = ' '.join('-' if c is None else ('0' if c[0] == 0 else f"{c[0]:.1e}") for c in row)
            print(f"    {kind:<22s} {sum(c[1] for c in row if c):5d}  {cells}")
        zl = {p: n for (ww, p), n in ZERO_LIVE.items() if ww == w}
        if zl:
            print(f"    launches with no live edge (accumulator unchanged): {zl}")
    kinds = defaultdict(lambda: [0.0, 0])
    for (w, k), (e, n) in KIND_TABLE.items():
        if not w.startswith('mutation'):
            kinds[k][0], kinds[k][1] = max(kinds[k][0], e), kinds[k][1] + n
    print("[captured replay] over the unmutated workloads:")
    for k, (e, n) in sorted(kinds.items()):
        print(f"  {k:<24s} {n:6d} launches  max {e:.3e}")
    print(f"  total {sum(n for _, n in kinds.values())} launches checked")


# ---------------------------------------------------------------------------------------------------------------------
# workloads
SMALL = {
    'torch_noise': dict(rng=None),
    'philox_crop20': dict(rng='philox', seed=21, crop_beyond=20.0),
    'no_random_crop4': dict(no_random=True, crop_beyond=4.0),
    'no_random_crop1': dict(no_random=True, crop_beyond=1.0),
}


def _small_workload(mode):
    """A fresh ns 16 / nv 4 CGModel, its arguments, 3 poses of a 300-residue complex and the sampling() options of
    ``mode``.  The Philox run keeps its ligands within reach of the receptor (tr_sigma_max 5), as the eager sampler it is
    compared with in the mutation test needs."""
    from diffdock_b200.synthetic import make_pose_list
    from tests.parity_helpers import make_model_pair
    kw = dict(SMALL[mode])
    crop = kw.pop('crop_beyond', None)
    a = _small_args(tr_sigma_max=5.0) if mode == 'philox_crop20' else _small_args()
    a.crop_beyond = crop
    _, p = make_model_pair(a, seed=15, lm=False)
    poses = make_pose_list(3, n_res=300, n_atoms=25, seed=12, tr_sigma_max=a.tr_sigma_max, lm_dim=0)
    return p, a, poses, kw


def _sample(monkeypatch, name, model, args, poses, steps, mutate=None, **kw):
    """sampling(cuda_graph=True) of one batch with every launch replayed; returns (CapturedReplay, final coordinates)."""
    from diffdock_b200.diffusion_utils import get_t_schedule, t_to_sigma
    from diffdock_b200.sampling import sampling
    rec = Recorder(monkeypatch)
    rec.call_mutation.update(mutate or {})
    cap = CapturedReplay(monkeypatch, rec, name, model)
    sched = get_t_schedule('expbeta', steps)
    rec.start()
    out, _ = sampling([q.clone() for q in poses], model, steps, sched, sched, sched, DEV, partial(t_to_sigma, args=args),
                      args, batch_size=len(poses), no_final_step_noise=True, cuda_graph=True, **kw)
    rec.stop()
    return cap, torch.stack([d['ligand'].pos for d in out]).cpu()


@pytest.mark.parametrize('mode', list(SMALL))
def test_captured_sampler_20_steps(built_lib, monkeypatch, mode):
    """CGModel ns 16 / nv 4, 3 poses, a 20-step expbeta schedule: torch noise drawn inside the graph, Philox noise with
    the per-step crop at 20 A, and no noise with the crop at 4 A (the last steps keep 10 of 900 residues) and at 1 A (late
    steps keep none: edge groups whose device live count is 0)."""
    p, a, poses, kw = _small_workload(mode)
    torch.manual_seed(0)
    name = f"cg16 {mode}"
    cap, _ = _sample(monkeypatch, name, p, a, poses, 20, **kw)
    assert not cap.failures, cap.failures[:8]
    cap.summary(20, 'pose_update_dev', crop=a.crop_beyond is not None)
    if mode == 'torch_noise':
        assert len(cap.noise) == 20
        bad = noise_failures(cap.noise)
        assert not bad, bad
    if a.crop_beyond is not None:
        assert cap.kept[19][0] < cap.kept[19][1], cap.kept        # the late crop drops residues
    if mode == 'no_random_crop1':
        assert ZERO_LIVE[(name, 'fused.fused_conv')] > 0, "no convolution launch with an empty live group"


def test_captured_sampler_diffdock_l_shape(built_lib, monkeypatch):
    """CGModel at DiffDock-L shape (ns 48, nv 10, 6 layers), 2 poses of a 400-residue / 40-atom complex, 20 steps with
    Philox noise and the per-step crop at 20 A: the 48/10 tile kinds under capture."""
    from diffdock_b200.synthetic import default_model_args, make_pose_list
    from tests.parity_helpers import make_model_pair
    a = default_model_args(ns=48, nv=10, sh_lmax=2, num_conv_layers=6, crop_beyond=20.0)
    _, p = make_model_pair(a, seed=3)
    poses = make_pose_list(2, n_res=400, n_atoms=40, seed=4, tr_sigma_max=a.tr_sigma_max)
    cap, _ = _sample(monkeypatch, "cg_l 400 res", p, a, poses, 20, rng='philox', seed=5)
    assert not cap.failures, cap.failures[:8]
    cap.summary(20, 'pose_update_dev', crop=True)


def _packed_model(which):
    from tests import test_packed_aa_gpu as aa, test_packed_gpu as pk
    if which == 'aa':
        model, args = aa._aa_model(False)
        return model, args, aa._complexes()
    model, args = pk._old_model(False) if which == 'old' else pk._cg_model(False)
    if which == 'cg_crop':
        args.crop_beyond = 20.0
    return model, args, pk._complexes(shared=True)


def _sample_packed(monkeypatch, name, model, args, cx, steps=6, mutate=None, conf_model=None, **kw):
    from diffdock_b200.diffusion_utils import get_t_schedule, t_to_sigma
    from diffdock_b200.sampling import sample_packed
    rec = Recorder(monkeypatch, conf_model=conf_model)
    rec.call_mutation.update(mutate or {})
    cap = CapturedReplay(monkeypatch, rec, name, model)
    sched = get_t_schedule('expbeta', steps)
    if conf_model is not None:
        kw['confidence_model'] = conf_model
    rec.start()
    out = sample_packed([[d.clone() for d in p] for p in cx], model, steps, sched, sched, sched, DEV,
                        partial(t_to_sigma, args=args), args, seed=11, complex_ids=[5, 9, 2, 7][:len(cx)],
                        no_final_step_noise=True, cuda_graph=True, **kw)
    rec.stop()
    return cap, rec, out


@pytest.mark.parametrize('which', ['cg_crop', 'old', 'aa'])
def test_captured_sample_packed(built_lib, monkeypatch, which):
    """sample_packed of three complexes (two sharing a receptor) in one captured batch, 6 steps: the packed pose update,
    with the per-step crop (CGModel), the swapped launches of the v1.0 score model (CGOldModel), and the layer-0 receptor
    messages computed once per distinct receptor (AAModel)."""
    model, args, cx = _packed_model(which)
    name = f"packed {which}"
    cap, _, _ = _sample_packed(monkeypatch, name, model, args, cx)
    assert not cap.failures, cap.failures[:8]
    cap.summary(6, 'pose_update_packed', crop=which == 'cg_crop')
    if which == 'old':
        assert all(c['fused_conv_swap'] >= 1 for c in cap.per_step.values()), cap.per_step
    if which == 'aa':
        assert 'shared_static' in cap.batches[0]['receptor', 'receptor']._b200aa


@pytest.mark.parametrize('ranker', ['CGOldModel', 'AAOldModel'])
def test_packed_ranking(built_lib, monkeypatch, ranker):
    """sample_packed with a v1.0 ranker: the captured score steps, then one eager confidence forward over the whole
    ranking pack, whose confidence head reads a ``lig_ptr`` spanning every complex."""
    from argparse import Namespace
    from tests.test_packed_rank_gpu import _complexes as rank_complexes, _ranker
    conf, cargs = _ranker(ranker, False)
    if ranker == 'AAOldModel':
        model, args, cx = _packed_model('aa')
    else:
        from tests.parity_helpers import make_model_pair
        args = _small_args(num_conv_layers=3)
        model = make_model_pair(args, seed=3, lm=False)[1]
        cx = rank_complexes(False)[:4]            # receptor A for complexes 0, 2 and 3, B for 1
    assert isinstance(cargs, Namespace) and cargs.crop_beyond is None
    name = f"ranked {ranker}"
    cap, rec, out = _sample_packed(monkeypatch, name, model, args, cx, conf_model=conf,
                                   confidence_data=[[d.clone() for d in p] for p in cx], confidence_model_args=cargs)
    assert not cap.failures, cap.failures[:8]
    cap.summary(6, 'pose_update_packed')
    heads = [r for r in rec.records if r[0] == 'ops.confidence_head']
    assert len(heads) == 1, len(heads)                                      # one ranking pack
    assert heads[0][1]['lig_ptr'].shape[0] - 1 == sum(len(p) for p in cx)   # its lig_ptr spans every complex's poses
    res = replay(rec, f"{name} ranking", table=KIND_TABLE)
    bad = {k: v[3][:5] for k, v in res.items() if v[3]}
    assert not bad, bad
    assert res['confidence_head'][2] == 1 and sum(v[2] for k, v in res.items() if k.startswith('fused_conv')) >= 3, sorted(res)
    print(f"  ranking: {sum(v[2] for v in res.values())} launches checked, confidence head max {res['confidence_head'][0]:.2e}")
    for _, c in out:
        assert torch.isfinite(c).all()


# ---------------------------------------------------------------------------------------------------------------------
# mutations the captured replay must catch
def test_mutation_crop_reads_row_0_at_every_step(built_lib, monkeypatch):
    """ddb200_crop_flags launched with step_dev NULL: the captured crop uses the first step's cut-off at every step.  The
    replay flags crop_flags at a later step; whether the captured-vs-eager 2e-3 comparison of the final coordinates
    notices is printed."""
    p, a, poses, kw = _small_workload('philox_crop20')
    cap, got = _sample(monkeypatch, "mutation crop step NULL", p, a, poses, 20,
                       mutate={'ddb200_crop_flags': lambda x: x[:6] + (None,) + x[7:]}, **kw)
    steps = cap.flagged('ops.crop_flags')
    assert steps and steps[0] > 0, cap.failures[:8]
    assert all(w == 'ops.crop_flags' for _, w, _ in cap.failures), cap.failures[:8]
    monkeypatch.undo()
    from diffdock_b200.diffusion_utils import get_t_schedule, t_to_sigma
    from diffdock_b200.sampling import sampling
    sched = get_t_schedule('expbeta', 20)
    eager, _ = sampling([q.clone() for q in poses], p, 20, sched, sched, sched, DEV, partial(t_to_sigma, args=a), a,
                        batch_size=len(poses), no_final_step_noise=True, cuda_graph=False, **kw)
    d = float((torch.stack([q['ligand'].pos for q in eager]).cpu() - got).abs().max())
    print(f"\n[captured replay] crop step NULL: replay flags crop_flags at steps {steps}; captured vs eager final "
          f"coordinates differ by {d:.2e}, which the 2e-3 comparison {'notices' if d >= 2e-3 else 'misses'}")


def test_mutation_packed_pose_update_reads_row_0(built_lib, monkeypatch):
    """ddb200_pose_update_packed launched with step_dev NULL: SDE coefficients and noise of step 0 at every replay."""
    model, args, cx = _packed_model('cg_crop')
    cap, _, _ = _sample_packed(monkeypatch, "mutation pose step NULL", model, args, cx,
                               mutate={'ddb200_pose_update_packed': lambda x: x[:14] + (None,) + x[15:]})
    assert cap.flagged('pose_update_packed') == list(range(1, 6)), cap.failures[:8]


def test_mutation_noise_drawn_once_before_the_capture(built_lib, monkeypatch):
    """torch.normal returning, inside the capture, the tensor of the same shape drawn by the eager warm-up step: every
    replay reuses the same noise.  Each launch is still consistent with its inputs; the noise invariant fails."""
    p, a, poses, kw = _small_workload('torch_noise')
    real, drawn = torch.normal, {}

    def normal(*args, **kwargs):
        if torch.cuda.is_current_stream_capturing():
            return drawn[tuple(kwargs['size'])]
        z = real(*args, **kwargs)
        drawn[tuple(kwargs['size'])] = z.clone()
        return z
    monkeypatch.setattr(torch, 'normal', normal)
    cap, _ = _sample(monkeypatch, "mutation noise fixed", p, a, poses, 20, **kw)
    assert not cap.failures, cap.failures[:8]
    bad = noise_failures(cap.noise)
    assert any('identical' in b for b in bad), bad
