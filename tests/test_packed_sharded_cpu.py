"""CPU, gloo, 2 and 3 ranks: the host side of ``distributed.sample_packed_sharded`` with ``sampling.sample_packed`` replaced
in the workers by a deterministic stand-in - each rank's share, in ascending order, with the global indices as complex ids;
``load`` only for owned complexes; every complex's coordinates and confidences (None, [P], [P, 1], [P, 4]) gathered in
complex order on every rank, ranks that own nothing included; a failure on one rank, or ranks that disagree on confidence
graphs, raised on every rank.  Each process group meets through a file and has a short timeout, and the children are
terminated when a test runs past its deadline, so a regression fails instead of hanging."""
import itertools
import time
from datetime import timedelta

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

SIZES = [(3, 5), (4, 7), (2, 9), (5, 4), (3, 6)]        # (poses, ligand atoms) per complex
RESIDUES = [30, 10, 50, 20, 40]
SCHED = [1.0, 0.5]
_STORES = itertools.count()


def _costs(n):
    return [p * a * r for (p, a), r in zip(SIZES[:n], RESIDUES)]


def _poses(k):
    from diffdock_b200.hetero import HeteroGraph
    P, a = SIZES[k]
    out = []
    for _ in range(P):
        g = HeteroGraph()
        g['ligand'].pos = torch.zeros(a, 3)
        out.append(g)
    return out


def _final_pos(k):
    """What the stand-in leaves as complex k's final coordinates: a value of the complex and pose only."""
    P, a = SIZES[k]
    return torch.arange(P * a * 3, dtype=torch.float32).reshape(P, a, 3) + 1000 * k


def _confidence(k, kind):
    base = torch.arange(SIZES[k][0], dtype=torch.float32) + 100 * k
    return {None: None, 'P': base, 'P1': base[:, None], 'P4': base[:, None] + torch.arange(4) / 8}[kind]


def _stub(calls, fail=False):
    """Stands in for ``sampling.sample_packed``; the ranker keyword carries the confidence shape to return."""
    def sample_packed(complexes, model, inference_steps, tr_schedule, rot_schedule, tor_schedule, device, t_to_sigma,
                      model_args, *, seed, complex_ids, confidence_data, confidence_model, **kw):
        calls.append(dict(ids=list(complex_ids), n=len(complexes), graphs=confidence_data, seed=seed, kw=kw,
                          args=(model, inference_steps, device)))
        if fail:
            raise ValueError("stand-in refusal")
        for k, poses in zip(complex_ids, complexes):
            for i, d in enumerate(poses):
                d['ligand'].pos = _final_pos(k)[i]
        return [(poses, _confidence(k, confidence_model)) for k, poses in zip(complex_ids, complexes)]
    return sample_packed


def _call(n, kind, load, group_kw=None):
    from diffdock_b200.distributed import sample_packed_sharded
    return sample_packed_sharded(n, _costs(n), SIZES[:n], load, 'model', 2, SCHED, SCHED, SCHED, 'cuda:0', None, None,
                                 seed=5, confidence_model=kind, max_pairs=77, **(group_kw or {}))


def _check(out, n, kind):
    assert len(out) == n
    for k, (pos, conf) in enumerate(out):
        assert torch.equal(pos, _final_pos(k)), k
        want = _confidence(k, kind)
        if want is None:
            assert conf is None
        else:
            assert conf.shape == want.shape and torch.equal(conf, want), (k, conf, want)


def _init(rank, world, store):
    dist.init_process_group('gloo', init_method=f'file://{store}', rank=rank, world_size=world,
                            timeout=timedelta(seconds=30))


def _run(fn, world, tmp_path, *args, deadline=150):
    """Runs ``fn(rank, world, store, *args)`` in ``world`` spawned processes; a child's exception fails the test, and no
    child outlives it."""
    store = tmp_path / f'store{next(_STORES)}'
    ctx = mp.start_processes(fn, args=(world, str(store)) + args, nprocs=world, join=False, start_method='spawn')
    t0 = time.monotonic()
    try:
        while not ctx.join(timeout=1):
            if time.monotonic() - t0 > deadline:
                raise TimeoutError(f"workers still running after {deadline} s")
    finally:
        for p in ctx.processes:
            if p.is_alive():
                p.terminate()
            p.join()


# ---------------------------------------------------------------------------------------------------------------------
def _worker_gather(rank, world, store, n, kind, graphs):
    _init(rank, world, store)
    try:
        import diffdock_b200.sampling as S
        from diffdock_b200.distributed import assign_balanced
        calls, loads = [], []
        S.sample_packed = _stub(calls)

        def load(k):
            loads.append(k)
            return _poses(k), ([f'confidence graph {k}.{i}' for i in range(SIZES[k][0])] if graphs else None)
        out = _call(n, kind, load)
        mine = assign_balanced(_costs(n), world)[rank]
        assert loads == mine == sorted(mine)
        if mine:
            assert len(calls) == 1
            c = calls[0]
            assert c['ids'] == mine and c['n'] == len(mine) and c['seed'] == 5 and c['kw'] == {'max_pairs': 77}
            assert c['args'] == ('model', 2, 'cuda:0')
            assert c['graphs'] == ([[f'confidence graph {k}.{i}' for i in range(SIZES[k][0])] for k in mine]
                                   if graphs else None)
        else:
            assert calls == []
        _check(out, n, kind)
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize('world,n,kind,graphs', [
    (2, 5, None, False), (2, 5, 'P', True), (3, 5, 'P1', True), (3, 5, 'P4', False),
    (3, 2, 'P4', True),                                  # rank 2 owns nothing
    (2, 1, 'P', False),                                  # rank 1 owns nothing
])
def test_every_rank_gets_every_complex_in_order(tmp_path, world, n, kind, graphs):
    from diffdock_b200.distributed import assign_balanced
    if n < world:
        assert [] in assign_balanced(_costs(n), world)
    _run(_worker_gather, world, tmp_path, n, kind, graphs)


def _worker_failure(rank, world, store, bad, where):
    _init(rank, world, store)
    try:
        import diffdock_b200.sampling as S
        calls = []
        S.sample_packed = _stub(calls, fail=rank == bad and where == 'sample_packed')

        def load(k):
            if rank == bad and where == 'load':
                raise KeyError(f"no complex {k} here")
            return _poses(k), None
        with pytest.raises(RuntimeError) as e:
            _call(5, 'P', load)
        msg = str(e.value)
        assert f"rank(s) [{bad}] failed" in msg, msg
        if rank == bad:
            assert ('stand-in refusal' if where == 'sample_packed' else 'no complex') in msg
            assert e.value.__cause__ is not None
        else:
            assert 'refusal' not in msg and e.value.__cause__ is None
        dist.barrier()                                   # every rank is still in step: nobody waits in the gather
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize('world,bad,where', [(2, 1, 'sample_packed'), (3, 0, 'load')])
def test_a_failure_on_one_rank_is_raised_on_every_rank(tmp_path, world, bad, where):
    _run(_worker_failure, world, tmp_path, bad, where)


def _worker_disagree(rank, world, store):
    _init(rank, world, store)
    try:
        import diffdock_b200.sampling as S
        S.sample_packed = _stub([])
        with pytest.raises(RuntimeError, match='disagree'):
            _call(5, 'P', lambda k: (_poses(k), ['graph'] * SIZES[k][0] if rank == 0 else None))
    finally:
        dist.destroy_process_group()


def test_ranks_that_disagree_on_confidence_graphs_raise_on_every_rank(tmp_path):
    """One sample_packed over all these complexes would refuse the mix of complexes with and without confidence graphs."""
    _run(_worker_disagree, 2, tmp_path)


# ---------------------------------------------------------------------------------------------------------------------
def test_single_process_is_one_sample_packed_call(monkeypatch):
    import diffdock_b200.sampling as S
    assert not dist.is_initialized()
    calls, loads = [], []
    monkeypatch.setattr(S, 'sample_packed', _stub(calls))
    out = _call(5, 'P1', lambda k: (loads.append(k), (_poses(k), None))[1])
    assert loads == [0, 1, 2, 3, 4] and len(calls) == 1 and calls[0]['ids'] == [0, 1, 2, 3, 4]
    _check(out, 5, 'P1')
    with pytest.raises(ValueError, match='every complex or for none'):
        _call(5, 'P', lambda k: (_poses(k), None if k else ['graph'] * SIZES[k][0]))
    with pytest.raises(ValueError, match='shapes'):
        _call(5, 'P', lambda k: (_poses(k)[1:], None))
