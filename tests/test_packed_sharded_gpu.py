"""GPU: ``distributed.sample_packed_sharded`` - the result of every complex does not depend on the number of ranks.

On one GPU the ranks of worlds 1, 2 and 3 are emulated by running each rank's share (``assign_balanced``) through the code
a rank runs (``distributed._sample_owned``: one ``sample_packed`` with the global complex ids), for a ``CGModel`` with
per-step cropping and a ``CGOldModel`` ranker, an ``AAModel`` with an ``AAOldModel`` ranker, and a ranker without
confidence graphs; every complex must match one ``sample_packed`` over all complexes, and the comparison must fail when
the ranks key their noise by local indices.  Then two real processes (gloo, both on cuda:0, gather on the CPU) return the
single-process result on both ranks, and a refusal met only by the rank that owns the complex is raised on both ranks."""
from functools import partial
from types import SimpleNamespace

import numpy as np
import pytest
import torch
import torch.distributed as dist

from tests.test_packed_sharded_cpu import _init, _run

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
STEPS = 6
SEED = 11
CG_SIZES = [(60, 12), (70, 20), (60, 9), (50, 15), (80, 11)]        # (residues, ligand atoms)
AA_SIZES = [(40, 12), (48, 20), (40, 9), (36, 15), (44, 11)]
N_POSES = [3, 2, 4, 3, 2]


def _setup(case):
    """(score model, its args, ``sample_packed`` keywords, load, costs, shapes) of one seeded workload of five complexes."""
    from diffdock_b200.synthetic import make_pose_list
    if case == 'aa':
        from tests.test_packed_aa_gpu import _aa_model
        from tests.test_packed_rank_gpu import _ranker
        model, args = _aa_model(False)
        conf, cargs = _ranker('AAOldModel', False)
        sizes = AA_SIZES
        mk = lambda k: make_pose_list(N_POSES[k], n_res=sizes[k][0], n_atoms=sizes[k][1], seed=5 + k, tr_sigma_max=5.0,
                                      lm_dim=0, all_atoms=True)
    else:
        from diffdock_b200.diffusion_utils import get_timestep_embedding
        from diffdock_b200.old_cg_model import CGOldModel
        from diffdock_b200.synthetic import default_model_args
        from tests.parity_helpers import make_model_pair
        args = default_model_args(ns=16, nv=4, sh_lmax=2, num_conv_layers=3, distance_embed_dim=16,
                                  cross_distance_embed_dim=16, sigma_embed_dim=16,
                                  crop_beyond=20.0 if case == 'cg_crop' else None)
        _, model = make_model_pair(args, seed=3)
        torch.manual_seed(4)
        conf = CGOldModel(None, torch.device(DEV), get_timestep_embedding('sinusoidal', 16, args.embedding_scale), ns=16,
                          nv=4, num_conv_layers=2, sigma_embed_dim=16, distance_embed_dim=16, cross_distance_embed_dim=16,
                          confidence_mode=True, use_old_atom_encoder=True, lm_embedding_type='esm',
                          lm_embedding_dim=1280, dynamic_max_cross=True, cross_max_distance=80.0).eval().to(DEV)
        cargs = SimpleNamespace(crop_beyond=None, all_atoms=False)
        sizes = CG_SIZES
        mk = lambda k: make_pose_list(N_POSES[k], n_res=sizes[k][0], n_atoms=sizes[k][1], seed=5 + k, tr_sigma_max=5.0)
    graphs = case != 'cg_no_graphs'

    def load(k):
        poses = mk(k)
        if k == 1:                                       # a ligand without rotatable bonds, as in the packed tests
            for d in poses:
                d['ligand'].edge_mask = torch.zeros_like(d['ligand'].edge_mask)
                d['ligand'].mask_rotate = [np.zeros((0, d['ligand'].num_nodes), dtype=bool)]
        return poses, ([d.clone() for d in poses] if graphs else None)
    costs = [n * r * a for n, (r, a) in zip(N_POSES, sizes)]
    shapes = [(n, a) for n, (_, a) in zip(N_POSES, sizes)]
    kw = dict(confidence_model=conf, confidence_model_args=cargs, no_final_step_noise=True)
    return model, args, kw, load, costs, shapes


def _sample_args(model, args):
    from diffdock_b200.diffusion_utils import get_t_schedule, t_to_sigma
    sched = get_t_schedule('expbeta', STEPS)
    return (model, STEPS, sched, sched, sched, DEV, partial(t_to_sigma, args=args), args)


def _one_call(model, args, kw, load, n):
    """One ``sample_packed`` over all complexes (complex ids 0 .. n-1)."""
    from diffdock_b200.sampling import sample_packed
    loaded = [load(k) for k in range(n)]
    graphs = [c for _, c in loaded]
    out = sample_packed([p for p, _ in loaded], *_sample_args(model, args), seed=SEED,
                        confidence_data=graphs if graphs[0] is not None else None, **kw)
    return [(torch.stack([d['ligand'].pos for d in dl]), c) for dl, c in out]


def _emulated(model, args, kw, load, costs, shapes, world):
    """Every complex's result when each rank of ``world`` runs its own share."""
    from diffdock_b200.distributed import _sample_owned, assign_balanced
    got = {}
    for share in assign_balanced(costs, world):
        got.update(zip(share, _sample_owned(share, shapes, load, _sample_args(model, args), SEED, kw)[0]))
    return [got[k] for k in range(len(costs))]


def _close(got, ref, tol):
    got, ref = got.float().cpu(), ref.float().cpu()
    return got.shape == ref.shape and float((got - ref).abs().max()) <= tol * max(1.0, float(ref.abs().max()))


def _compare(got, ref, conf_tol):
    """Largest coordinate difference; asserts the confidences agree within ``conf_tol`` (relative, as in
    test_packed_rank_gpu)."""
    d = 0.0
    for (p, c), (q, e) in zip(got, ref):
        assert p.shape == q.shape and torch.isfinite(p).all()
        d = max(d, float((p.cpu() - q.cpu()).abs().max()))
        assert c.shape == e.shape and torch.isfinite(c).all() and _close(c, e, conf_tol), (c, e)
    return d


CASES = {'cg_crop': 1e-4, 'aa': 2.5e-5, 'cg_no_graphs': 1e-4}     # confidence tolerance per workload


@pytest.mark.parametrize('case', list(CASES))
def test_result_independent_of_world_size(built_lib, case):
    from diffdock_b200.distributed import assign_balanced
    model, args, kw, load, costs, shapes = _setup(case)
    assert model.sync_free_capable()
    ref = _one_call(model, args, kw, load, len(costs))
    for world in (1, 2, 3):
        parts = assign_balanced(costs, world)
        assert all(parts)
        assert _compare(_emulated(model, args, kw, load, costs, shapes, world), ref, CASES[case]) < 2e-3, world


def test_mutation_local_complex_ids_are_caught(built_lib, monkeypatch):
    import diffdock_b200.sampling as S
    model, args, kw, load, costs, shapes = _setup('cg_crop')
    ref = _one_call(model, args, kw, load, len(costs))
    real = S.sample_packed
    monkeypatch.setattr(S, 'sample_packed', lambda cx, *a, complex_ids, **k: real(cx, *a, complex_ids=range(len(cx)), **k))
    got = _emulated(model, args, kw, load, costs, shapes, 3)
    assert max(float((p - q).abs().max()) for (p, _), (q, _) in zip(got, ref)) > 2e-3


# ---------------------------------------------------------------------------------------------------------------------
# two processes on one GPU
def _worker_two(rank, world, store, out_path):
    torch.cuda.set_device(0)
    _init(rank, world, store)
    try:
        from diffdock_b200.distributed import sample_packed_sharded
        model, args, kw, load, costs, shapes = _setup('cg_crop')
        out = sample_packed_sharded(len(costs), costs, shapes, load, *_sample_args(model, args), seed=SEED, **kw)
        assert all(p.device.type == 'cpu' and c.device.type == 'cpu' for p, c in out)     # gloo gathers on the CPU
        torch.save(out, f'{out_path}.{rank}')
    finally:
        dist.destroy_process_group()


def test_two_processes_return_the_single_process_result(built_lib, tmp_path):
    from diffdock_b200.distributed import sample_packed_sharded
    model, args, kw, load, costs, shapes = _setup('cg_crop')
    single = sample_packed_sharded(len(costs), costs, shapes, load, *_sample_args(model, args), seed=SEED, **kw)
    _run(_worker_two, 2, tmp_path, str(tmp_path / 'out'), deadline=600)
    for rank in (0, 1):
        got = torch.load(tmp_path / f'out.{rank}')
        assert len(got) == len(costs)
        assert _compare(got, single, CASES['cg_crop']) < 2e-3, rank


def _worker_refusal(rank, world, store):
    torch.cuda.set_device(0)
    _init(rank, world, store)
    try:
        from diffdock_b200.distributed import assign_balanced, sample_packed_sharded
        from tests.test_packed_aa_gpu import _aa_model
        from diffdock_b200.synthetic import make_pose_list
        model, args = _aa_model(False)
        args.crop_beyond = 20.0                          # sample_packed refuses all-atom receptors cropped per step
        assert assign_balanced([1.0], world) == [[0], []]
        load = lambda k: (make_pose_list(2, n_res=40, n_atoms=12, seed=5, tr_sigma_max=5.0, lm_dim=0, all_atoms=True), None)
        with pytest.raises(RuntimeError, match=r'rank\(s\) \[0\] failed') as e:
            sample_packed_sharded(1, [1.0], [(2, 12)], load, *_sample_args(model, args), seed=SEED)
        assert isinstance(e.value.__cause__, NotImplementedError) == (rank == 0)
    finally:
        dist.destroy_process_group()


def test_refusal_on_the_owning_rank_is_raised_on_both(built_lib, tmp_path):
    _run(_worker_refusal, 2, tmp_path, deadline=600)
