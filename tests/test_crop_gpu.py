"""GPU: per-step receptor cropping (crop_beyond, utils/sampling.py:104-109) inside the sync-free forward and the captured
sampler step.  The device crop flags are compared bit for bit with the oracle's expression, the edge selection exactly with
boolean-mask indexing, and the cropped forward / sampler with the oracle run on the reference's cropped, re-collated batch."""
import copy
from functools import partial

import numpy as np
import pytest
import torch

from tests.parity_helpers import make_model_pair, rel_err

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def _args(**over):
    from diffdock_b200.synthetic import default_model_args
    kw = dict(ns=16, nv=4, sh_lmax=2, num_conv_layers=3, distance_embed_dim=16, cross_distance_embed_dim=16, sigma_embed_dim=16)
    kw.update(over)
    return default_model_args(**kw)


def _oracle_keep(lig, rec, cutoff):
    """``keep`` of oracle/diffusion.py:crop_beyond for ONE complex, read back from which residues survive the crop."""
    from diffdock_b200.hetero import HeteroGraph
    from oracle.diffusion import crop_beyond
    g = HeteroGraph()
    g['ligand'].pos = lig
    g['receptor'].pos, g['receptor'].x = rec, torch.arange(rec.shape[0]).unsqueeze(1)
    g['receptor', 'receptor'].edge_index = torch.zeros((2, 0), dtype=torch.long)
    crop_beyond(g, cutoff)
    keep = torch.zeros(rec.shape[0], dtype=torch.bool)
    keep[g['receptor'].x[:, 0]] = True
    return keep


def _boundary_residues(lig, c2):
    """Residue positions whose smallest squared distance to ``lig`` (float32, as torch computes it) is one ulp below, equal
    to and one ulp above ``c2``: offsets from the ligand atom of largest x along +x (every other atom is then farther)."""
    f = np.float32
    j = int(torch.argmax(lig[:, 0]))
    lx, ly, lz = (f(v) for v in lig[j].tolist())
    want = {np.nextafter(f(c2), f(0)): None, f(c2): None, np.nextafter(f(c2), f(np.inf)): None}
    for k in range(64):
        ry = f(ly + f(k) * f(2 ** -9))
        dy = f(ly - ry)
        base = f(lx + f(np.sqrt(max(float(c2) - float(dy) * float(dy), 0.0))))
        rx = base
        for _ in range(16):
            rx = np.nextafter(rx, f(-np.inf))
        for _ in range(33):
            dx = f(lx - rx)
            d2 = f(f(f(dx * dx) + f(dy * dy)) + f(0))
            if d2 in want and want[d2] is None:
                want[d2] = (rx, ry, lz)
            rx = np.nextafter(rx, f(np.inf))
        if all(v is not None for v in want.values()):
            break
    assert all(v is not None for v in want.values()), "no float32 positions at the cut-off found"
    return torch.tensor([list(map(float, v)) for v in want.values()], dtype=torch.float32)


def _cut2_table(args, n=20):
    from diffdock_b200.diffusion_utils import get_t_schedule, t_to_sigma
    from diffdock_b200.sampling import crop_cutoff2
    sched = get_t_schedule('expbeta', n)
    t2s = partial(t_to_sigma, args=args)
    cut = [float(t2s(t, t, t)[0]) * 3 + 20.0 for t in sched]
    return cut, [crop_cutoff2(t2s, t, t, t, 20.0) for t in sched]


def test_crop_flags_match_oracle_bit_for_bit(built_lib):
    from diffdock_b200 import ops
    args = _args()
    cuts, rows = _cut2_table(args)
    table = torch.tensor(rows, dtype=torch.float32, device=DEV)
    gen = torch.Generator().manual_seed(0)
    # several complexes of different sizes (one without residues), then four copies of one receptor with their own ligand
    sizes = [(12, 50), (40, 300), (1, 7), (25, 0), (33, 129)]
    shared = torch.randn(90, 3, generator=gen) * 25.0
    sizes += [(17, 90)] * 4
    n_kept = n_all = 0
    for step, cut in enumerate(cuts):
        ligs, recs = [], []
        for k, (n_lig, n_rec) in enumerate(sizes):
            lig = torch.randn(n_lig, 3, generator=gen) * 4.0 + torch.randn(3, generator=gen) * 10.0
            rec = shared.clone() if n_rec == 90 else torch.randn(n_rec, 3, generator=gen) * (8.0 + n_rec / 10.0)
            if n_rec and n_lig > 1:     # one ulp inside, on and one ulp outside the cut-off
                rec = torch.cat([rec, _boundary_residues(lig, np.float32(rows[step]))])
            ligs.append(lig)
            recs.append(rec)
        ref = torch.cat([_oracle_keep(l, r, cut) if r.shape[0] else torch.zeros(0, dtype=torch.bool)
                         for l, r in zip(ligs, recs)])
        lig_ptr = torch.tensor([0] + np.cumsum([l.shape[0] for l in ligs]).tolist(), dtype=torch.int32, device=DEV)
        rec_batch = torch.cat([torch.full((r.shape[0],), i, dtype=torch.int32) for i, r in enumerate(recs)]).to(DEV)
        rec_all = torch.cat(recs).to(DEV)
        step_dev = torch.tensor([step], dtype=torch.int32, device=DEV)
        keep, masked = ops.crop_flags(torch.cat(ligs).to(DEV), lig_ptr, rec_all, rec_batch, table, step_dev)
        keep, masked = keep.cpu(), masked.cpu()
        assert torch.equal(keep, ref), step
        assert torch.equal(masked[keep], rec_all.cpu()[keep]) and bool(torch.isposinf(masked[~keep]).all())
        # the boundary residues: inside kept, on and outside dropped (unless another atom is nearer, which cannot happen)
        tail = [sum(r.shape[0] for r in recs[:i + 1]) for i, (n_lig, n_rec) in enumerate(sizes) if n_rec and n_lig > 1]
        for end in tail:
            assert keep[end - 3:end].tolist() == [True, False, False]
        n_kept, n_all = n_kept + int(ref.sum()), n_all + ref.shape[0]
    assert 0 < n_kept < n_all


@pytest.mark.parametrize("n_edges,p", [(0, 0.5), (1, 1.0), (255, 0.5), (256, 0.5), (257, 0.7), (5000, 1.0), (5000, 0.0),
                                       (100003, 0.6)])
def test_crop_edge_selection_matches_boolean_mask(built_lib, n_edges, p):
    from diffdock_b200 import ops
    gen = torch.Generator().manual_seed(n_edges)
    n_rec = 700
    tgt = torch.sort(torch.randint(0, n_rec, (n_edges,), generator=gen)).values
    src = torch.randint(0, n_rec, (n_edges,), generator=gen)
    gid = torch.randint(0, 9, (n_edges,), generator=gen)
    keep = torch.rand(n_rec, generator=gen) < p
    ok = keep[tgt] & keep[src]
    i32 = lambda t: t.to(torch.int32).to(DEV).contiguous()
    out_t, out_s, perm, out_g, n_dev = ops.crop_select_edges(i32(tgt), i32(src), keep.to(DEV), i32(gid), offset=11)
    n = int(n_dev.item())
    assert n == int(ok.sum())
    assert torch.equal(perm[:n].cpu().long(), torch.nonzero(ok).reshape(-1))
    assert torch.equal(out_t[:n].cpu().long(), tgt[ok] + 11) and torch.equal(out_s[:n].cpu().long(), src[ok] + 11)
    assert torch.equal(out_g[:n].cpu().long(), gid[ok])


def _model_cases():
    return [('lmax2', {}), ('lmax1', {'sh_lmax': 1}), ('prot_emb', {'num_prot_emb_layers': 1}),
            ('cfg_l2', dict(ns=48, nv=10, num_conv_layers=6, distance_embed_dim=64, cross_distance_embed_dim=64,
                            sigma_embed_dim=64))]


def _cropped_pair(p, o, args, poses, t, crop_beyond):
    """(product scores of the sync-free cropped forward on a shared-receptor batch, oracle scores on the reference's cropped
    re-collated batch, residues kept, residues in all)."""
    from diffdock_b200.diffusion_utils import set_time, t_to_sigma
    from diffdock_b200.hetero import collate, collate_shared_receptor
    from diffdock_b200.sampling import crop_cutoff2
    from oracle.diffusion import crop_beyond as o_crop, set_time as o_set_time, t_to_sigma as o_t2s
    B = len(poses)
    g = collate_shared_receptor([q.clone() for q in poses], DEV)
    set_time(g, None, t, t, t, B, False, DEV)
    g._uniform_t = True
    table = torch.tensor([crop_cutoff2(partial(t_to_sigma, args=args), t, t, t, crop_beyond)], device=DEV)
    g._crop = (table, torch.zeros(1, dtype=torch.int32, device=DEV))
    got = p(g)
    torch.cuda.synchronize()
    cutoff = o_t2s(t, t, t, args)[0] * 3 + crop_beyond
    cropped = [o_crop(q, cutoff) for q in copy.deepcopy(poses)]
    kept = sum(q['receptor'].pos.shape[0] for q in cropped)
    g_cpu = collate(cropped)
    o_set_time(g_cpu, t, t, t, B, 'cpu')
    with torch.no_grad():
        ref = o(g_cpu)
    return got, ref, kept, sum(q['receptor'].pos.shape[0] for q in poses)


@pytest.mark.parametrize("name,over", _model_cases(), ids=[c[0] for c in _model_cases()])
def test_cropped_forward_matches_oracle_on_cropped_batch(built_lib, name, over):
    from diffdock_b200.synthetic import make_pose_list
    args = _args(**over)
    # the full-width model and poses of test_full_width_sync_free_vs_oracle (well conditioned against the oracle uncropped)
    model_seed, n_poses, n_res, n_atoms, pose_seed = (5, 2, 90, 15, 21) if name == 'cfg_l2' else (17, 3, 80, 12, 5)
    o, p = make_model_pair(args, seed=model_seed)
    assert p.sync_free_crop_capable()
    seen = set()
    for t, crop_beyond in ((1.0, 20.0), (0.5, 6.0), (0.2, 5.0)):
        poses = make_pose_list(n_poses, n_res=n_res, n_atoms=n_atoms, seed=pose_seed, tr_sigma_max=args.tr_sigma_max * t)
        got, ref, kept, total = _cropped_pair(p, o, args, poses, t, crop_beyond)
        seen.add('all' if kept == total else ('part' if kept else 'none'))
        for a, b in zip(got[:3], ref[:3]):
            assert a.shape == b.shape
            if b.numel():
                assert rel_err(a, b) < 1e-4, (t, crop_beyond, kept, total)
    assert {'all', 'part'} <= seen, seen


def _sample(p, args, poses, crop_beyond, steps=6, **kw):
    from diffdock_b200.diffusion_utils import get_t_schedule, t_to_sigma
    from diffdock_b200.sampling import sampling
    a = copy.copy(args)
    a.crop_beyond = crop_beyond
    sched = get_t_schedule('expbeta', steps)
    out, _ = sampling([q.clone() for q in poses], p, steps, sched, sched, sched, DEV, partial(t_to_sigma, args=a), a,
                      batch_size=len(poses), no_final_step_noise=True, **kw)
    torch.cuda.synchronize()
    return torch.stack([d['ligand'].pos for d in out]).cpu()


def _recording_graphed_steps(monkeypatch):
    from diffdock_b200 import sampling as smod
    made = []

    class Recorder(smod.GraphedSteps):
        def __init__(self, *a, **k):
            super().__init__(*a, **k)
            made.append(self)

    monkeypatch.setattr(smod, 'GraphedSteps', Recorder)
    return made


def test_graphed_crop_sampler_matches_eager_crop_sampler(built_lib, monkeypatch):
    from diffdock_b200.synthetic import make_pose_list
    # a small translation scale keeps every ligand within reach of some residue: the eager crop path cannot take a batch
    # whose crop keeps no residue at all
    args = _args(tr_sigma_max=5.0)
    _, p = make_model_pair(args, seed=9)
    poses = make_pose_list(4, n_res=120, n_atoms=12, seed=41, tr_sigma_max=args.tr_sigma_max)
    made = _recording_graphed_steps(monkeypatch)
    graphed = _sample(p, args, poses, 20.0, rng='philox', seed=123, cuda_graph=True)
    assert len(made) == 1 and made[0].crop is not None        # captured, with the per-step crop
    eager = _sample(p, args, poses, 20.0, rng='philox', seed=123, cuda_graph=False)
    assert len(made) == 1
    assert torch.isfinite(graphed).all()
    assert float((eager - graphed).abs().max()) < 2e-3      # 6 chained steps; scatter order differs run to run


@pytest.mark.parametrize("crop_beyond", [20.0, 4.0])
def test_graphed_crop_sampler_20_steps_vs_oracle(built_lib, monkeypatch, crop_beyond):
    from diffdock_b200.diffusion_utils import get_t_schedule
    from diffdock_b200.synthetic import make_pose_list
    from oracle.diffusion import t_to_sigma as o_t2s
    from oracle.sampling import sampling as o_sampling
    args = _args()
    o, p = make_model_pair(args, seed=29)
    poses = make_pose_list(3, n_res=120, n_atoms=12, seed=61, tr_sigma_max=args.tr_sigma_max)
    made = _recording_graphed_steps(monkeypatch)
    got = _sample(p, args, poses, crop_beyond, steps=20, no_random=True, cuda_graph=True)
    assert len(made) == 1 and made[0].crop is not None
    a = copy.copy(args)
    a.crop_beyond = crop_beyond
    sched = get_t_schedule('expbeta', 20)
    ref, _ = o_sampling([q.clone() for q in poses], o, 20, sched, sched, sched, 'cpu', partial(o_t2s, args=a), a,
                        no_random=True, batch_size=3, no_final_step_noise=True)
    worst = max(rel_err(g_, r['ligand'].pos) for g_, r in zip(got, ref))
    assert worst < 1e-3, worst


def test_graphed_crop_step_is_sync_free(built_lib):
    from diffdock_b200.diffusion_utils import get_t_schedule, t_to_sigma
    from diffdock_b200.hetero import collate_shared_receptor
    from diffdock_b200.sampling import GraphedSteps, crop_cutoff2, step_coefficients
    from diffdock_b200.synthetic import make_pose_list
    args = _args(num_prot_emb_layers=1)
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
        steps.step.fill_(5)
        out = p(g)                    # the cropped forward launched op by op, at the last step's cut-off
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert int(done.item()) == 6 and torch.isfinite(steps.pos).all() and torch.isfinite(out[0]).all()


def test_one_full_size_cropped_pose_matches_oracle(built_lib):
    """The 1500-residue / 40-atom CFG-L2 complex at a late diffusion time: the crop drops most residues."""
    from diffdock_b200.synthetic import default_model_args, make_pose_list
    args = default_model_args()
    o, p = make_model_pair(args, seed=0)
    assert p.sync_free_crop_capable()
    t = 0.1
    poses = make_pose_list(1, n_res=1500, n_atoms=40, seed=100, tr_sigma_max=args.tr_sigma_max * t)
    torch.set_num_threads(min(torch.get_num_threads(), 32))
    got, ref, kept, total = _cropped_pair(p, o, args, poses, t, 20.0)
    assert 0 < kept < total, (kept, total)
    errs = [rel_err(a, b) for a, b in zip(got[:3], ref[:3]) if b.numel()]
    assert max(errs) < 1e-4, errs
