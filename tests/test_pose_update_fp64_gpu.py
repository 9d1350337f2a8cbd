"""GPU: the reverse-diffusion pose update (csrc/pose.cu: pose_update_kernel behind ddb200_pose_update and
ddb200_pose_update_dev) against a float64 reference built from the oracle's dtype-generic sampler functions
(oracle.diffusion.axis_angle_to_matrix, torsion_update_batch, kabsch_batch) applied to the float32 inputs upcast to float64,
with the perturbation a * score + c * z formed in float64 from the float32 coefficients.

The error of a pose is max |out - ref| over its coordinates divided by its extent (the largest distance of a reference atom
from the reference centroid, at least 1 A); coordinates are compared, not the Kabsch rotation, which is not unique when
singular values coincide.  Unwritten output is NaN-filled, so a pose the kernel skips or a row it writes twice shows up.

Cases: ligands of 4 to 150 atoms on both sides of the CTA's 128 threads, 1943 and 1944 atoms either side of the 48 KB
shared-memory opt-in (24 n + 2512 bytes), 8428 atoms (the largest accepted; 8429 returns DDB200_ESMEM); 0 to 30 rotatable
bonds of tree ligands and nested masks whose later bonds turn about axes the earlier ones moved;
1, 3 and 40 poses; rotation vectors of norm 0, 1e-7, 1e-6, pi - 1e-4 and 3 pi, torsion angles 0, +-pi and +-7, ligands 100 A
from the origin; injected noise, use_torsion = 0, the device coefficient table row of step_dev, in-place updates, in-kernel
Philox noise with its block / slot layout (translation block 0, rotation block 1, torsion r block 2 + r / 4, slot r % 4),
the Box-Muller transform of the raw Philox words in float64, planar, torsion-free and collinear ligands, argument errors.

Largest errors measured on an NVIDIA H100 80GB HBM3 (400 W power limit), and the tolerances (about 3x):
  4 to 150 atoms, every bond of a tree ligand      8.51e-6 (127 atoms, 108 bonds in sequence)     -> TOL_SIZES 2.6e-5
  1943, 1944 and 8428 atoms                        2.81e-7                                        -> TOL_LARGE 1e-6
  0 to 30 bonds, 1 to 40 poses, nested masks       4.66e-6 (30 bonds, 40 poses)                   -> TOL_BONDS 1.5e-5
  rotation norms, torsion angles, 100 A, no tor    5.44e-6                                        -> TOL_VALUES 1.6e-5
  device table, in place, Philox noise             6.02e-7 (Philox)                               -> TOL_DEV 2e-6
  planar, zero torsions, collinear                 2.57e-7 (planar)                               -> TOL_DEGEN 1e-6
  Box-Muller normals vs float64 (12,288 blocks)    6.70e-6 absolute                               -> BM_TOL 2e-5
The Box-Muller error is largest where u1 is close to 1 (sqrt(-2 ln u1) is steep there); the blocks are fixed, so the
bound holds for them."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
TOL_SIZES, TOL_LARGE, TOL_BONDS, TOL_VALUES, TOL_DEV, TOL_DEGEN = 2.6e-5, 1e-6, 1.5e-5, 1.6e-5, 2e-6, 1e-6
BM_TOL = 2e-5
EINVAL, ESMEM = -1, -3


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


class Lig:
    """One ligand: base coordinates [n, 3] and its rotatable bonds (u, v) with mask rows (v's side, u excluded)."""

    def __init__(self, pos, bonds, mask):
        self.pos = np.asarray(pos, dtype=np.float32)
        self.n = self.pos.shape[0]
        self.bonds = np.ascontiguousarray(bonds, dtype=np.int64).reshape(-1, 2)
        self.mask = np.ascontiguousarray(mask, dtype=bool).reshape(-1, self.n)
        for (u, v), m in zip(self.bonds, self.mask):
            assert not m[u] and m[v]

    def first(self, nb):
        assert nb <= len(self.bonds)
        return Lig(self.pos, self.bonds[:nb], self.mask[:nb])


def tree_ligand(n, seed):
    from diffdock_b200.synthetic import _ligand
    pos, ei, _, _, emask, mrot = _ligand(n, np.random.default_rng(seed))
    return Lig(pos, ei[:, emask].T, mrot)


def cloud_ligand(n, nb, seed):
    """A random cloud with nb bonds whose masks are random halves (v in, u out), for sizes where a tree is slow to build."""
    rng = np.random.default_rng(seed)
    pos = rng.normal(size=(n, 3)) * 1.5 * n ** (1 / 3)
    bonds, mask = [], []
    for _ in range(nb):
        u, v = rng.choice(n, 2, replace=False)
        m = rng.uniform(size=n) < 0.5
        m[u], m[v] = False, True
        bonds.append((u, v))
        mask.append(m)
    return Lig(pos, bonds, mask)


def nested_ligand():
    """A zigzag chain of 12 atoms; bond r turns atoms > k_r about (k_r, k_r + 1) with k_r = 8, 6, 4, 2: each bond's side
    contains the previous bond, so every rotation after the first turns about an axis that the earlier ones have moved."""
    pos = [[1.3 * i, 0.8 * (i % 2), 0.3 * ((i // 2) % 2)] for i in range(12)]
    ks = [8, 6, 4, 2]
    return Lig(pos, [(k, k + 1) for k in ks], [[i > k for i in range(12)] for k in ks])


def poses_of(lig, n_poses, seed, shift=(0.0, 0.0, 0.0)):
    """n_poses copies of the ligand, each randomly rotated and moved, float32 [n_poses * n, 3] on the device."""
    from oracle.diffusion import axis_angle_to_matrix
    g = torch.Generator().manual_seed(seed)
    R = axis_angle_to_matrix(torch.randn(n_poses, 3, generator=g, dtype=torch.float64))
    base = torch.from_numpy(lig.pos).double()
    P = base[None] @ R.transpose(1, 2) + torch.randn(n_poses, 1, 3, generator=g, dtype=torch.float64) * 3
    P = P + torch.tensor(shift, dtype=torch.float64)
    return P.reshape(-1, 3).float().cuda()


def scores(n_poses, nb, seed, tr=2.0, rot=1.0, tor=2.0):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s, k=1.0: (torch.randn(*s, generator=g) * k).cuda()
    return r(n_poses, 3, k=tr), r(n_poses, 3, k=rot), r(n_poses, nb, k=tor)


def device_bonds(lig):
    if len(lig.bonds) == 0:
        return None, None, None
    bu = torch.from_numpy(lig.bonds[:, 0]).int().cuda()
    bv = torch.from_numpy(lig.bonds[:, 1]).int().cuda()
    return bu, bv, torch.from_numpy(lig.mask.astype(np.uint8)).cuda()


def run(lig, pos, n_poses, tr, rot, tor, coef, tr_z=None, rot_z=None, tor_z=None, use_torsion=True, out=None,
        n_atoms=None, check=True):
    """ddb200_pose_update into a NaN-filled output; returns (rc, out)."""
    from diffdock_b200 import _lib
    bu, bv, mk = device_bonds(lig)
    if out is None:
        out = torch.full_like(pos, float('nan'))
    c6 = (C.c_float * 6)(*[float(v) for v in coef])
    rc = _lib.lib().ddb200_pose_update(_p(pos), n_poses, lig.n if n_atoms is None else n_atoms, len(lig.bonds), _p(bu),
                                       _p(bv), _p(mk), _p(tr), _p(rot), _p(tor), _p(tr_z), _p(rot_z), _p(tor_z),
                                       C.cast(c6, C.c_void_p), int(use_torsion), _p(out), _stream())
    torch.cuda.synchronize()
    if check:
        assert rc == 0, rc
    return rc, out


def run_dev(lig, pos, n_poses, tr, rot, tor, table, step=None, seed=0, keys=None, tr_z=None, rot_z=None, tor_z=None,
            use_torsion=True, out=None):
    from diffdock_b200 import _lib
    bu, bv, mk = device_bonds(lig)
    if out is None:
        out = torch.full_like(pos, float('nan'))
    rc = _lib.lib().ddb200_pose_update_dev(_p(pos), n_poses, lig.n, len(lig.bonds), _p(bu), _p(bv), _p(mk), _p(tr), _p(rot),
                                           _p(tor), _p(tr_z), _p(rot_z), _p(tor_z), _p(table), _p(step),
                                           C.c_uint64(seed & 0xFFFFFFFFFFFFFFFF), _p(keys), int(use_torsion), _p(out),
                                           _stream())
    torch.cuda.synchronize()
    assert rc == 0, rc
    return out


def reference(lig, pos, n_poses, tr, rot, tor, coef, tr_z=None, rot_z=None, tor_z=None, use_torsion=True):
    """float64 restatement: perturbation, rigid move about the centroid, sequential torsions, Kabsch onto the rigid pose."""
    from oracle.diffusion import axis_angle_to_matrix, kabsch_batch, torsion_update_batch
    d = lambda t: t.detach().double().cpu()
    a = [float(np.float32(v)) for v in coef]
    z = lambda t, like: d(t) if t is not None else torch.zeros_like(d(like))
    tr_u = a[0] * d(tr) + a[1] * z(tr_z, tr)
    rot_u = a[2] * d(rot) + a[3] * z(rot_z, rot)
    P = d(pos).reshape(n_poses, lig.n, 3)
    cen = P.mean(1, keepdim=True)
    rigid = torch.bmm(P - cen, axis_angle_to_matrix(rot_u).transpose(1, 2)) + tr_u[:, None] + cen
    if not use_torsion or len(lig.bonds) == 0:
        return rigid
    tor_u = a[4] * d(tor) + a[5] * z(tor_z, tor)
    flex = torsion_update_batch(rigid, lig.bonds, torch.from_numpy(lig.mask), tor_u)
    R, t = kabsch_batch(flex, rigid)
    return torch.bmm(flex, R.transpose(1, 2)) + t.transpose(1, 2)


def pose_err(out, ref):
    """Per-pose max |out - ref| over the pose's extent; the largest over the poses."""
    o = out.detach().double().cpu().reshape(ref.shape)
    assert bool(torch.isfinite(o).all()), "non-finite coordinates"
    ext = (ref - ref.mean(1, keepdim=True)).norm(dim=-1).amax(1).clamp_min(1.0)
    return float(((o - ref).abs().amax((1, 2)) / ext).max())


def check(name, out, ref, tol):
    e = pose_err(out, ref)
    print(f"{name}: max err {e:.3e}")
    assert e < tol, (name, e)
    return e


COEF = (0.7, 0.35, 1.3, 0.2, 0.9, 0.45)


# ---- sizes, bonds, poses ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_atoms", [4, 31, 32, 33, 127, 128, 129, 150])
def test_ligand_sizes_around_the_cta_width(built_lib, n_atoms):
    lig = tree_ligand(n_atoms, n_atoms)
    pos = poses_of(lig, 3, n_atoms)
    tr, rot, tor = scores(3, len(lig.bonds), n_atoms)
    tz, rz, qz = scores(3, len(lig.bonds), n_atoms + 1, 1.0, 1.0, 1.0)
    _, out = run(lig, pos, 3, tr, rot, tor, COEF, tz, rz, qz)
    check(f"n_atoms={n_atoms} bonds={len(lig.bonds)}",
          out, reference(lig, pos, 3, tr, rot, tor, COEF, tz, rz, qz), TOL_SIZES)


@pytest.mark.parametrize("n_atoms", [1943, 1944, 8428])
def test_large_ligands_above_the_48k_opt_in(built_lib, n_atoms):
    lig = cloud_ligand(n_atoms, 5, n_atoms)
    pos = poses_of(lig, 2, n_atoms)
    tr, rot, tor = scores(2, 5, n_atoms, tor=0.3)
    _, out = run(lig, pos, 2, tr, rot, tor, COEF)
    check(f"n_atoms={n_atoms}", out, reference(lig, pos, 2, tr, rot, tor, COEF), TOL_LARGE)


def test_too_large_a_ligand_returns_esmem(built_lib):
    lig = cloud_ligand(8429, 2, 1)
    pos = poses_of(lig, 1, 1)
    tr, rot, tor = scores(1, 2, 1)
    rc, out = run(lig, pos, 1, tr, rot, tor, COEF, check=False)
    assert rc == ESMEM and bool(torch.isnan(out).all())


@pytest.mark.parametrize("n_bonds,n_poses", [(0, 3), (1, 1), (3, 40), (4, 3), (5, 1), (8, 40), (9, 3), (30, 40)])
def test_bond_counts_and_pose_counts(built_lib, n_bonds, n_poses):
    lig = tree_ligand(60, 7).first(n_bonds)
    pos = poses_of(lig, n_poses, n_bonds)
    tr, rot, tor = scores(n_poses, n_bonds, 100 + n_bonds)
    _, out = run(lig, pos, n_poses, tr, rot, tor, COEF)
    check(f"bonds={n_bonds} poses={n_poses}", out, reference(lig, pos, n_poses, tr, rot, tor, COEF), TOL_BONDS)


def test_nested_masks_apply_in_bond_order(built_lib):
    lig = nested_ligand()
    pos = poses_of(lig, 3, 3)
    tr, rot, tor = scores(3, 4, 3, tor=1.5)
    _, out = run(lig, pos, 3, tr, rot, tor, COEF)
    check("nested masks", out, reference(lig, pos, 3, tr, rot, tor, COEF), TOL_BONDS)


# ---- values -------------------------------------------------------------------------------------------------------------
def test_rotation_norms_torsion_angles_far_from_the_origin(built_lib):
    """Pose b rotates by a vector of norm ROT[b] (a = 1, c = 0: the score is the update) and turns its bonds by angles
    cycled from TOR; the ligand sits about 100 A from the origin."""
    rots = [0.0, 1e-7, 1e-6, math.pi - 1e-4, 3 * math.pi]
    tors = [0.0, math.pi, -math.pi, 7.0, -7.0]
    lig = tree_ligand(40, 4).first(10)
    n_poses = len(rots)
    pos = poses_of(lig, n_poses, 5, shift=(60.0, -70.0, 40.0))
    g = torch.Generator().manual_seed(1)
    dirs = torch.nn.functional.normalize(torch.randn(n_poses, 3, generator=g), dim=1)
    rot = (dirs * torch.tensor(rots)[:, None]).float().cuda()
    tor = torch.tensor([[tors[(b + r) % 5] for r in range(10)] for b in range(n_poses)]).float().cuda()
    tr = torch.randn(n_poses, 3, generator=g).cuda()
    coef = (1.0, 0.0, 1.0, 0.0, 1.0, 0.0)
    _, out = run(lig, pos, n_poses, tr, rot, tor, coef)
    check("rotation norms / torsion angles at 100 A", out, reference(lig, pos, n_poses, tr, rot, tor, coef), TOL_VALUES)


def test_use_torsion_off_gives_the_rigid_pose(built_lib):
    lig = tree_ligand(33, 2)
    pos = poses_of(lig, 3, 8, shift=(100.0, 0.0, 0.0))
    tr, rot, tor = scores(3, len(lig.bonds), 8)
    tz, rz, _ = scores(3, 0, 9, 1.0, 1.0)
    _, out = run(lig, pos, 3, tr, rot, None, COEF, tz, rz, use_torsion=False)
    check("use_torsion=0", out, reference(lig, pos, 3, tr, rot, None, COEF, tz, rz, use_torsion=False), TOL_VALUES)


# ---- device coefficient table, in place, Philox ------------------------------------------------------------------------
def test_dev_table_row_of_step_and_in_place(built_lib):
    lig = tree_ligand(50, 5).first(6)
    tr, rot, tor = scores(3, 6, 12)
    tz, rz, qz = scores(3, 6, 13, 1.0, 1.0, 1.0)
    table = torch.tensor([[0.5 + 0.1 * k, 0.2 * k, 1.0 - 0.05 * k, 0.1 + 0.03 * k, 0.3 + 0.2 * k, 0.4 - 0.02 * k]
                          for k in range(5)]).cuda()
    for k in (None, 0, 3, 4):
        pos = poses_of(lig, 3, 20)
        ref = reference(lig, pos, 3, tr, rot, tor, table[k or 0].tolist(), tz, rz, qz)
        step = torch.tensor([k], dtype=torch.int32).cuda() if k is not None else None
        out = run_dev(lig, pos, 3, tr, rot, tor, table, step, tr_z=tz, rot_z=rz, tor_z=qz)
        check(f"table row step={k}", out, ref, TOL_DEV)
        run_dev(lig, pos, 3, tr, rot, tor, table, step, tr_z=tz, rot_z=rz, tor_z=qz, out=pos)    # out aliases pos
        assert torch.equal(pos, out), f"in-place update differs (step={k})"


def _probe(seed, key, step, n_blocks):
    from diffdock_b200 import _lib
    z = torch.full((n_blocks, 4), float('nan'), device='cuda')
    raw = torch.zeros((n_blocks, 4), dtype=torch.int32, device='cuda')
    rc = _lib.lib().ddb200_philox_probe(C.c_uint64(seed), key, step, 0, n_blocks, _p(z), _p(raw), _stream())
    torch.cuda.synchronize()
    assert rc == 0
    return z, raw


def test_philox_noise_blocks_and_slots(built_lib):
    """In-kernel noise = the probe's normals at (seed, pose_key[b], step): translation block 0, rotation block 1, torsion r
    block 2 + r // 4 slot r % 4.  Keys carry a complex id in the high word; one is negative."""
    nb, seed, step = 9, 0x0123456789ABCDEF, 3
    lig = tree_ligand(45, 6).first(nb)
    keys = [(7 << 32) | 0, (7 << 32) | 1, (123456 << 32) | 5, -5]
    n_poses = len(keys)
    tr, rot, tor = scores(n_poses, nb, 30)
    table = torch.tensor([[0.0] * 6] * 3 + [[0.6, 0.8, 1.1, 0.5, 0.9, 0.7]]).cuda()
    tz, rz, qz = [], [], []
    for key in keys:
        z, _ = _probe(seed, key, step, 2 + (nb + 3) // 4)
        z = z.cpu()
        tz.append(z[0, :3])
        rz.append(z[1, :3])
        qz.append(torch.stack([z[2 + r // 4, r % 4] for r in range(nb)]))
    tz, rz, qz = torch.stack(tz), torch.stack(rz), torch.stack(qz)
    pos = poses_of(lig, n_poses, 31)
    out = run_dev(lig, pos, n_poses, tr, rot, tor, table, torch.tensor([step], dtype=torch.int32).cuda(), seed=seed,
                  keys=torch.tensor(keys, dtype=torch.int64).cuda())
    check("philox noise", out, reference(lig, pos, n_poses, tr, rot, tor, table[step].tolist(), tz, rz, qz), TOL_DEV)


def test_philox_box_muller_against_float64(built_lib):
    """The probe's normals against Box-Muller recomputed in float64 from its raw words: u = ((w >> 8) + 0.5) / 2^24,
    z = sqrt(-2 ln u1) (cos, sin)(2 pi u2) for the word pairs (0, 1) and (2, 3) of each block."""
    worst = 0.0
    for seed, key, step in ((0, 0, 0), (0x0123456789ABCDEF, (7 << 32) | 3, 11), (2 ** 64 - 1, -5, 19)):
        z, raw = _probe(seed, key, step, 4096)
        w = raw.cpu().numpy().view(np.uint32).astype(np.float64)
        u = (np.floor(w / 256) + 0.5) / 2 ** 24
        rad = np.sqrt(-2 * np.log(u[:, 0::2]))
        ref = np.empty_like(u)
        ref[:, 0::2] = rad * np.cos(2 * np.pi * u[:, 1::2])
        ref[:, 1::2] = rad * np.sin(2 * np.pi * u[:, 1::2])
        worst = max(worst, float(np.abs(z.cpu().double().numpy() - ref).max()))
    print(f"Box-Muller: max abs err {worst:.3e}")
    assert worst < BM_TOL, worst


# ---- degenerate geometry ------------------------------------------------------------------------------------------------
def test_planar_ligand(built_lib):
    lig = tree_ligand(30, 9).first(6)
    lig = Lig(lig.pos * np.array([1, 1, 0], dtype=np.float32), lig.bonds, lig.mask)
    pos = torch.from_numpy(np.tile(lig.pos, (3, 1)) + np.float32(5)).cuda()
    tr, _, tor = scores(3, 6, 40)
    rot = torch.zeros(3, 3, device='cuda')
    _, out = run(lig, pos, 3, tr, rot, tor, COEF)
    check("planar", out, reference(lig, pos, 3, tr, rot, tor, COEF), TOL_DEGEN)


def test_zero_torsions_give_the_rigid_pose(built_lib):
    lig = tree_ligand(64, 10).first(12)
    pos = poses_of(lig, 3, 41)
    tr, rot, _ = scores(3, 12, 41)
    tor = torch.zeros(3, 12, device='cuda')
    _, out = run(lig, pos, 3, tr, rot, tor, COEF)
    _, rigid = run(lig, pos, 3, tr, rot, None, COEF, use_torsion=False)
    check("zero torsions vs rigid kernel", out, rigid.double().cpu().reshape(3, lig.n, 3), TOL_DEGEN)
    check("zero torsions vs reference", out, reference(lig, pos, 3, tr, rot, None, COEF, use_torsion=False), TOL_DEGEN)


@pytest.mark.parametrize("off_axis", [False, True])
def test_collinear_ligand_stays_finite(built_lib, off_axis):
    """The heavy atoms of 2-butyne (C-C#C-C, collinear) with its central bond rotatable: a zero rotation update keeps every
    atom on the line, so the Kabsch covariance has rank 1.  The output must be the rigid pose, not NaN."""
    x = np.array([0.0, 1.46, 2.66, 4.12], dtype=np.float32)
    pos = np.stack([x, np.zeros(4, np.float32), np.zeros(4, np.float32)], 1)
    if off_axis:
        pos = pos @ np.array([[0.36, 0.48, -0.8], [-0.8, 0.6, 0.0], [0.48, 0.64, 0.6]], dtype=np.float32)
    lig = Lig(pos, [(1, 2)], [[False, False, True, True]])
    P = torch.from_numpy(np.tile(lig.pos, (3, 1))).cuda()
    tr = torch.tensor([[0.0, 0.0, 0.0], [0.5, 0.0, 0.0], [0.0, -1.0, 2.0]]).cuda()
    rot = torch.zeros(3, 3, device='cuda')
    tor = torch.tensor([[0.0], [1.0], [-2.5]]).cuda()
    coef = (1.0, 0.0, 1.0, 0.0, 1.0, 0.0)
    _, out = run(lig, P, 3, tr, rot, tor, coef)
    check(f"collinear off_axis={off_axis}", out, reference(lig, P, 3, tr, rot, tor, coef), TOL_DEGEN)
    check(f"collinear off_axis={off_axis} vs rigid",
          out, reference(lig, P, 3, tr, rot, None, coef, use_torsion=False), TOL_DEGEN)


# ---- argument errors ----------------------------------------------------------------------------------------------------
def test_argument_errors_and_no_poses(built_lib):
    """Every DDB200_EINVAL combination returns before a launch (the output keeps its NaN fill); n_poses = 0 is a no-op."""
    from diffdock_b200 import _lib
    L = _lib.lib()
    lig = tree_ligand(20, 11).first(3)
    pos = poses_of(lig, 2, 50)
    tr, rot, tor = scores(2, 3, 50)
    bu, bv, mk = device_bonds(lig)
    table = torch.ones(1, 6, device='cuda')
    c6 = (C.c_float * 6)(*COEF)
    out = torch.full_like(pos, float('nan'))
    base = dict(pos=pos, n=2, na=lig.n, nb=3, bu=bu, bv=bv, mk=mk, tr=tr, rot=rot, tor=tor, coef=c6, ut=1, out=out)
    bad = [dict(pos=None), dict(out=None), dict(tr=None), dict(rot=None), dict(coef=None), dict(n=-1), dict(na=0),
           dict(na=-3), dict(nb=-1), dict(bu=None), dict(bv=None), dict(mk=None), dict(tor=None)]

    def call(a, dev):
        coef = C.cast(a['coef'], C.c_void_p) if a['coef'] is not None else None
        if dev:
            coef = _p(table) if a['coef'] is not None else None
            return L.ddb200_pose_update_dev(_p(a['pos']), a['n'], a['na'], a['nb'], _p(a['bu']), _p(a['bv']), _p(a['mk']),
                                            _p(a['tr']), _p(a['rot']), _p(a['tor']), None, None, None, coef, None,
                                            C.c_uint64(0), None, a['ut'], _p(a['out']), _stream())
        return L.ddb200_pose_update(_p(a['pos']), a['n'], a['na'], a['nb'], _p(a['bu']), _p(a['bv']), _p(a['mk']),
                                    _p(a['tr']), _p(a['rot']), _p(a['tor']), None, None, None, coef, a['ut'], _p(a['out']),
                                    _stream())

    for dev in (False, True):
        for b in bad:
            assert call({**base, **b}, dev) == EINVAL, (dev, b)
        # without torsions the bond arrays are not needed
        assert call({**base, 'bu': None, 'bv': None, 'mk': None, 'tor': None, 'ut': 0}, dev) == 0
        assert call({**base, 'bu': None, 'bv': None, 'mk': None, 'tor': None, 'nb': 0}, dev) == 0
        torch.cuda.synchronize()
        out.fill_(float('nan'))
        assert call({**base, 'n': 0}, dev) == 0
        torch.cuda.synchronize()
        assert bool(torch.isnan(out).all()), "n_poses = 0 wrote output"
