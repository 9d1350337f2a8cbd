"""CPU: the reference's rule for the frames ``sampling(..., visualization_list=...)`` leaves in the caller's objects
(tests/golden/ref_sampling_visualisation.pt, recorded from the unmodified reference), the host helper that hands them
over, and the captured step no longer being refused for visualisation."""
import pytest
import torch

from tests.parity_helpers import load_golden
from tests.visualisation_helpers import max_rel_diff, prepopulated


@pytest.fixture(scope='module')
def fx():
    return load_golden('ref_sampling_visualisation.pt')


@pytest.mark.parametrize("run", ['a', 'b'])
def test_reference_keeps_the_final_pose_at_order_2(fx, run):
    steps = fx['steps']
    r = fx['runs'][run]
    assert len(r['content']) == len(fx['poses']) == 2 * fx['batch_size']
    for content, final, center in zip(r['content'], r['final_pos'], fx['original_center']):
        part = content[1]
        assert sorted(part) == list(range(1, steps + 2))
        assert torch.equal(part[2], part[steps + 1])            # order 2 is the last frame, not the first
        assert torch.equal(part[2], final + center)
        assert not torch.equal(part[2], part[3])


@pytest.mark.parametrize("run", ['a', 'b'])
def test_add_frames_rebuilds_the_reference_content(fx, run):
    from diffdock_b200.hetero import graph_from_dict
    from diffdock_b200.sampling import _add_frames
    steps, bs = fx['steps'], fx['batch_size']
    r = fx['runs'][run]
    poses = [graph_from_dict(d) for d in fx['poses']]
    # the frames the device would hold: the recorded coordinates minus original_center; frame 0 is not in the reference's
    # result (order 2 is overwritten), so it holds NaN, which must not reach any recorder
    frames = torch.full((steps, len(poses)) + tuple(r['final_pos'][0].shape), float('nan'))
    for i, (content, center) in enumerate(zip(r['content'], fx['original_center'])):
        frames[steps - 1, i] = r['final_pos'][i]
        for t in range(1, steps - 1):
            frames[t, i] = content[1][t + 2] - center
    vis = prepopulated(poses, fx['crystal'])
    for b0 in range(0, len(poses), bs):
        _add_frames(vis, poses, b0, frames[:, b0:b0 + bs])
    for v, ref in zip(vis, r['content']):
        assert max_rel_diff(v.content(), ref) == 0.0


def test_cuda_graph_is_not_refused_for_visualisation():
    from argparse import Namespace
    from functools import partial
    from diffdock_b200.cg_model import CGModel
    from diffdock_b200.diffusion_utils import get_timestep_embedding, t_to_sigma
    from diffdock_b200.sampling import _use_cuda_graph
    from tests.visualisation_helpers import RecordingPDB
    case = load_golden('ref_sampling_visualisation.pt')['fused_case']
    a = Namespace(**case['args'])
    m = CGModel(partial(t_to_sigma, args=a), torch.device('cpu'), get_timestep_embedding('sinusoidal', 8, a.embedding_scale),
                **case['kw'])
    assert m.sync_free_capable()
    assert _use_cuda_graph(m, a, None, [RecordingPDB()], 1, 1, None)
    assert _use_cuda_graph(m, a, None, [RecordingPDB()], 1, 1, True)
    with pytest.raises(RuntimeError):
        _use_cuda_graph(m, a, lambda k, s: torch.zeros(s), None, 1, 1, True)
