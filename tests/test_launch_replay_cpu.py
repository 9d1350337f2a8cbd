"""CPU: every entry point of the library's signature table (diffdock_b200/_lib.py:SIGNATURES) is either made by a wrapper
that tests/test_launch_replay_gpu.py records and replays, or on its exempt list with a reason - so that a new entry point
cannot skip the launch replay unnoticed."""
import importlib

from diffdock_b200 import _lib
from tests.test_launch_replay_gpu import CHECKS, EXEMPT, SIZE_QUERIES, WRAPPED


def test_every_entry_point_is_wrapped_or_exempt():
    names = set(_lib.SIGNATURES)
    exempt = {k.split(':')[0] for k in EXEMPT if ':' not in k}
    assert not set(WRAPPED) & exempt, "an entry point is both replayed and exempt"
    assert set(WRAPPED) | exempt == names, (sorted(names - set(WRAPPED) - exempt), sorted(set(WRAPPED) | exempt - names))
    for k in EXEMPT:          # qualified exemptions (a size query of a replayed entry point) name a real entry point
        assert k.split(':')[0] in names and EXEMPT[k]
    assert set(SIZE_QUERIES) <= names


def test_every_wrapper_exists_and_has_a_replay():
    for paths in WRAPPED.values():
        for path in paths:
            mod, name = path.split('.')
            assert callable(getattr(importlib.import_module(f'diffdock_b200.{mod}'), name)), path
            assert path in CHECKS, f"{path} is wrapped but has no per-launch reference"
