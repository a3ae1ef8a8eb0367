"""End-to-end engine on one H100 (ps + worker in one process): trajectories vs a PyTorch re-implementation."""
import pytest

pytestmark = pytest.mark.gpu


def test_smoke_entry_point():
    import __graft_entry__ as g
    g.smoke()


def test_lockstep_trajectories_all_models_and_modes():
    from bench_tools import gpu_e2e
    assert gpu_e2e.check_traj()


def test_pipelined_steps_in_flight_and_group_graphs():
    from bench_tools import gpu_e2e
    assert gpu_e2e.check_pipelined()
