"""The CLI task harness of tests/_harness.py on the cpu backend: a task that misses its timeout fails the test, and
every task the block started, the ps that nothing else would stop included, is killed and reaped."""
import _harness
import pytest


@pytest.mark.timeout(120)
def test_a_timed_out_task_fails_the_test_and_no_task_outlives_the_block():
    with pytest.raises(pytest.fail.Exception, match="process timed out"):
        with _harness.Tasks(n_workers=1) as t:
            ps = t.spawn("ps", 0, ["--train_steps", "1000000"])          # no --ps_exit_when_done: it never exits
            w0 = t.spawn("worker", 0, ["--train_steps", "1000000"])
            t.finish(w0, 1)
    assert t.procs == [ps, w0]
    assert ps.returncode is not None and w0.returncode is not None
