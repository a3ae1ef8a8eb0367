"""The comparator of tests/test_gpu_fused_push_exact.py, proved on the CPU: an fp32 emulation of the fused step kernel's
arithmetic (bench_tools/fused_push_ref.emulate) stays inside the fp64 reference's per-element bound with dpre converted
to tf32 by truncation and by round-to-nearest, and each plausible kernel bug (a dropped batch row or row tile, a zeroed
k-chunk or hidden row, a missing ReLU mask, the loss normalised by the padded batch, sm_w transposed or shifted by a
class) lands far outside it at every case of the shape matrix whose coverage admits that bug."""
import pytest

from bench_tools import fused_push_ref as R

MATRIX = R.shape_matrix()


@pytest.mark.parametrize("name,shape,saturate", MATRIX, ids=[m[0] for m in MATRIX])
def test_emulated_kernel_is_inside_the_bound_and_mutants_are_not(name, shape, saturate):
    case = R.case_for(shape, saturate)
    x, y = case.batches[0]
    assert R.check_case(case, x, y) == []
    ref = R.reference(case.spec, case.params, x, y)
    H, C, I, B, _ = shape
    for mode in ("trunc", "rne"):
        v = R.compare(R.emulate(case.spec, case.params, x, y, mode), ref)
        print(f"[{name} seed {case.seed}] emulated, tf32 {mode}: {v.line()}")
        assert v.ok, (mode, v.worst, v.where)
        assert v.worst["hid_w"] < 0.6, v.worst       # the tf32 term leaves room: 2^-9 is twice the truncation error
    muts = R.mutant_instances(case, ref)
    if C == 1:
        assert muts == []
        got = R.emulate(case.spec, case.params, x, y)
        assert all(float(g.abs().max()) == 0.0 for g in got.grads.values()) and got.loss == 0.0
        return
    kinds = {m for m, _ in muts}
    expect = {"drop_row", "zero_chunk", "zero_hidden_row", "sm_w_class_shift"}
    expect |= {"drop_tile"} if B > 32 else set()
    expect |= {"loss_32T"} if B % 32 else set()
    expect |= {"sm_w_transposed"} if H >= 2 else set()
    assert expect <= kinds, (expect - kinds)
    for mode in ("trunc", "rne"):
        for mut, arg in muts:
            v = R.compare(R.emulate(case.spec, case.params, x, y, mode, mut, arg), ref)
            assert v.max > 4.0, (mode, mut, arg, v.worst)


def test_saturated_case_exercises_the_clamp_on_both_sides():
    case = R.case_for((100, 10, 784, 32, "book"), R.SATURATE)
    ref = R.reference(case.spec, case.params, *case.batches[0])
    clamped = int((ref.p_true < R.CLAMP).sum())
    assert 0 < clamped < 32
    assert float(ref.p_true.min()) < 1e-20   # far below the clamp, not at its edge
    # a clamped row pushes nothing
    assert float(ref.dl[ref.p_true < R.CLAMP].abs().max()) == 0.0


def test_hidden_weight_and_inputs_are_exact_in_tf32():
    """Every case of the matrix, and the multi-batch cases of the GPU tests, on every batch."""
    cases = [R.case_for(shape, sat) for _, shape, sat in MATRIX]
    cases += [R.case_for((100, 10, 784, b, "book"), n_batches=12, seed=2) for b in (32, 33, 100, 256)]
    cases += [R.case_for((100, 10, 784, b, "book"), n_batches=8, seed=3) for b in (32, 256)]
    for case in cases:
        assert R.exact_inputs(case) == [], case.name
        assert all(R.check_case(case, x, y) == [] for x, y in case.batches), case.name
    broken = R.case_for((17, 3, 260, 33, "xent"))
    broken.params["hid_w"] = broken.params["hid_w"] + 2.0 ** -20
    assert any("hid_w" in m for m in R.exact_inputs(broken))


def test_tf32_conversions():
    import torch

    v = torch.tensor([1.0 + 2.0 ** -11, 1.0 + 3 * 2.0 ** -11, 1.0 + 2.0 ** -12, -(1.0 + 2.0 ** -11 + 2.0 ** -13)])
    assert R.to_tf32(v, "trunc").tolist() == [1.0, 1.0 + 2.0 ** -10, 1.0, -1.0]
    assert R.to_tf32(v, "rne").tolist() == [1.0, 1.0 + 2.0 ** -9, 1.0, -(1.0 + 2.0 ** -10)]


def test_comparator_reports_the_element_of_a_wrong_value():
    case = R.case_for((100, 10, 260, 33, "xent"))
    x, y = case.batches[0]
    ref = R.reference(case.spec, case.params, x, y)
    got = R.emulate(case.spec, case.params, x, y)
    got.grads["hid_w"][57, 259] += 1e-3
    v = R.compare(got, ref)
    assert not v.ok and v.where["hid_w"][:2] == (57, 259)
    got = R.emulate(case.spec, case.params, x, y)
    got.grads["sm_b"][3] *= 1.01
    v = R.compare(got, ref)
    assert v.worst["sm_b"] > 1 and v.where["sm_b"] == (3,)
    got = R.emulate(case.spec, case.params, x, y)
    got.correct = ref.correct_hi + 1
    assert not R.compare(got, ref).ok
