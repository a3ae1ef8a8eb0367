"""Centered RMSProp and AdagradDA on the parameter server, cpu backend: defaults, validation and flags; the cpu serve
loop against scalar fp64 evaluations of TF 1.15's ApplyCenteredRMSProp / ApplyAdagradDA over several passes (per push
and merged, AdagradDA's T counted across passes and continued from a restored sched_step); the shard layout with the
third slot; checkpoints of the third slot and their refusals; the worker / ps agreement; lock-step and CLI training."""
import ctypes as C
import dataclasses
import math
import tempfile

import _harness
import pytest
import torch

from bench_tools.gpu_e2e import tf1_apply
from dist_mnist_b200 import _native as N
from dist_mnist_b200 import cli
from dist_mnist_b200.cluster import ClusterSpec
from dist_mnist_b200.models import mlp
from dist_mnist_b200.parallel.config import EngineConfig, LrSchedule, OptimizerConfig
from dist_mnist_b200.parallel.ps import ParameterServer, shard_carver
from dist_mnist_b200.parallel.sharding import build_layout
from dist_mnist_b200.parallel.worker import Worker
from dist_mnist_b200.session import InProcessCluster, free_port, train_loop
from dist_mnist_b200.utils import ckpt, data

RULES = {
    "centered": OptimizerConfig("rmsprop", 1e-3, centered=True),
    "centered_momentum": OptimizerConfig("rmsprop", 1e-3, centered=True, momentum=0.9, decay=0.8, eps=1e-6),
    "adagrad_da": OptimizerConfig("adagrad_da", 0.1),
    "adagrad_da_l1_l2": OptimizerConfig("adagrad_da", 0.1, l1_regularization_strength=1e-4,
                                        l2_regularization_strength=1e-2),
}


# ---- config and CLI ---------------------------------------------------------------------------------------------


def test_defaults_and_validation():
    c = OptimizerConfig("rmsprop", centered=True)
    assert (c.decay, c.momentum, c.eps, c.centered, c.uses_mg) == (0.9, 0.0, 1e-10, True, True)
    assert c.slot_init() == (0.0, 1.0)
    assert not OptimizerConfig("rmsprop").uses_mg and not OptimizerConfig("rmsprop").centered
    d = OptimizerConfig("adagrad_da")
    assert (d.initial_accumulator_value, d.l1_regularization_strength, d.l2_regularization_strength) == (0.1, 0.0, 0.0)
    assert d.slot_init() == (0.0, 0.1) and not d.uses_mg and d.native_kind == N.OPT_ADAGRAD_DA == 9
    assert OptimizerConfig("adagrad_da", initial_accumulator_value=0.5).slot_init() == (0.0, 0.5)
    for kind in ("adam", "sgd", "momentum", "adagrad", "adadelta", "ftrl", "adagrad_da"):
        with pytest.raises(ValueError, match="centered"):
            OptimizerConfig(kind, centered=True)
    for bad in (0.0, -0.1, float("nan"), float("inf")):
        with pytest.raises(ValueError):
            OptimizerConfig("adagrad_da", initial_accumulator_value=bad)
    for name in ("l1_regularization_strength", "l2_regularization_strength"):
        for bad in (-1e-3, float("nan"), float("inf")):
            with pytest.raises(ValueError):
                OptimizerConfig("adagrad_da", **{name: bad})
    for bad in (float("nan"), float("inf")):
        with pytest.raises(ValueError):
            OptimizerConfig("adagrad_da", bad)
        for name in ("momentum", "decay", "eps", "lr"):
            with pytest.raises(ValueError):
                OptimizerConfig("rmsprop", **{name: bad, "centered": True})
    with pytest.raises(ValueError, match="no hyper-parameter"):
        OptimizerConfig("adagrad_da", rho=0.9)
    with pytest.raises(ValueError, match="no hyper-parameter"):
        OptimizerConfig("adagrad_da", momentum=0.9)
    # the non-centered rule keeps accepting what it accepted
    assert OptimizerConfig("rmsprop", float("inf")).lr == float("inf")
    # schedules and moving averages combine with both
    OptimizerConfig("adagrad_da", 0.1, schedule=LrSchedule("exponential_decay", decay_steps=2, decay_rate=0.5),
                    moving_average_decay=0.9)
    OptimizerConfig("rmsprop", 0.1, centered=True, moving_average_decay=0.9,
                    schedule=LrSchedule("cosine_decay", decay_steps=10))


def _opt(argv):
    return cli.optimizer_config_from_args(cli.build_parser().parse_args(argv))


def test_cli_flags():
    o = _opt(["--optimizer", "rmsprop", "--centered", "--momentum", "0.5"])
    assert (o.kind, o.centered, o.momentum) == ("rmsprop", True, 0.5)
    assert not _opt(["--optimizer", "rmsprop"]).centered
    o = _opt(["--optimizer", "adagrad_da", "--initial_accumulator_value", "0.3", "--l1_regularization_strength",
              "0.01", "--l2_regularization_strength", "0.02", "--learning_rate", "0.5"])
    assert (o.kind, o.initial_accumulator_value, o.l1_regularization_strength, o.l2_regularization_strength,
            o.lr) == ("adagrad_da", 0.3, 0.01, 0.02, 0.5)
    for kind in ("adam", "sgd", "momentum", "adagrad", "adagrad_da", "ftrl"):
        with pytest.raises(ValueError, match="--centered"):
            _opt(["--optimizer", kind, "--centered"])
    # AdagradDA's flags are refused by the kinds that do not use them
    for flag in ("--initial_accumulator_value", "--l1_regularization_strength", "--l2_regularization_strength"):
        for kind in ("adam", "momentum", "rmsprop", "adadelta"):
            with pytest.raises(ValueError, match=flag):
                _opt(["--optimizer", kind, flag, "0.1"])
    for flag in ("--rho", "--momentum", "--rmsprop_decay", "--epsilon", "--learning_rate_power",
                 "--l2_shrinkage_regularization_strength"):
        with pytest.raises(ValueError, match=flag):
            _opt(["--optimizer", "adagrad_da", flag, "0.1"])
    with pytest.raises(ValueError):
        _opt(["--optimizer", "adagrad_da", "--initial_accumulator_value", "0"])


# ---- the cpu serve loop against scalar fp64 -----------------------------------------------------------------------


def _f32(x):
    return float(torch.tensor(x, dtype=torch.float32))


def _scalar_centered(opt, p, mom, ms, mg, g):
    """ApplyCenteredRMSProp on Python floats (fp64)."""
    ms = ms + (g * g - ms) * (1 - opt.decay)
    mg = mg + (g - mg) * (1 - opt.decay)
    mom = mom * opt.momentum + g * opt.lr / math.sqrt(ms - mg * mg + opt.eps)
    return p - mom, mom, ms, mg


def _scalar_da(opt, p, ga, gga, g, T):
    """ApplyAdagradDA on Python floats (fp64), T already an fp32 value."""
    ga, gga = ga + g, gga + g * g
    lr, l1, l2 = opt.lr, opt.l1_regularization_strength, opt.l2_regularization_strength
    den = l2 * T * lr + math.sqrt(gga)
    if l1 > 0:
        p = -lr * math.copysign(max(abs(ga) - T * l1, 0.0), ga) / den
    else:
        p = -lr * ga / den
    return p, ga, gga


def _serve_cpu(opt, apply_mode, grads, p0, sched0=0):
    """Stage every push of grads[w][s] (one 1 x 4 item) in the mailboxes, run the cpu serve loop until it has applied
    them all, and return (params, adam_m, adam_v, mg, final sched_step). The loop takes one push per worker per pass:
    pass s applies push s of every worker, workers in order."""
    n_workers, n_push = len(grads), len(grads[0])
    nslots, n = n_push + 1, 4
    m0, v0 = opt.slot_init()
    params = torch.tensor(p0, dtype=torch.float32)
    m, v, mg = torch.full((n,), m0), torch.full((n,), v0), torch.zeros(n)
    mailbox = torch.zeros(n_workers, nslots, n)
    flags = torch.zeros(n_workers, nslots, 1, dtype=torch.int32)
    for w in range(n_workers):
        for s in range(1, n_push + 1):
            mailbox[w, s % nslots] = torch.tensor(grads[w][s - 1], dtype=torch.float32)
            flags[w, s % nslots, 0] = s
    next_seq = torch.ones(n_workers, 1, dtype=torch.int32)
    consumed = torch.zeros(n_workers, nslots, dtype=torch.int32)
    ctrl = torch.zeros(4, dtype=torch.int32)
    done = torch.full((n_workers,), n_push + 1, dtype=torch.int32)
    items = (N.PsItem * 1)()
    items[0].offset, items[0].rows, items[0].cols, items[0].ld, items[0].flag_index = 0, 1, n, n, 0
    state = (N.PsItemState * 1)()
    state[0].t, state[0].beta1_pow, state[0].beta2_pow, state[0].sched_step = 0, 1.0, 1.0, sched0
    table = (C.c_void_p * N.MAX_WORKERS)()
    P = N.PsServeParams()
    P.params, P.adam_m, P.adam_v = params.data_ptr(), m.data_ptr(), v.data_ptr()
    P.items, P.item_state = C.addressof(items), C.addressof(state)
    P.n_items, P.n_flags, P.n_workers, P.nslots = 1, 1, n_workers, nslots
    P.opt, P.apply_mode = opt.native_kind, N.APPLY_MERGED if apply_mode == "merged" else N.APPLY_PER_PUSH
    P.lr, P.beta1, P.beta2, P.eps = opt.lr, opt.beta1, opt.beta2, opt.eps
    opt.fill_native_rule(P)
    opt.schedule.fill_native(P)
    P.mg = mg.data_ptr() if opt.uses_mg else None
    P.mailbox, P.arena_elems = mailbox.data_ptr(), n
    P.flags, P.next_seq, P.consumed = flags.data_ptr(), next_seq.data_ptr(), consumed.data_ptr()
    P.global_step, P.host_stop, P.exit_counter = ctrl.data_ptr(), ctrl.data_ptr() + 4, ctrl.data_ptr() + 8
    P.worker_done = done.data_ptr()
    P.inbox_table = C.addressof(table)
    lib = N.lib()
    h = lib.dm_cpu_ps_start(C.addressof(P))
    lib.dm_cpu_ps_join(h)
    assert int(ctrl[0]) == n_workers * n_push
    return params.tolist(), m.tolist(), v.tolist(), mg.tolist(), state[0].sched_step


GRADS = [[[0.5, -0.25, 0.125, 2.0], [-0.75, 0.5, 0.25, -1.0], [0.3, 0.1, -0.6, 0.2]],
         [[0.1, -0.2, 0.3, -0.4], [1.5, 0.25, -0.5, 0.75], [-0.05, 0.4, 0.2, -0.3]]]
P0 = [1.0, -0.5, 0.25, 2.0]


def _expected(opt, apply_mode, sched0):
    """Element by element in fp64, in the serve loop's order; T = sched0 + the pass position of the step's last push
    + 1, rounded to fp32 once."""
    nw, npush = len(GRADS), len(GRADS[0])
    m0, v0 = opt.slot_init()
    out = []
    for j in range(4):
        p, m, v, mg = P0[j], m0, _f32(v0), 0.0
        steps = []
        for s in range(npush):
            if apply_mode == "merged":
                steps.append((sum(_f32(GRADS[w][s][j]) for w in range(nw)), (s + 1) * nw))
            else:
                steps += [(_f32(GRADS[w][s][j]), s * nw + w + 1) for w in range(nw)]
        for g, n in steps:
            if opt.kind == "adagrad_da":
                p, m, v = _scalar_da(opt, p, m, v, g, _f32(sched0 + n))
            else:
                p, m, v, mg = _scalar_centered(opt, p, m, v, mg, g)
        out.append((p, m, v, mg))
    return out


# AdagradDA also from a restored sched_step, and across 2^24 (2^24 - 3 + 6 pushes): T keeps counting there, without an
# off-by-one or a wrap. Its fp32 rounding moves these results by ~6e-8, below the bound:
# test_adagrad_da_T_is_rounded_to_fp32 checks the rounding itself.
SERVE_CASES = [("centered", 0), ("centered_momentum", 0)] + [
    (rule, s0) for rule in ("adagrad_da", "adagrad_da_l1_l2") for s0 in (0, 5, (1 << 24) - 3)]


@pytest.mark.parametrize("apply_mode", ["per_push", "merged"])
@pytest.mark.parametrize("rule,sched0", SERVE_CASES)
def test_cpu_serve_loop_matches_scalar_fp64(rule, sched0, apply_mode):
    opt = RULES[rule]
    p, m, v, mg, steps = _serve_cpu(opt, apply_mode, GRADS, P0, sched0)
    want = _expected(opt, apply_mode, sched0)
    for j, (wp, wm, wv, wg) in enumerate(want):
        assert p[j] == pytest.approx(wp, rel=2e-6, abs=1e-9), (j, p[j], wp)
        assert m[j] == pytest.approx(wm, rel=2e-6, abs=1e-9), j
        assert v[j] == pytest.approx(wv, rel=2e-6, abs=1e-9), j
        if opt.uses_mg:
            assert mg[j] == pytest.approx(wg, rel=2e-6, abs=1e-9), j
        else:
            assert mg[j] == 0.0
    # AdagradDA advances sched_step by one per push in both modes; a constant-rate RMSProp leaves it alone
    assert steps == (sched0 + 6 if opt.kind == "adagrad_da" else 0)


def test_adagrad_da_T_is_rounded_to_fp32():
    """One push at sched_step 2^24, so T = 2^24 + 1, whose fp32 value is 2^24. With l1 = 2^-20 and g = 16 + 2^-19
    (both exact in fp32), |g_acc| - T l1 is 2^-19 with the rounded T and 2^-20 with the exact one: the two differ by a
    factor of 2, so the cpu serve loop's result shows which T it used."""
    g, l1 = 16.0 + 2.0 ** -19, 2.0 ** -20
    opt = OptimizerConfig("adagrad_da", 1.0, l1_regularization_strength=l1)
    p, m, v, _, steps = _serve_cpu(opt, "per_push", [[[g] * 4]], [0.5] * 4, sched0=1 << 24)
    assert steps == (1 << 24) + 1 and m == [g] * 4
    den = math.sqrt(_f32(_f32(0.1) + _f32(g * g)))
    rounded, exact = -(g - _f32((1 << 24) + 1) * l1) / den, -(g - ((1 << 24) + 1) * l1) / den
    assert rounded == pytest.approx(2 * exact, rel=1e-12)
    for x in p:
        assert x == pytest.approx(rounded, rel=1e-5), (x, rounded, exact)
    # the reference rounds T the same way
    one = lambda x: torch.tensor([x], dtype=torch.float64)   # noqa: E731
    rp, _, _ = tf1_apply(opt, one(0.5), one(0.0), one(_f32(0.1)), one(g), global_step=(1 << 24) + 1)
    assert float(rp) == pytest.approx(rounded, rel=1e-6)


def test_adagrad_da_l1_zeroes_and_hand_values():
    """Hand-computed one-element values of ApplyAdagradDA (and the reference's): lr 0.5, T 2, g_acc 0 -> 0.5, gg_acc
    0.1 -> 0.35. l1 = 0, l2 = 0.25: p = -0.5 * 0.5 / (2 * 0.5 * 0.25 + sqrt(0.35)); l1 = 0.1: |0.5| - 0.2 = 0.3 in
    the numerator; l1 = 0.3: |g_acc| <= T l1, an exact zero."""
    one = lambda x: torch.tensor([x], dtype=torch.float64)   # noqa: E731
    den = 2 * 0.5 * 0.25 + math.sqrt(0.35)
    for l1, want in ((0.0, -0.25 / den), (0.1, -0.15 / den), (0.3, 0.0)):
        opt = OptimizerConfig("adagrad_da", 0.5, l1_regularization_strength=l1, l2_regularization_strength=0.25)
        p, m, v = tf1_apply(opt, one(7.0), one(0.0), one(0.1), one(0.5), global_step=2)
        assert float(p) == pytest.approx(want, rel=1e-12) and float(m) == 0.5 and float(v) == pytest.approx(0.35)
    # centered RMSProp, decay 0.5, momentum 0.5, eps 0: ms 1 -> 0.625, mg 0 -> 0.25, mom 0.2 -> 0.1 + 0.5 * lr / 0.75
    opt = OptimizerConfig("rmsprop", 0.3, centered=True, decay=0.5, momentum=0.5, eps=0.0)
    p, m, v, g = tf1_apply(opt, one(1.0), one(0.2), one(1.0), one(0.5), mg=one(0.0))
    assert (float(v), float(g)) == (0.625, 0.25)
    assert float(m) == pytest.approx(0.1 + 0.15 / math.sqrt(0.5625), rel=1e-12)
    assert float(p) == pytest.approx(1.0 - float(m), rel=1e-12)


# ---- layout, lock-step, checkpoints, agreement --------------------------------------------------------------------


def test_shard_carver_adds_mg_last():
    spec = mlp.book_model(100)
    layout = build_layout(spec, 2, "round_robin", 64)
    for sh in layout.shards:
        for ema in (False, True):
            off = shard_carver(sh, 2, 2, ema).table()
            on = shard_carver(sh, 2, 2, ema, centered=True).table()
            assert list(on) == list(off) and list(on)[-1] == "mg"
            assert off["mg"][1] == 0 and on["mg"][1] == sh.arena_elems * 4
            for r in off:
                if r != "mg":
                    assert on[r] == off[r], r
            assert on["mg"][0] >= off["ema"][0] + off["ema"][1]


@pytest.mark.parametrize("apply_mode", ["per_push", "merged"])
@pytest.mark.parametrize("nps", [1, 2])
@pytest.mark.parametrize("rule", list(RULES))
def test_lockstep_trajectory_matches_tf1_formulas(rule, nps, apply_mode):
    _harness.cpu_optimizer_lockstep(RULES[rule], nps, apply_mode)


@pytest.mark.parametrize("rule", ["centered_momentum", "adagrad_da_l1_l2"])
def test_lockstep_under_a_schedule_and_moving_averages(rule):
    opt = dataclasses.replace(RULES[rule], schedule=LrSchedule("exponential_decay", decay_steps=2, decay_rate=0.5),
                              moving_average_decay=0.9)
    _harness.cpu_optimizer_lockstep(opt, 2, "per_push")


@pytest.mark.parametrize("rule", ["centered", "adagrad_da"])
def test_training_lowers_the_loss(rule):
    opt = dataclasses.replace(RULES[rule], lr=0.01 if rule == "centered" else 0.5)
    spec = mlp.book_model(64)
    ds = data.synthetic_mnist(2048, seed=0)
    with InProcessCluster(spec, opt, EngineConfig(backend="cpu"), batch_size=32, num_ps=2) as cl:
        res = train_loop(cl.worker, ds, train_steps=300, log_every=0, chunk=50)
        loss, acc = cl.worker.evaluate(ds.images[:512], ds.labels[:512])
    assert res.steps_run == 300
    assert loss < 0.5 * 2.3, loss


def test_mg_region_only_when_centered():
    spec = mlp.book_model(32)
    with InProcessCluster(spec, OptimizerConfig("rmsprop", 1e-3), EngineConfig(backend="cpu"), batch_size=16) as cl:
        with pytest.raises(ValueError, match="mg"):
            cl.worker.read_variables("mg")
    with InProcessCluster(spec, RULES["centered"], EngineConfig(backend="cpu"), batch_size=16) as cl:
        assert all(float(t.abs().max()) == 0.0 for t in cl.worker.read_variables("mg").values())


def test_checkpoint_roundtrip_keeps_all_three_slots_bit_identical():
    spec = mlp.book_model(64)
    opt = RULES["centered_momentum"]
    cfg = EngineConfig(backend="cpu")
    ds = data.synthetic_mnist(512, seed=0)
    d = tempfile.mkdtemp()
    with InProcessCluster(spec, opt, cfg, batch_size=32, num_ps=2) as cl:
        train_loop(cl.worker, ds, train_steps=30, log_every=0, checkpoint_dir=d, chunk=10)
        before = {r: cl.worker.read_variables(r) for r in ("params", "adam_m", "adam_v", "mg")}
    assert any(float(t.abs().max()) > 0 for t in before["mg"].values())
    state = torch.load(ckpt.latest_checkpoint(d), weights_only=False)
    assert state["optimizer"]["centered"] is True and set(state["mg"]) == set(before["mg"])
    with InProcessCluster(spec, opt, cfg, batch_size=32, num_ps=2, restore_dir=d) as cl:
        assert cl.worker.read_global_step() == 30
        for r, vals in before.items():
            got = cl.worker.read_variables(r)
            for k in vals:
                assert torch.equal(got[k], vals[k]), (r, k)
        res = train_loop(cl.worker, ds, train_steps=40, log_every=0, chunk=10)
        assert res.steps_run == 10
    # a non-centered RMSProp run restores the same checkpoint and ignores its mg (TF1's Saver restores what it has)
    with InProcessCluster(spec, OptimizerConfig("rmsprop", 1e-3), cfg, batch_size=32, num_ps=2) as cl:
        assert ckpt.restore_latest(cl.worker, d) == 30


def test_checkpoint_refusals_and_older_checkpoints():
    spec = mlp.book_model(32)
    cfg = EngineConfig(backend="cpu")
    ds = data.synthetic_mnist(256, seed=0)
    d = tempfile.mkdtemp()
    with InProcessCluster(spec, OptimizerConfig("rmsprop", 1e-3), cfg, batch_size=16) as cl:
        train_loop(cl.worker, ds, train_steps=10, log_every=0, checkpoint_dir=d, chunk=10)
    state = torch.load(ckpt.latest_checkpoint(d), weights_only=False)
    assert "mg" not in state and "centered" not in state["optimizer"]
    with InProcessCluster(spec, RULES["centered"], cfg, batch_size=16) as cl:   # a centered run needs mg
        with pytest.raises(RuntimeError, match="mg"):
            ckpt.restore_latest(cl.worker, d)
    # a checkpoint written before `centered` existed restores into a non-centered run
    with InProcessCluster(spec, OptimizerConfig("rmsprop", 1e-3), cfg, batch_size=16) as cl:
        assert ckpt.restore_latest(cl.worker, d) == 10
    # adagrad and adagrad_da checkpoints refuse each other
    da = tempfile.mkdtemp()
    with InProcessCluster(spec, OptimizerConfig("adagrad_da", 0.1), cfg, batch_size=16) as cl:
        train_loop(cl.worker, ds, train_steps=10, log_every=0, checkpoint_dir=da, chunk=10)
    with InProcessCluster(spec, OptimizerConfig("adagrad", 0.1), cfg, batch_size=16) as cl:
        with pytest.raises(RuntimeError, match="optimizer slots"):
            ckpt.restore_latest(cl.worker, da)
    ad = tempfile.mkdtemp()
    with InProcessCluster(spec, OptimizerConfig("adagrad", 0.1), cfg, batch_size=16) as cl:
        train_loop(cl.worker, ds, train_steps=10, log_every=0, checkpoint_dir=ad, chunk=10)
    with InProcessCluster(spec, OptimizerConfig("adagrad_da", 0.1), cfg, batch_size=16) as cl:
        with pytest.raises(RuntimeError, match="optimizer slots"):
            ckpt.restore_latest(cl.worker, ad)
    # an AdagradDA restore continues T at the restored global step
    with InProcessCluster(spec, OptimizerConfig("adagrad_da", 0.1), cfg, batch_size=16, restore_dir=da) as cl:
        assert set(cl.worker.read_sched_steps(0)) == {10}
        train_loop(cl.worker, ds, train_steps=15, log_every=0, chunk=5)
        assert set(cl.worker.read_sched_steps(0)) == {15}


@pytest.mark.parametrize("ps_opt,w_opt", [
    (OptimizerConfig("rmsprop", 1e-3, centered=True), OptimizerConfig("rmsprop", 1e-3)),
    (OptimizerConfig("rmsprop", 1e-3), OptimizerConfig("rmsprop", 1e-3, centered=True)),
    (OptimizerConfig("adagrad", 1e-3), OptimizerConfig("adagrad_da", 1e-3)),
    (OptimizerConfig("adagrad_da", 1e-3), OptimizerConfig("adagrad", 1e-3)),
])
def test_worker_refuses_a_ps_with_another_rule(ps_opt, w_opt):
    spec = mlp.book_model(32)
    cfg = EngineConfig(backend="cpu")
    cluster = ClusterSpec((f"127.0.0.1:{free_port()}",), (f"127.0.0.1:{free_port()}",))
    ps = ParameterServer(cluster, 0, spec, ps_opt, cfg)
    try:
        w = Worker(cluster, 0, spec, w_opt, cfg)
        with pytest.raises(RuntimeError, match="different engine configuration"):
            w.connect()
    finally:
        ps.close()


@pytest.mark.timeout(180)
def test_cli_adagrad_da_one_ps_two_worker_processes():
    common = ["--train_steps", "300", "--learning_rate", "0.5", "--optimizer", "adagrad_da"]
    with _harness.Tasks() as t:
        ps = t.spawn("ps", 0, common + ["--ps_exit_when_done"])
        ws = [t.spawn("worker", i, common) for i in (1, 0)]
        outs = [t.finish(w, 120) for w in ws]
        outp = t.finish(ps, 60)
    for w, o in zip(ws, outs):
        assert w.returncode == 0, o
    assert ps.returncode == 0, outp
    gstep = int(outp.split("exiting: global_step=")[1].split()[0])
    total = sum(int(l.split("local_steps=")[1].split()[0]) for o in outs for l in o.splitlines() if "local_steps=" in l)
    assert gstep == total >= 300
    losses = [float(l.split("loss: ")[1]) for o in outs for l in o.splitlines() if l.startswith("Train step ")]
    assert losses and min(losses) < 0.1
