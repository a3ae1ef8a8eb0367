"""Gradient clipping on the worker before the push (TF1's `compute_gradients` -> `clip_by_global_norm` /
`clip_by_norm` / `clip_by_value` -> `apply_gradients`), cpu backend: the fp32 reference clip against hand-computed TF1
values, validation of `GradClip` and the CLI flags, lock-step runs checked after every step against an fp32 torch loop
that clips with the reference, a clipping worker against a ps started without clipping, and a multi-process CLI run."""
import _harness
import pytest
import torch

from bench_tools.gpu_e2e import ref_slots
from dist_mnist_b200 import cli
from dist_mnist_b200.cluster import ClusterSpec
from dist_mnist_b200.models import mlp
from dist_mnist_b200.parallel.config import EngineConfig, GradClip, OptimizerConfig
from dist_mnist_b200.parallel.ps import ParameterServer
from dist_mnist_b200.parallel.worker import Worker
from dist_mnist_b200.session import InProcessCluster, free_port
from dist_mnist_b200.utils import data

F32 = torch.float32


def _t(*v):
    return torch.tensor(v, dtype=F32)


# ---------------------------------------------------------------------------------------------------------------
# the reference clip
# ---------------------------------------------------------------------------------------------------------------
def test_clip_by_global_norm_matches_tf1():
    g = {"a": _t(3.0, 0.0), "b": _t(4.0)}                       # global norm 5
    out = mlp.clip_gradients(g, GradClip("global_norm", clip_norm=2.5))
    # scale = 2.5 * min(1/5, 1/2.5) = 2.5 * fl(0.2) = 0.5 exactly in fp32
    assert torch.equal(out["a"], _t(1.5, 0.0)) and torch.equal(out["b"], _t(2.0))
    # unclipped (n = 5 <= 41), yet scaled by 41 * fl(1/41) = 1 - 2^-24 in fp32, as TF1 does
    s = 41.0 * float(torch.tensor(1.0, dtype=F32) / 41.0)
    assert float(torch.tensor(s, dtype=F32)) != 1.0
    out = mlp.clip_gradients(g, GradClip("global_norm", clip_norm=41.0))
    scale = _t(1.0 - 2.0 ** -24)[0]
    assert torch.equal(out["a"], g["a"] * scale) and torch.equal(out["b"], g["b"] * scale)
    assert not torch.equal(out["b"], g["b"])
    # zero gradients: 1/n = inf, min picks 1/clip_norm, the result stays zero
    z = mlp.clip_gradients({"a": torch.zeros(3), "b": torch.zeros(2)}, GradClip("global_norm", clip_norm=1.0))
    assert all(torch.equal(v, torch.zeros_like(v)) for v in z.values())
    # an inf norm makes the scale NaN (TF adds n - n), and so every clipped gradient
    bad = mlp.clip_gradients({"a": _t(float("inf"), 1.0), "b": _t(2.0)}, GradClip("global_norm", clip_norm=1.0))
    assert all(torch.isnan(v).all() for v in bad.values())
    # overflow of the sum of squares is an inf norm too
    bad = mlp.clip_gradients({"a": _t(3e38, 3e38)}, GradClip("global_norm", clip_norm=1.0))
    assert torch.isnan(bad["a"]).all()


def test_clip_by_norm_matches_tf1():
    g = {"a": _t(3.0, 4.0), "b": _t(0.0, 0.0, 0.0), "c": _t(0.5)}
    out = mlp.clip_gradients(g, GradClip("norm", clip_norm=1.0))
    # a: norm 5 > 1 -> (g * 1) / 5, an IEEE divide
    assert torch.equal(out["a"], _t(3.0 / 5.0, 4.0 / 5.0))
    # b: l2 == 0 -> norm = l2 = 0, (0 * c) / max(0, c) = 0: an all-zero variable is unchanged
    assert torch.equal(out["b"], g["b"])
    # c: norm 0.5 <= 1 -> (0.5 * 1) / 1, unchanged
    assert torch.equal(out["c"], g["c"])
    # multiply first, then divide: (g * c) / max(norm, c) rounds differently from g * (c / norm)
    g = {"a": _t(0.1, 0.7, 1.3)}
    c = 0.3
    out = mlp.clip_gradients(g, GradClip("norm", clip_norm=c))
    n = torch.sqrt((g["a"] * g["a"]).sum())
    assert torch.equal(out["a"], (g["a"] * _t(c)[0]) / n)


def test_clip_by_value_matches_tf1():
    g = {"a": _t(-2.0, -0.5, 0.0, 0.25, 3.0), "b": _t(1.0)}
    out = mlp.clip_gradients(g, GradClip("value", value_min=-1.0, value_max=0.5))
    assert torch.equal(out["a"], _t(-1.0, -0.5, 0.0, 0.25, 0.5)) and torch.equal(out["b"], _t(0.5))
    # value_min == value_max pins every element
    out = mlp.clip_gradients(g, GradClip("value", value_min=0.125, value_max=0.125))
    assert all(torch.equal(v, torch.full_like(v, 0.125)) for v in out.values())


def test_grad_clip_off_leaves_gradients_alone():
    g = {"a": _t(1e30, -1e30)}
    assert GradClip().apply(g) is g and not GradClip().enabled


# ---------------------------------------------------------------------------------------------------------------
# configuration and CLI
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kw", [
    {"kind": "l2"},
    {"kind": "global_norm"},                                     # clip_norm required
    {"kind": "norm"},
    {"kind": "global_norm", "clip_norm": 0.0},
    {"kind": "norm", "clip_norm": -1.0},
    {"kind": "global_norm", "clip_norm": float("inf")},
    {"kind": "global_norm", "clip_norm": float("nan")},
    {"kind": "global_norm", "clip_norm": True},
    {"kind": "value", "value_min": -1.0},                         # both bounds required
    {"kind": "value", "value_max": 1.0},
    {"kind": "value", "value_min": 1.0, "value_max": -1.0},       # min > max
    {"kind": "value", "value_min": float("-inf"), "value_max": 1.0},
    {"kind": "value", "value_min": -1.0, "value_max": 1.0, "clip_norm": 1.0},   # a parameter the kind does not use
    {"kind": "global_norm", "clip_norm": 1.0, "value_max": 1.0},
    {"clip_norm": 1.0},                                          # parameters without a kind
    {"value_min": -1.0, "value_max": 1.0},
])
def test_grad_clip_validation(kw):
    with pytest.raises(ValueError):
        GradClip(**kw)


def test_grad_clip_in_optimizer_config():
    assert OptimizerConfig("adam").clip == GradClip()
    o = OptimizerConfig("sgd", 0.1, clip=GradClip("norm", clip_norm=2))
    assert o.clip.clip_norm == 2.0 and isinstance(o.clip.clip_norm, float)
    assert o.as_dict()["clip"] == {"kind": "norm", "clip_norm": 2.0, "value_min": None, "value_max": None}
    assert GradClip.from_dict(o.as_dict()["clip"]) == o.clip and GradClip.from_dict(None) == GradClip()
    with pytest.raises(ValueError):
        OptimizerConfig("sgd", 0.1, clip={"kind": "norm", "clip_norm": 1.0})


def test_atomic_push_mode_refuses_clipping():
    opt = OptimizerConfig("sgd", 0.1, clip=GradClip("global_norm", clip_norm=1.0))
    with pytest.raises(ValueError, match="clipping"):
        EngineConfig(backend="cuda", push_mode="atomic").validate(opt)
    EngineConfig(backend="cuda", push_mode="mailbox").validate(opt)
    EngineConfig(backend="cuda", push_mode="atomic").validate(OptimizerConfig("sgd", 0.1))


def _opt(argv):
    return cli.optimizer_config_from_args(cli.build_parser().parse_args(argv))


def test_cli_clip_flags():
    assert _opt([]).clip == GradClip()
    assert _opt(["--clip_gradients", "global_norm", "--clip_norm", "5"]).clip == GradClip("global_norm", clip_norm=5.0)
    assert _opt(["--clip_gradients", "norm", "--clip_norm", "0.5"]).clip == GradClip("norm", clip_norm=0.5)
    assert (_opt(["--clip_gradients", "value", "--clip_value_min", "-0.1", "--clip_value_max", "0.2"]).clip
            == GradClip("value", value_min=-0.1, value_max=0.2))
    for argv in (["--clip_norm", "1"],                                           # no --clip_gradients
                 ["--clip_value_min", "-1", "--clip_value_max", "1"],
                 ["--clip_value_max", "1"],
                 ["--clip_gradients", "global_norm"],                            # missing --clip_norm
                 ["--clip_gradients", "norm"],
                 ["--clip_gradients", "value", "--clip_value_min", "-1"],        # missing --clip_value_max
                 ["--clip_gradients", "value", "--clip_value_max", "1"],
                 ["--clip_gradients", "value", "--clip_value_min", "1", "--clip_value_max", "-1"],
                 ["--clip_gradients", "global_norm", "--clip_norm", "0"],
                 ["--clip_gradients", "global_norm", "--clip_norm", "-2"],
                 ["--clip_gradients", "global_norm", "--clip_norm", "inf"],
                 ["--clip_gradients", "norm", "--clip_norm", "nan"],
                 ["--clip_gradients", "global_norm", "--clip_norm", "1", "--clip_value_min", "-1"],   # unused flags
                 ["--clip_gradients", "value", "--clip_value_min", "-1", "--clip_value_max", "1", "--clip_norm", "1"]):
        with pytest.raises(ValueError):
            _opt(argv)
    with pytest.raises(SystemExit):
        cli.build_parser().parse_args(["--clip_gradients", "l2"])


def test_cli_atomic_push_mode_refuses_clipping():
    args = cli.build_parser().parse_args(["--push_mode", "atomic", "--optimizer", "sgd", "--clip_gradients", "norm",
                                          "--clip_norm", "1"])
    with pytest.raises(ValueError, match="clipping"):
        cli.engine_config_from_args(args, "cuda").validate(cli.optimizer_config_from_args(args))


# ---------------------------------------------------------------------------------------------------------------
# lock-step runs
# ---------------------------------------------------------------------------------------------------------------
def _ref_step(spec, params, m, v, t, x, y, opt):
    """One fp32 training step in place with the gradients clipped by the reference; returns (loss, t, clipped)."""
    loss, grads, _ = mlp.manual_loss_and_grads(spec, params, x, y)
    c = opt.clip
    if c.kind == "global_norm":
        clipped = float(torch.sqrt(sum((g * g).sum() for g in grads.values()))) > c.clip_norm
    elif c.kind == "norm":
        clipped = any(float(torch.sqrt((g * g).sum())) > c.clip_norm for g in grads.values())
    else:
        clipped = any(bool(((g < c.value_min) | (g > c.value_max)).any()) for g in grads.values())
    grads = mlp.clip_gradients(grads, c)
    t += 1
    for k in params:
        g = grads[k]
        if opt.kind == "sgd":
            params[k] = params[k] - opt.lr * g
        else:
            m[k] = opt.beta1 * m[k] + (1 - opt.beta1) * g
            v[k] = opt.beta2 * v[k] + (1 - opt.beta2) * g * g
            lr_t = opt.lr * (1 - opt.beta2 ** t) ** 0.5 / (1 - opt.beta1 ** t)
            params[k] = params[k] - lr_t * m[k] / (v[k].sqrt() + opt.eps)
    return float(loss), t, clipped


# Chosen so that some of the 10 steps are clipped and others are not (asserted below): over these steps the book
# model's gradient has a global norm of about 0.15-0.21, hid_w a norm of about 0.14-0.2 (the other variables stay
# below 0.07) and a largest element of about 0.008-0.014.
CLIPS = {"global_norm": GradClip("global_norm", clip_norm=0.17),
         "norm": GradClip("norm", clip_norm=0.16),
         "value": GradClip("value", value_min=-0.012, value_max=0.0105)}
RATES = {"sgd": 0.5, "adam": 1e-3}
SHARDINGS = [(1, "round_robin"), (2, "round_robin"), (2, "row_split")]


@pytest.mark.parametrize("shards", SHARDINGS, ids=[f"{n}ps-{s}" for n, s in SHARDINGS])
@pytest.mark.parametrize("kind", ["sgd", "adam"])
@pytest.mark.parametrize("clip", list(CLIPS))
def test_lockstep_trajectory_with_clipping(clip, kind, shards):
    """1 worker, --lanes 1 --strict_steps: the parameters after every step match fp32 torch with the reference clip
    (the tolerances of tests/test_moving_average_cpu.py)."""
    nps, sharding = shards
    opt = OptimizerConfig(kind, RATES[kind], clip=CLIPS[clip])
    spec = mlp.book_model(100)
    cfg = EngineConfig(backend="cpu", lanes=1, strict_steps=True, sharding=sharding)
    ds = data.synthetic_mnist(512, seed=2)
    it = data.BatchIterator(ds, seed=0)
    params = mlp.init_params(spec, seed=5)
    rp = {k: v.clone() for k, v in params.items()}
    rm, rv = ref_slots(opt, params)
    t = 0
    clipped = []
    with InProcessCluster(spec, opt, cfg, batch_size=32, num_ps=nps, params=params) as cl:
        w = cl.worker
        for i in range(10):
            x, y = it.next_batch(32)
            r = w.step(x, y)
            w.wait_applied()
            lref, t, c = _ref_step(spec, rp, rm, rv, t, x, y, opt)
            clipped.append(c)
            assert r.loss == pytest.approx(lref, rel=1e-4)
            got = w.read_variables()
            for k in got:
                assert torch.allclose(got[k], rp[k], rtol=1e-4, atol=1e-6), (i, k)
    assert any(clipped) and not all(clipped), clipped


def test_clipping_changes_the_trajectory():
    """The same run without clipping ends elsewhere: the lock-step runs above do exercise the clip."""
    spec = mlp.book_model(100)
    ds = data.synthetic_mnist(512, seed=2)
    ends = []
    for clip in (GradClip(), CLIPS["global_norm"]):
        it = data.BatchIterator(ds, seed=0)
        opt = OptimizerConfig("sgd", RATES["sgd"], clip=clip)
        with InProcessCluster(spec, opt, EngineConfig(backend="cpu", lanes=1, strict_steps=True), batch_size=32,
                              params=mlp.init_params(spec, seed=5)) as cl:
            for _ in range(4):
                cl.worker.step(*it.next_batch(32))
            cl.worker.wait_applied()
            ends.append(cl.worker.read_variables())
    assert not torch.allclose(ends[0]["hid_w"], ends[1]["hid_w"], rtol=1e-4, atol=1e-6)


# ---------------------------------------------------------------------------------------------------------------
# ps / worker agreement and the CLI
# ---------------------------------------------------------------------------------------------------------------
def test_nan_propagates_like_tf1():
    nan = float("nan")
    # clip_by_value keeps a NaN element NaN (TF's minimum / maximum propagate it)
    out = mlp.clip_gradients({"a": _t(nan, 2.0, -2.0)}, GradClip("value", value_min=-1.0, value_max=1.0))
    assert torch.isnan(out["a"][0]) and torch.equal(out["a"][1:], _t(1.0, -1.0))
    # clip_by_norm: a NaN element makes the norm NaN and so the whole variable; the other variables are unaffected
    out = mlp.clip_gradients({"a": _t(nan, 1.0), "b": _t(3.0, 4.0)}, GradClip("norm", clip_norm=1.0))
    assert torch.isnan(out["a"]).all() and torch.equal(out["b"], _t(0.6, 0.8))
    # clip_by_global_norm: every variable
    out = mlp.clip_gradients({"a": _t(nan, 1.0), "b": _t(3.0, 4.0)}, GradClip("global_norm", clip_norm=1.0))
    assert all(torch.isnan(v).all() for v in out.values())


@pytest.mark.parametrize("kind", ["adam", "momentum"])   # momentum: the ps / worker optimizer dicts are compared
def test_clipping_worker_connects_to_a_ps_without_clipping(kind):
    spec = mlp.book_model(32)
    cfg = EngineConfig(backend="cpu")
    cluster = ClusterSpec((f"127.0.0.1:{free_port()}",), (f"127.0.0.1:{free_port()}",))
    ps = ParameterServer(cluster, 0, spec, OptimizerConfig(kind, 1e-3), cfg)
    try:
        w = Worker(cluster, 0, spec, OptimizerConfig(kind, 1e-3, clip=GradClip("global_norm", clip_norm=1.0)), cfg)
        try:
            w.connect()
        finally:
            w.close()
    finally:
        ps.close()


@pytest.mark.timeout(900)
def test_cli_clip_by_global_norm_one_ps_two_workers():
    common = ["--learning_rate", "0.001", "--log_every", "1000", "--lanes", "1", "--clip_gradients", "global_norm",
              "--clip_norm", "0.1"]
    with _harness.Tasks() as t:
        ps = t.spawn("ps", 0, common + ["--ps_exit_when_done"])
        ws = [t.spawn("worker", i, common) for i in (1, 0)]
        outs = [t.finish(w, 780) for w in ws]
        outp = t.finish(ps, 60)
    for w, o in zip(ws, outs):
        assert w.returncode == 0, o
        assert "done: local_steps=" in o, o
    assert ps.returncode == 0, outp
    gstep = int(outp.split("global_step=")[1].split()[0])
    assert gstep >= 4000, outp
    logged = [l for o in outs for l in o.splitlines() if l.startswith("Train step ")]
    assert logged and all(", loss: " in l for l in logged)
