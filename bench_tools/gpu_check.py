"""Bring-up checks for the sm_90a kernels against plain PyTorch fp32 references.

Each group runs in its own process (a kernel trap poisons the CUDA context) and keeps going after a
mismatch so one GPU call yields the full picture:

    python -m bench_tools.gpu_check all            # spawns one subprocess per group
    python -m bench_tools.gpu_check gemm_fwd       # a single group in-process
"""
from __future__ import annotations

import ctypes as C
import dataclasses
import struct
import subprocess
import sys
import time
import traceback
from typing import Optional

import torch

GROUPS = ["gemm_fwd", "gemm_dw", "gemm_dx", "head", "accuracy", "ps_serve", "dense_apply", "p2p_local"]


def rel_err(a: torch.Tensor, b: torch.Tensor) -> float:
    a = a.float()
    b = b.float()
    return float((a - b).norm() / (b.norm() + 1e-12))


def report(name: str, ok: bool, detail: str) -> bool:
    print(f"[{'PASS' if ok else 'FAIL'}] {name}: {detail}", flush=True)
    return ok


def tdtype(dt):
    from dist_mnist_b200 import _native as N
    return torch.float32 if dt == N.DT_F32 else torch.bfloat16


def round_operand(t: torch.Tensor, dt) -> torch.Tensor:
    """Operand as the tensor core sees it, for a fair fp32 reference."""
    from dist_mnist_b200 import _native as N
    if dt == N.DT_BF16:
        return t.to(torch.bfloat16).float()
    # tf32 keeps 10 mantissa bits (truncation of the low 13 bits)
    return (t.view(torch.int32) & ~0x1FFF).view(torch.float32)


def padded(t: torch.Tensor, dt) -> torch.Tensor:
    """Copy a [R, C] fp32 tensor into a [R, padded_ld(C)] buffer of the compute dtype; returns the buffer."""
    from dist_mnist_b200.ops import gemm
    R, Cc = t.shape
    buf = torch.zeros(R, gemm.padded_ld(Cc), device=t.device, dtype=tdtype(dt))
    buf[:, :Cc] = t.to(tdtype(dt))
    return buf


# Tolerances against an UN-ROUNDED reference (fp64 math on the fp32 inputs — what the reference's fp32 TensorFlow ops
# compute up to fp32 rounding): operand rounding to tf32 (10-bit mantissa, truncation) / bf16 (8-bit) bounds the
# relative error of a dot product by ~2^-10 / ~2^-8 per term; measured values are printed next to the bound.
TOL_EXACT = {0: 4e-3, 1: 2.5e-2}


def exact(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    return (a.double() @ b.double()).float()


def random_shapes(n: int, seed: int, max_b: int = 256):
    """Seeded random (O, I, B) shapes on top of the fixed ones (SURVEY section 4.3: shapes should not be hand-picked
    only): O in [1, 1100], I in [8, 1100] multiple of 8, B in [1, max_b]."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(n):
        O = int(torch.randint(1, 1101, (1,), generator=g))
        I = int(torch.randint(1, 138, (1,), generator=g)) * 8
        B = int(torch.randint(1, max_b + 1, (1,), generator=g))
        out.append((O, I, B))
    return out


def check_gemm_fwd(activation: str = "relu") -> bool:
    """The forward epilogue without an activation and with `activation` (an mlp.ACTIVATIONS name): fp32 and bf16 out,
    padding rows zero."""
    from dist_mnist_b200 import _native as N
    from dist_mnist_b200.models import mlp
    from dist_mnist_b200.ops import gemm
    ok = True
    dev = "cuda"
    for dt, tol in ((N.DT_F32, 2e-3), (N.DT_BF16, 8e-3)):
        for (O, I, B) in [(100, 784, 32), (128, 64, 16), (1024, 784, 64), (500, 500, 100), (1024, 1024, 256)] + random_shapes(6, 1234):
            B_pad = gemm.round_up(B, 16)
            torch.manual_seed(O + I + B)
            w = torch.randn(O, I, device=dev) * 0.05
            x = torch.zeros(B_pad, I, device=dev)
            x[:B] = torch.randn(B, I, device=dev)
            bias = torch.randn(O, device=dev) * 0.1
            wd, xd = padded(w, dt), padded(x, dt)
            outp = torch.zeros(B_pad, gemm.padded_ld(O), device=dev, dtype=tdtype(dt))
            out = outp[:, :O]
            for act in (None, activation):
                outp.zero_()
                plan = gemm.forward_plan(w_ptr=wd.data_ptr(), x_ptr=xd.data_ptr(), out_ptr=outp.data_ptr(),
                                         bias_ptr=bias.data_ptr(), O=O, I=I, B=B, B_pad=B_pad, dtype=dt,
                                         act=N.ACT_NONE if act is None else mlp.activation_code(act),
                                         ldw=wd.shape[1], ldx=xd.shape[1], ldo=outp.shape[1])
                plan.launch()
                torch.cuda.synchronize()
                ref = round_operand(x[:B], dt) @ round_operand(w, dt).t() + bias
                if act is not None:
                    ref = mlp.activate(act, ref)
                e = rel_err(out[:B], ref)
                ref_x = exact(x[:B], w.t()) + bias          # un-rounded operands
                if act is not None:
                    ref_x = mlp.activate(act, ref_x)
                ex = rel_err(out[:B], ref_x)
                pad_zero = bool((outp[B:] == 0).all() and (outp[:, O:] == 0).all())
                ok &= report(f"fwd dt={dt} O={O} I={I} B={B} act={act}", e < tol and ex < TOL_EXACT[dt] and pad_zero,
                             f"rel_err={e:.2e} vs_unrounded_fp32={ex:.2e} pad_zero={pad_zero} stages={plan.params.stages}")
    return ok


def check_gemm_dw() -> bool:
    from dist_mnist_b200 import _native as N
    from dist_mnist_b200.ops import gemm
    ok = True
    dev = "cuda"
    for dt, tol in ((N.DT_F32, 2e-3), (N.DT_BF16, 8e-3)):
        for (O, I, B) in [(100, 784, 32), (128, 64, 64), (1024, 784, 64), (500, 500, 112), (1024, 1024, 256)] + [
                (o, i, (b + 15) // 16 * 16) for (o, i, b) in random_shapes(4, 99)]:
            torch.manual_seed(O * 3 + I + B)
            dy = torch.randn(B, O, device=dev) * 0.1
            x = torch.randn(B, I, device=dev)
            dyd, xd = padded(dy, dt), padded(x, dt)
            ldw = gemm.padded_ld(I)
            ref = round_operand(dy, dt).t() @ round_operand(x, dt)
            ref_x = exact(dy.t(), x)
            for mode in ("local", "atomic"):
                g = torch.zeros(O * ldw + 64, device=dev)
                off = 64
                if mode == "local":
                    push = gemm.local_push(g.data_ptr())
                else:
                    push = N.PushTarget()
                    push.mode = N.PUSH_ATOMIC
                    push.scale = -0.5
                    push.base = g.data_ptr()
                    push.nslots = 1
                plan = gemm.dw_plan(dy_ptr=dyd.data_ptr(), x_ptr=xd.data_ptr(), O=O, I=I, B_pad=B, dtype=dt,
                                    push=push, push_offset=off, lddy=dyd.shape[1], ldx=xd.shape[1], ldw=ldw)
                plan.launch()
                torch.cuda.synchronize()
                got = g[off:].view(O, ldw)[:, :I]
                want = ref if mode == "local" else -0.5 * ref
                e = rel_err(got, want)
                ex = rel_err(got, ref_x if mode == "local" else -0.5 * ref_x)
                guard = bool((g[:off] == 0).all())
                ok &= report(f"dw dt={dt} O={O} I={I} B={B} mode={mode}", e < tol and ex < TOL_EXACT[dt] and guard,
                             f"rel_err={e:.2e} vs_unrounded_fp32={ex:.2e} guard={guard} grid={plan.grid}")
    return ok


def _act_scale(activation: str) -> float:
    """Spread of the pre-activations the dX and head checks draw: wide enough for saturated sigmoid / tanh units and
    relu6's upper kink (ReLU keeps its standard normal inputs)."""
    return 1.0 if activation == "relu" else 4.0


def check_gemm_dx(activation: str = "relu") -> bool:
    """The dX epilogue: dx = (dy . W) * f'(h) for `activation` f, with h = f(random), and its bias-gradient sums."""
    from dist_mnist_b200 import _native as N
    from dist_mnist_b200.models import mlp
    from dist_mnist_b200.ops import gemm
    ok = True
    dev = "cuda"
    for dt, tol in ((N.DT_F32, 2e-3), (N.DT_BF16, 8e-3)):
        for (O, I, B) in ((1024, 1024, 32), (500, 500, 100), (128, 256, 16), (10, 100, 32), (1024, 784, 256)):
            B_pad = gemm.round_up(B, 16)
            torch.manual_seed(O * 7 + I + B)
            w = torch.randn(O, I, device=dev) * 0.05
            dy = torch.zeros(B_pad, O, device=dev)
            dy[:B] = torch.randn(B, O, device=dev) * 0.1
            h = torch.zeros(B_pad, I, device=dev)
            h[:B] = mlp.activate(activation, _act_scale(activation) * torch.randn(B, I, device=dev))
            wd, dyd, hd = (padded(t, dt) for t in (w, dy, h))
            outp = torch.zeros(B_pad, gemm.padded_ld(I), device=dev, dtype=tdtype(dt))
            out = outp[:, :I]
            gb = torch.zeros(I + 32, device=dev)
            plan = gemm.dx_plan(w_ptr=wd.data_ptr(), dy_ptr=dyd.data_ptr(), out_ptr=outp.data_ptr(),
                                mask_ptr=hd.data_ptr(), O=O, I=I, B=B, B_pad=B_pad, dtype=dt,
                                act=mlp.activation_code(activation), ldw=wd.shape[1], lddy=dyd.shape[1], ldo=outp.shape[1],
                                colsum=gemm.local_push(gb.data_ptr()), colsum_offset=32)
            plan.launch()
            torch.cuda.synchronize()
            ref = mlp.activation_grad(activation, round_operand(h[:B], dt),
                                      round_operand(dy[:B], dt) @ round_operand(w, dt))
            e = rel_err(out[:B], ref)
            eb = rel_err(gb[32:], ref.sum(dim=0))
            pad_zero = bool((outp[B:] == 0).all())
            ok &= report(f"dx dt={dt} O={O} I={I} B={B} act={activation}", e < tol and eb < tol and pad_zero,
                         f"rel_err={e:.2e} bias_grad_err={eb:.2e} pad_zero={pad_zero}")
    return ok


def check_head(activation: str = "relu", loss: Optional[str] = None, label_smoothing: float = 0.0) -> bool:
    """The head kernel on h = f(random) of `activation` f: loss, correct count, small gradients and dpre = dh * f'(h),
    under `loss` with `label_smoothing` (loss None: book and xent, unsmoothed)."""
    from dist_mnist_b200 import _native as N
    from dist_mnist_b200.models import mlp
    from dist_mnist_b200.ops import gemm, head
    ok = True
    dev = "cuda"
    loss_names = ("book", "xent") if loss is None else (loss,)   # (`loss` names the reference's value below)
    for act_bf16 in (False, True):
        for loss_name in loss_names:
            loss_kind = mlp.loss_code(loss_name)
            for (H, B) in ((100, 32), (1024, 100), (500, 256), (37, 5)):
                Cn = 10
                B_pad = gemm.round_up(B, 16)
                torch.manual_seed(H + B)
                adt = torch.bfloat16 if act_bf16 else torch.float32
                h = torch.zeros(B_pad, H, device=dev)
                h[:B] = mlp.activate(activation, _act_scale(activation) * torch.randn(B, H, device=dev))
                hq = h.to(adt)
                w = (torch.randn(Cn, H, device=dev) / H ** 0.5).contiguous()
                b = torch.randn(Cn, device=dev) * 0.1
                labels = torch.zeros(B_pad, Cn, device=dev)
                labels[torch.arange(B), torch.randint(0, Cn, (B,))] = 1.0
                dpre = torch.full((B_pad, H), 7.0, device=dev).to(adt)
                n_small = Cn * H + Cn + H
                g = torch.zeros(n_small + 16, device=dev)
                off_w, off_b, off_bh = 16, 16 + Cn * H, 16 + Cn * H + Cn
                res = torch.zeros(4, dtype=torch.int32, device=dev)
                plan = head.head_plan(h_ptr=hq.data_ptr(), labels_ptr=labels.data_ptr(), w_last_ptr=w.data_ptr(),
                                      b_last_ptr=b.data_ptr(), dpre_ptr=dpre.data_ptr(), result_ptr=res.data_ptr(),
                                      B=B, B_pad=B_pad, H=H, num_classes=Cn, loss_kind=loss_kind, act_bf16=act_bf16,
                                      act=mlp.activation_code(activation), label_smoothing=label_smoothing,
                                      push=gemm.local_push(g.data_ptr()), off_w_last=off_w, off_b_last=off_b,
                                      off_b_hidden=off_bh)
                plan.launch()
                torch.cuda.synchronize()
                # reference
                hf = hq[:B].float().requires_grad_(True)
                wr = w.clone().requires_grad_(True)
                br = b.clone().requires_grad_(True)
                logits = hf @ wr.t() + br
                spec = mlp.MLPSpec(loss=loss_name, label_smoothing=label_smoothing)
                loss = mlp.loss_from_logits(spec, logits, labels[:B])
                gh, gw, gb_ = torch.autograd.grad(loss, [hf, wr, br])
                dpre_ref = mlp.activation_grad(activation, hf.detach(), gh)
                got_loss = res[:1].view(torch.float32).item()
                got_correct = int(res[2].item())
                e_loss = abs(got_loss - loss.item()) / (abs(loss.item()) + 1e-12)
                e_w = rel_err(g[off_w:off_w + Cn * H].view(Cn, H), gw)
                e_b = rel_err(g[off_b:off_b + Cn], gb_)
                e_bh = rel_err(g[off_bh:off_bh + H], dpre_ref.sum(dim=0))
                e_dp = rel_err(dpre[:B], dpre_ref)
                pad_ok = bool((dpre[B:].float() == 0).all())
                corr_ref = mlp.accuracy_count(logits.detach(), labels[:B])
                tol = 2e-2 if act_bf16 else 1e-4
                good = (e_loss < 1e-4 and e_w < 1e-4 and e_b < 1e-4 and e_bh < tol and e_dp < tol and pad_ok
                        and got_correct == corr_ref)
                ok &= report(f"head bf16={act_bf16} loss={loss_name} ls={label_smoothing:g} H={H} B={B} "
                             f"act={activation}", good,
                             f"loss {got_loss:.6f}/{loss.item():.6f} e_w={e_w:.1e} e_b={e_b:.1e} e_bh={e_bh:.1e} "
                             f"e_dpre={e_dp:.1e} pad_ok={pad_ok} correct {got_correct}/{corr_ref}")
    return ok


def check_accuracy() -> bool:
    from dist_mnist_b200.ops import head
    ok = True
    for (B, Cn) in ((32, 10), (10000, 10), (777, 100)):
        torch.manual_seed(B)
        logits = torch.randn(B, Cn, device="cuda")
        labels = torch.zeros(B, Cn, device="cuda")
        labels[torch.arange(B), torch.randint(0, Cn, (B,))] = 1.0
        got = int(head.accuracy_count(logits, labels).item())
        want = int((logits.argmax(-1) == labels.argmax(-1)).sum())
        ok &= report(f"accuracy B={B} C={Cn}", got == want, f"{got} vs {want}")
    return ok


def check_ps_serve(ieee: bool = False, schedule=None, sched_step: int = 0, moving_average_decay=None) -> bool:
    """Single-GPU test of the persistent PS kernel: mailboxes and inboxes are local buffers. `ieee`: the
    `--adam_math ieee` instantiation (correctly rounded sqrt / divide). `schedule` (an LrSchedule): the scheduled
    instantiations, every item starting at schedule step `sched_step`; the reference then runs in fp64.
    `moving_average_decay`: the averaging instantiations (num_updates on), shadows checked against fp64 as well."""
    from dist_mnist_b200 import _native as N
    from dist_mnist_b200.parallel.config import OptimizerConfig
    avg = OptimizerConfig("sgd", 1e-2, moving_average_decay=moving_average_decay) if moving_average_decay else None
    ok = True
    dev = "cuda"
    for opt, apply_mode in ((N.OPT_SGD, N.APPLY_PER_PUSH), (N.OPT_ADAM, N.APPLY_PER_PUSH), (N.OPT_ADAM, N.APPLY_MERGED),
                            (N.OPT_SGD, N.APPLY_MERGED)):
        torch.manual_seed(5)
        n_workers, nslots, n_push = 3, 2, 2
        rows, cols, ld = 100, 784, 784
        bn = 64
        items = []
        for c0 in range(0, cols, bn):
            items.append((0 + c0, rows, min(bn, cols - c0), ld))
        small_off = rows * ld
        items.append((small_off, 1, 1110, 1110))
        arena = small_off + 1110 + 2  # deliberately not a multiple of 4 at the tail
        arena = (arena + 3) // 4 * 4
        n_items = len(items)
        params = torch.randn(arena, device=dev)
        p0 = params.clone()
        m = torch.zeros(arena, device=dev)
        v = torch.zeros(arena, device=dev)
        shadow = torch.zeros(arena, dtype=torch.bfloat16, device=dev)
        mailbox = torch.zeros(n_workers, nslots, arena, device=dev)
        flags = torch.zeros(n_workers, nslots, n_items, dtype=torch.int32, device=dev)
        next_seq = torch.ones(n_workers, n_items, dtype=torch.int32, device=dev)
        consumed = torch.zeros(n_workers, nslots, dtype=torch.int32, device=dev)
        gstep = torch.zeros(1, dtype=torch.int32, device=dev)
        done = torch.zeros(n_workers, dtype=torch.int32, device=dev)
        stop = torch.zeros(1, dtype=torch.int32, device=dev)
        exitc = torch.zeros(1, dtype=torch.int32, device=dev)
        inbox = torch.zeros(n_workers, 2, dtype=torch.int32, device=dev)
        items_t = torch.zeros(n_items, C.sizeof(N.PsItem) // 4, dtype=torch.int32, device=dev)
        host_items = (N.PsItem * n_items)()
        for i, (off, r, c, l) in enumerate(items):
            host_items[i].offset, host_items[i].rows, host_items[i].cols, host_items[i].ld = off, r, c, l
            host_items[i].flags = 1
            host_items[i].flag_index = i
        items_t.view(torch.uint8).view(-1).copy_(torch.frombuffer(bytearray(bytes(host_items)), dtype=torch.uint8).cuda())
        state = torch.zeros(n_items, 4, dtype=torch.int32, device=dev)
        st_host = (N.PsItemState * n_items)()
        for i in range(n_items):
            st_host[i].t, st_host[i].beta1_pow, st_host[i].beta2_pow = 0, 1.0, 1.0
            st_host[i].sched_step = sched_step
        state.view(torch.uint8).view(-1).copy_(torch.frombuffer(bytearray(bytes(st_host)), dtype=torch.uint8).cuda())
        # gradients: worker w push s
        grads = torch.randn(n_workers, n_push, arena, device=dev) * 0.1
        for w in range(n_workers):
            for s in range(1, n_push + 1):
                mailbox[w, s % nslots] = grads[w, s - 1]
                flags[w, s % nslots, :] = s
            done[w] = n_push + 1
        P = N.PsServeParams()
        P.params, P.adam_m, P.adam_v, P.shadow_bf16 = params.data_ptr(), m.data_ptr(), v.data_ptr(), shadow.data_ptr()
        P.items, P.item_state = items_t.data_ptr(), state.data_ptr()
        P.n_items, P.n_workers, P.nslots, P.opt, P.apply_mode = n_items, n_workers, nslots, opt, apply_mode
        P.n_flags = n_items
        P.lr, P.beta1, P.beta2, P.eps = 1e-2, 0.9, 0.999, 1e-8
        P.ieee_math = 1 if ieee else 0
        if schedule is not None:
            schedule.fill_native(P)
        ema = params.clone() if avg is not None else None
        if ema is not None:
            P.ema, P.ema_decay, P.ema_num_updates = ema.data_ptr(), avg.moving_average_decay, 1
        P.mailbox, P.arena_elems = mailbox.data_ptr(), arena
        P.flags, P.next_seq, P.consumed = flags.data_ptr(), next_seq.data_ptr(), consumed.data_ptr()
        P.global_step, P.worker_done, P.host_stop = gstep.data_ptr(), done.data_ptr(), stop.data_ptr()
        table = torch.tensor([inbox[w].data_ptr() for w in range(n_workers)], dtype=torch.int64, device=dev)
        P.inbox_table = table.data_ptr()
        P.exit_counter = exitc.data_ptr()
        torch.cuda.synchronize()
        N.check(N.lib().dm_launch_ps_serve(C.addressof(P), 8, 1, N.current_stream_ptr()), "ps_serve")
        torch.cuda.synchronize()
        # reference: with everything pre-staged, the kernel sees (w0,w1,w2) ready for seq1, then for seq2
        mask_items = torch.zeros(arena, dtype=torch.bool, device=dev)
        for (off, r, c, l) in items:
            for rr in range(r):
                mask_items[off + rr * l: off + rr * l + c] = True
        dt = torch.float32 if schedule is None and avg is None else torch.float64
        pr, mr, vr = p0.to(dt), torch.zeros_like(p0, dtype=dt), torch.zeros_like(p0, dtype=dt)
        er = p0.to(dt)
        t = 0
        for s in range(n_push):
            group = [grads[w, s].to(dt) for w in range(n_workers)]
            # (gradient, position of its first push in the application order: round-major, workers in order)
            steps = ([(sum(group), s * n_workers)] if apply_mode == N.APPLY_MERGED
                     else [(g, s * n_workers + w) for w, g in enumerate(group)])
            for gg, pos in steps:
                t += 1
                lr = P.lr if schedule is None else schedule.lr_at(sched_step + pos, P.lr)
                if opt == N.OPT_SGD:
                    pr = pr - lr * gg
                else:
                    mr = 0.9 * mr + 0.1 * gg
                    vr = 0.999 * vr + 0.001 * gg * gg
                    lr_t = lr * (1 - 0.999 ** t) ** 0.5 / (1 - 0.9 ** t)
                    pr = pr - lr_t * mr / (vr.sqrt() + 1e-8)
                if avg is not None:   # the step ends at the round's last push (merged) or at its own
                    last = s * n_workers + n_workers - 1 if apply_mode == N.APPLY_MERGED else pos
                    er = er - (er - pr) * (1.0 - avg.ema_decay_at(sched_step + last + 1))
        pr = torch.where(mask_items, pr, p0.to(dt)).float()
        e = rel_err(params, pr)
        if avg is not None:
            e = max(e, rel_err(ema, torch.where(mask_items, er, p0.to(dt))))
        e_sh = rel_err(shadow.float()[mask_items], pr[mask_items].to(torch.bfloat16).float())
        gs = int(gstep.item())
        acks = inbox[:, 0].tolist()
        good = e < 1e-5 and gs == n_workers * n_push and acks == [n_push] * n_workers and e_sh < 1e-3
        sched = ""
        if schedule is not None or avg is not None:
            steps_now = sorted({int(x) & 0xFFFFFFFF for x in state[:, 3].tolist()})
            good &= steps_now == [(sched_step + n_workers * n_push) & 0xFFFFFFFF]
            kind = schedule.kind if schedule is not None else "constant"
            sched = f" schedule={kind} from={sched_step} sched_step={steps_now}"
        if avg is not None:
            sched += f" ema={moving_average_decay} (param_err includes the shadows)"
        ok &= report(f"ps_serve opt={opt} mode={apply_mode} math={'ieee' if ieee else 'fast'}{sched}", good,
                     f"param_err={e:.1e} shadow_err={e_sh:.1e} global_step={gs} acks={acks} exit={int(exitc.item())}")
    return ok


def _ref_apply(opt, p, m, v, g, lr, t, mg=None, global_step=None):
    """One optimizer step of any kind at rate `lr` (Adam: its t-th step), on tensors in their own dtype. `mg`: centered
    RMSProp's third slot (the result is then (p, m, v, mg)); `global_step`: AdagradDA's T."""
    if opt.kind == "sgd":
        return p - lr * g, m, v
    if opt.kind == "adam":
        # the kernel's fp32 hyper-parameters: 1 - fp32(0.999) is 1.3e-5 away from 0.001 (relative), more than the bound
        b1, b2, eps = (struct.unpack("f", struct.pack("f", x))[0] for x in (opt.beta1, opt.beta2, opt.eps))
        m = b1 * m + (1 - b1) * g
        v = b2 * v + (1 - b2) * g * g
        lr_t = lr * (1 - b2 ** t) ** 0.5 / (1 - b1 ** t)
        return p - lr_t * m / (v.sqrt() + eps), m, v
    from bench_tools.gpu_e2e import tf1_apply
    return tf1_apply(dataclasses.replace(opt, lr=lr), p, m, v, g, mg=mg, global_step=global_step)


def check_ps_serve_tf1(opt, apply_mode: int, resident: bool = False, sched_step: int = 0) -> bool:
    """The serve kernel's Momentum / Adagrad / RMSProp (centered too) / Adadelta / FTRL / ProximalAdagrad /
    ProximalGradientDescent / AdagradDA instantiations (`opt`: an OptimizerConfig; `opt.math` picks the fast or the ieee one) alone, set up as `check_ps_serve`: 3 workers with 3 pushes each, staged before the launch,
    against the TF1 formulas in fp64 (parameters and both slot buffers within 1e-5 relative error; the bf16 shadow,
    global_step and the acks exact). `resident`: one pushed push per worker and pass (lookahead 1) and one vectorisable
    item of <= 4096 elements per CTA, the geometry that keeps the item's state in registers from pass to pass.
    A non-constant `opt.schedule` runs the scheduled instantiation (Adam and SGD too), every item starting at schedule
    step `sched_step`; the check then includes every item's final sched_step. `opt.moving_average_decay` runs the
    averaging instantiation (any rule, any schedule): the shadows start at the initial parameters and are checked
    against fp64 within the same bound. Centered RMSProp's third slot mg is checked like the other two. AdagradDA
    runs in the scheduled instantiation whatever the schedule: the step whose last push sits at position q has
    T = sched_step + q + 1, and the final sched_step is checked."""
    from dist_mnist_b200 import _native as N
    dev = "cuda"
    torch.manual_seed(6)
    n_workers, nslots, n_push = 3, 3, 3
    if resident:
        rows, cols, blk = 100, 256, 16
        items = [(r0 * cols, min(blk, rows - r0), cols, cols) for r0 in range(0, rows, blk)]   # 16 x 256 = 4096
        arena = rows * cols
    else:
        rows, cols, ld, bn = 100, 784, 784, 64
        items = [(c0, rows, min(bn, cols - c0), ld) for c0 in range(0, cols, bn)]
        small_off = rows * ld
        items.append((small_off, 1, 1110, 1110))           # not vectorisable: the scalar path
        arena = (small_off + 1110 + 2 + 3) // 4 * 4
    n_items = len(items)
    m0, v0 = opt.slot_init()
    params = torch.randn(arena, device=dev)
    p0 = params.clone()
    m = torch.full((arena,), m0, device=dev)
    v = torch.full((arena,), v0, device=dev)
    mg = torch.zeros(arena, device=dev) if opt.uses_mg else None
    shadow = torch.zeros(arena, dtype=torch.bfloat16, device=dev)
    mailbox = torch.zeros(n_workers, nslots, arena, device=dev)
    flags = torch.zeros(n_workers, nslots, n_items, dtype=torch.int32, device=dev)
    next_seq = torch.ones(n_workers, n_items, dtype=torch.int32, device=dev)
    consumed = torch.zeros(n_workers, nslots, dtype=torch.int32, device=dev)
    gstep = torch.zeros(1, dtype=torch.int32, device=dev)
    done = torch.zeros(n_workers, dtype=torch.int32, device=dev)
    stop = torch.zeros(1, dtype=torch.int32, device=dev)
    exitc = torch.zeros(1, dtype=torch.int32, device=dev)
    inbox = torch.zeros(n_workers, 2, dtype=torch.int32, device=dev)
    host_items = (N.PsItem * n_items)()
    for i, (off, r, c, l) in enumerate(items):
        host_items[i].offset, host_items[i].rows, host_items[i].cols, host_items[i].ld = off, r, c, l
        host_items[i].flags, host_items[i].flag_index = 1, i
    items_t = torch.frombuffer(bytearray(bytes(host_items)), dtype=torch.uint8).to(dev)
    st_host = (N.PsItemState * n_items)()
    for i in range(n_items):
        st_host[i].t, st_host[i].beta1_pow, st_host[i].beta2_pow = 0, 1.0, 1.0
        st_host[i].sched_step = sched_step
    state = torch.frombuffer(bytearray(bytes(st_host)), dtype=torch.uint8).to(dev)
    grads = torch.randn(n_workers, n_push, arena, device=dev) * 0.1
    for w in range(n_workers):
        for s in range(1, n_push + 1):
            mailbox[w, s % nslots] = grads[w, s - 1]
            flags[w, s % nslots, :] = s
        done[w] = n_push + 1
    P = N.PsServeParams()
    P.params, P.adam_m, P.adam_v, P.shadow_bf16 = params.data_ptr(), m.data_ptr(), v.data_ptr(), shadow.data_ptr()
    P.items, P.item_state = items_t.data_ptr(), state.data_ptr()
    P.n_items, P.n_workers, P.nslots, P.opt, P.apply_mode = n_items, n_workers, nslots, opt.native_kind, apply_mode
    P.n_flags = n_items
    P.lr, P.beta1, P.beta2, P.eps = opt.lr, opt.beta1, opt.beta2, opt.eps
    opt.fill_native_rule(P)
    P.mg = mg.data_ptr() if mg is not None else None
    P.ieee_math = 1 if opt.math == "ieee" else 0
    opt.schedule.fill_native(P)
    ema = params.clone() if opt.moving_averages else None
    if ema is not None:
        P.ema, P.ema_decay, P.ema_num_updates = ema.data_ptr(), opt.moving_average_decay, int(opt.moving_average_num_updates)
    P.lookahead = 1 if resident else 0
    P.mailbox, P.arena_elems = mailbox.data_ptr(), arena
    P.flags, P.next_seq, P.consumed = flags.data_ptr(), next_seq.data_ptr(), consumed.data_ptr()
    P.global_step, P.worker_done, P.host_stop = gstep.data_ptr(), done.data_ptr(), stop.data_ptr()
    table = torch.tensor([inbox[w].data_ptr() for w in range(n_workers)], dtype=torch.int64, device=dev)
    P.inbox_table = table.data_ptr()
    P.exit_counter = exitc.data_ptr()
    torch.cuda.synchronize()
    n_ctas = n_items if resident else 8
    N.check(N.lib().dm_launch_ps_serve(C.addressof(P), n_ctas, 1, N.current_stream_ptr()), "ps_serve")
    torch.cuda.synchronize()
    # reference (fp64): the kernel applies round k (the k-th push of every worker, workers in order) before round k + 1
    mask = torch.zeros(arena, dtype=torch.bool, device=dev)
    for (off, r, c, l) in items:
        for rr in range(r):
            mask[off + rr * l: off + rr * l + c] = True
    pr, mr, vr = p0.double(), torch.full((arena,), m0, dtype=torch.float64, device=dev), \
        torch.full((arena,), v0, dtype=torch.float64, device=dev)
    # push w of round k sits at position k * n_workers + w of the application order and is applied at schedule step
    # sched_step + that position; a merged round at the position of its first push
    # moving averages: the step whose last push sits at position q moves the shadows by 1 - ema_decay_at(sched_step +
    # q + 1) (fp32 decay as the kernel computes it, the update in fp64)
    er = p0.double()
    gr = torch.zeros(arena, dtype=torch.float64, device=dev) if mg is not None else None
    t = 0
    for s in range(n_push):
        group = [grads[w, s].double() for w in range(n_workers)]
        steps = ([(sum(group), s * n_workers)] if apply_mode == N.APPLY_MERGED
                 else [(g, s * n_workers + w) for w, g in enumerate(group)])
        for gg, pos in steps:
            t += 1
            last = s * n_workers + n_workers - 1 if apply_mode == N.APPLY_MERGED else pos
            # AdagradDA's T: the item's applied pushes after this step, as a uint32 like PsItemState::sched_step
            da_t = (sched_step + last + 1) & 0xFFFFFFFF if opt.kind == "adagrad_da" else None
            out = _ref_apply(opt, pr, mr, vr, gg, opt.lr_at(sched_step + pos), t, mg=gr, global_step=da_t)
            if gr is not None:
                pr, mr, vr, gr = out
            else:
                pr, mr, vr = out
            if ema is not None:
                er = er - (er - pr) * (1.0 - opt.ema_decay_at(sched_step + last + 1))
    pr, mr, vr = torch.where(mask, pr, p0.double()), torch.where(mask, mr, m0), torch.where(mask, vr, v0)
    e_p, e_m, e_v = rel_err(params, pr), rel_err(m, mr), rel_err(v, vr)
    e_g = rel_err(mg, torch.where(mask, gr, 0.0)) if mg is not None else 0.0
    e_e = rel_err(ema, torch.where(mask, er, p0.double())) if ema is not None else 0.0
    shadow_exact = bool(torch.equal(shadow[mask], params[mask].to(torch.bfloat16)))
    gs = int(gstep.item())
    acks = inbox[:, 0].tolist()
    good = (max(e_p, e_m, e_v, e_e, e_g) < 1e-5 and shadow_exact and gs == n_workers * n_push
            and acks == [n_push] * n_workers and int(exitc.item()) == n_ctas)
    name = (f"ps_serve {opt.kind}{' nesterov' if opt.use_nesterov else ''}{' centered' if opt.centered else ''} "
            f"momentum={opt.momentum} math={opt.math} mode={apply_mode} resident={resident}")
    if opt.kind in ("adadelta", "ftrl", "proximal_adagrad", "proximal_sgd", "adagrad_da"):
        name += (f" rho={opt.rho} l1={opt.l1_regularization_strength} l2={opt.l2_regularization_strength} "
                 f"shrinkage={opt.l2_shrinkage_regularization_strength} lr_power={opt.learning_rate_power} "
                 f"accum0={opt.initial_accumulator_value}")
    extra = f" mg={e_g:.1e}" if mg is not None else ""
    if not opt.schedule.constant or ema is not None or opt.kind == "adagrad_da":
        steps_now = sorted({int(x) & 0xFFFFFFFF for x in state.view(torch.int32).view(n_items, 4)[:, 3].tolist()})
        good &= steps_now == [(sched_step + n_workers * n_push) & 0xFFFFFFFF]
        name += f" schedule={opt.schedule.kind} from={sched_step}"
        extra += f" sched_step={steps_now}"
    if ema is not None:
        name += f" ema={opt.moving_average_decay} num_updates={opt.moving_average_num_updates}"
        extra += f" err ema={e_e:.1e}"
    return report(name, good, f"err p={e_p:.1e} m={e_m:.1e} v={e_v:.1e} shadow_exact={shadow_exact} global_step={gs} "
                              f"acks={acks} exit={int(exitc.item())}{extra}")


def check_dense_apply() -> bool:
    from dist_mnist_b200 import _native as N
    ok = True
    n = 100003
    torch.manual_seed(1)
    p = torch.randn(n, device="cuda")
    g = torch.randn(n, device="cuda")
    for opt in (N.OPT_SGD, N.OPT_ADAM):
        pp, m, v = p.clone(), torch.zeros_like(p), torch.zeros_like(p)
        ref = torch.nn.Parameter(p.clone())
        o = torch.optim.SGD([ref], lr=1e-2) if opt == N.OPT_SGD else torch.optim.Adam([ref], lr=1e-2, eps=1e-8)
        for t in range(1, 4):
            N.check(N.lib().dm_launch_dense_apply(pp.data_ptr(), m.data_ptr(), v.data_ptr(), g.data_ptr(), None, n, opt,
                                                  1e-2, 0.9, 0.999, 1e-8, t, N.current_stream_ptr()))
            ref.grad = g.clone()
            o.step()
        torch.cuda.synchronize()
        e = rel_err(pp, ref.detach())
        # TF and torch Adam differ only in where epsilon enters; 1e-8 is negligible at these magnitudes
        ok &= report(f"dense_apply opt={opt}", e < 1e-4, f"rel_err vs torch.optim={e:.1e}")
    return ok


def check_p2p_local() -> bool:
    from dist_mnist_b200 import _native as N
    ok = True
    for mode in (0, 1):
        for nbytes in (1024, 16384 * 3 + 4096, 1 << 22):
            src = torch.randint(0, 255, (nbytes,), dtype=torch.uint8, device="cuda")
            dst = torch.zeros_like(src)
            flag = torch.zeros(1, dtype=torch.int32, device="cuda")
            N.check(N.lib().dm_launch_p2p_copy(dst.data_ptr(), src.data_ptr(), nbytes, mode, 8, flag.data_ptr(), 0,
                                               N.current_stream_ptr()))
            torch.cuda.synchronize()
            good = bool((src == dst).all()) and int(flag.item()) == 8
            ok &= report(f"p2p_copy mode={mode} bytes={nbytes}", good, f"flag={int(flag.item())}")
    return ok


CHECKS = {
    "gemm_fwd": check_gemm_fwd, "gemm_dw": check_gemm_dw, "gemm_dx": check_gemm_dx, "head": check_head,
    "accuracy": check_accuracy, "ps_serve": check_ps_serve, "dense_apply": check_dense_apply,
    "p2p_local": check_p2p_local,
}


def main(argv) -> int:
    which = argv[0] if argv else "all"
    if which == "all":
        rc = 0
        for g in GROUPS:
            t0 = time.time()
            print(f"===== {g} =====", flush=True)
            try:
                r = subprocess.run([sys.executable, "-m", "bench_tools.gpu_check", g], timeout=300)
                code = r.returncode
            except subprocess.TimeoutExpired:
                code = 124
            print(f"===== {g}: exit {code} ({time.time() - t0:.1f}s) =====", flush=True)
            rc |= int(code != 0)
        return rc
    try:
        ok = CHECKS[which]()
    except Exception:
        traceback.print_exc()
        ok = False
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main(sys.argv[1:]))
