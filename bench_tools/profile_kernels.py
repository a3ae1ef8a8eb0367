"""Stand-alone launcher of one worker step's kernels (+ one PS apply pass) for ncu.

The persistent PS kernel cannot run under ncu (ncu serialises and replays kernels; a kernel that waits for
another kernel's flags would never finish), so this script launches the *same* kernels with the same launch
plans against local buffers standing in for the PS shard:

    fwd0   wgmma forward GEMM     (W "pulled" by TMA, +bias, relu)
    head   fused softmax-CE head  (mailbox push of dW_last / db)
    dw0    wgmma dW GEMM          (epilogue = mailbox push + per-tile flags)
    ps     ps_serve_kernel        (flags pre-staged by the step above; exits after applying that one push)

    ncu --metrics gpu__time_duration.sum --clock-control none -s 20 -c 40 --csv --log-file profiles/launches.csv \
        python -m bench_tools.profile_kernels --model book --iters 15
    ncu --set full --clock-control none --import-source on -k regex:gemm_wgmma -s 6 -c 3 -o profiles/prof_gemm \
        python -m bench_tools.profile_kernels --model book --iters 6
"""
from __future__ import annotations

import argparse
import ctypes as C

import torch

from dist_mnist_b200 import _native as N
from dist_mnist_b200.models import mlp
from dist_mnist_b200.ops import gemm, head
from dist_mnist_b200.parallel import sharding


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="book")
    ap.add_argument("--dtype", default="fp32")
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--opt", default="adam")
    ap.add_argument("--time", action="store_true", help="CUDA-event timing of each kernel (not under ncu)")
    ap.add_argument("--graph_time", action="store_true", help="per-kernel time from CUDA-graph replays (warm caches)")
    ap.add_argument("--push", default="mailbox", choices=["mailbox", "local", "atomic"])
    ap.add_argument("--phases", action="store_true", help="print in-kernel phase timestamps of the GEMM kernels")
    ap.add_argument("--fwd_splits", type=int, default=None)
    ap.add_argument("--pdl", action="store_true", help="programmatic dependent launch for every kernel but the first")
    args = ap.parse_args()
    dev = "cuda"
    spec = mlp.get_model(args.model)
    lay = sharding.build_layout(spec, 1, dw_tile_n=sharding.dw_tile_n_for(args.dtype))
    sh = lay.shards[0]
    dt = N.DT_F32 if args.dtype == "fp32" else N.DT_BF16
    tdt = torch.float32 if args.dtype == "fp32" else torch.bfloat16
    B = args.batch
    B_pad = gemm.round_up(B, 16)
    nslots, n_items, arena = 2, sh.n_items, sh.arena_elems
    params = torch.zeros(arena, device=dev)
    init = mlp.init_params(spec, 0)
    for name, vl in lay.by_name.items():
        t = init[name]
        if t.dim() == 2:
            params[vl.offset: vl.offset + vl.rows * vl.ld].view(vl.rows, vl.ld)[:, :vl.cols] = t.to(dev)
        else:
            params[vl.offset: vl.offset + vl.cols] = t.to(dev)
    shadow = params.to(torch.bfloat16)
    m, v = torch.zeros_like(params), torch.zeros_like(params)
    mailbox = torch.zeros(1, nslots, arena, device=dev)
    flags = torch.zeros(1, nslots, n_items, dtype=torch.int32, device=dev)
    seq = torch.zeros(1, dtype=torch.int32, device=dev)
    names, sizes = spec.variable_names(), spec.layer_sizes
    L = len(sizes)
    ld_in = gemm.padded_ld(spec.in_features)
    x = torch.rand(B_pad, ld_in, device=dev).to(tdt)
    y = torch.zeros(B_pad, spec.num_classes, device=dev)
    y[torch.arange(B), torch.randint(0, spec.num_classes, (B,))] = 1
    act = [None] + [torch.zeros(B_pad, gemm.padded_ld(sizes[l][1]), dtype=tdt, device=dev) for l in range(L - 1)]
    dact = [None] + [torch.zeros_like(a) for a in act[1:]]
    res = torch.zeros(4, dtype=torch.int32, device=dev)

    def wptr(vl):
        return (shadow.data_ptr() + vl.offset * 2) if dt == N.DT_BF16 else (params.data_ptr() + vl.offset * 4)

    push = N.PushTarget()
    push.mode, push.scale, push.base, push.slot_stride = N.PUSH_MAILBOX, 1.0, mailbox.data_ptr(), arena
    push.flags, push.flag_slot_stride, push.nslots, push.seq_ptr = flags.data_ptr(), n_items, nslots, seq.data_ptr()
    if args.push == "local":
        push.mode = N.PUSH_LOCAL
    elif args.push == "atomic":
        push.mode, push.scale, push.base = N.PUSH_ATOMIC, -1e-4, params.data_ptr()

    plans = []
    for l in range(L - 1):
        wl, bl = lay.by_name[names[l][0]], lay.by_name[names[l][1]]
        fin, fout = sizes[l]
        plans.append(gemm.forward_plan(w_ptr=wptr(wl), x_ptr=x.data_ptr() if l == 0 else act[l].data_ptr(),
                                       out_ptr=act[l + 1].data_ptr(), bias_ptr=params.data_ptr() + bl.offset * 4,
                                       O=fout, I=fin, B=B, B_pad=B_pad, dtype=dt, act=N.ACT_RELU, ldw=wl.ld,
                                       ldx=ld_in if l == 0 else act[l].shape[1], ldo=act[l + 1].shape[1],
                                       bump_seq_ptr=seq.data_ptr() if l == 0 else 0, splits=args.fwd_splits,
                                       name=f"fwd{l}"))
    wl, bl = lay.by_name[names[L - 1][0]], lay.by_name[names[L - 1][1]]
    hb = lay.by_name[names[L - 2][1]]
    plans.append(head.head_plan(h_ptr=act[L - 1].data_ptr(), labels_ptr=y.data_ptr(),
                                w_last_ptr=params.data_ptr() + wl.offset * 4, b_last_ptr=params.data_ptr() + bl.offset * 4,
                                dpre_ptr=dact[L - 1].data_ptr(), result_ptr=res.data_ptr(), B=B, B_pad=B_pad,
                                H=sizes[L - 1][0], num_classes=spec.num_classes,
                                loss_kind=N.LOSS_BOOK if spec.loss == "book" else N.LOSS_XENT,
                                act_bf16=dt == N.DT_BF16, push=push, push_bh=push, push_bl=push,
                                off_w_last=wl.offset, off_b_last=bl.offset, off_b_hidden=hb.offset,
                                item_w_last_base=wl.item_base, item_b_last=bl.item_base,
                                item_b_hidden_base=hb.item_base, seq_ptr=seq.data_ptr(), nslots=nslots,
                                ldh=act[L - 1].shape[1]))
    for l in range(L - 2, -1, -1):
        wl = lay.by_name[names[l][0]]
        fin, fout = sizes[l]
        if l > 0:   # dX before dW of the same layer (see Worker._build_cuda)
            pb = lay.by_name[names[l - 1][1]]
            plans.append(gemm.dx_plan(w_ptr=wptr(wl), dy_ptr=dact[l + 1].data_ptr(), out_ptr=dact[l].data_ptr(),
                                      mask_ptr=act[l].data_ptr(), O=fout, I=fin, B=B, B_pad=B_pad, dtype=dt, act=N.ACT_RELU,
                                      ldw=wl.ld, lddy=dact[l + 1].shape[1], ldo=dact[l].shape[1], colsum=push,
                                      colsum_offset=pb.offset, colsum_item_base=pb.item_base, name=f"dx{l}"))
        plans.append(gemm.dw_plan(dy_ptr=dact[l + 1].data_ptr(), x_ptr=x.data_ptr() if l == 0 else act[l].data_ptr(),
                                  O=fout, I=fin, B_pad=B_pad, dtype=dt, push=push, push_offset=wl.offset,
                                  item_base=wl.item_base, bn=lay.dw_tile_n, lddy=dact[l + 1].shape[1],
                                  ldx=ld_in if l == 0 else act[l].shape[1], ldw=wl.ld, name=f"dw{l}"))

        plans[0].name = "fwd0+head"
        del plans[1]
    if args.pdl:
        for p_ in plans[1:]:
            p_.params.pdl = 1

    # PS serve kernel configured for one worker; `worker_done` is advanced every iteration so that each launch
    # applies exactly the push that the step just published and then exits.
    items = (N.PsItem * n_items)()
    for i, it in enumerate(sh.items):
        items[i].offset, items[i].rows, items[i].cols, items[i].ld = it.offset, it.rows, it.cols, it.ld
        items[i].flags = 1 if (it.shadow and dt == N.DT_BF16) else 0
        items[i].flag_index = i
    items_t = torch.frombuffer(bytearray(bytes(items)), dtype=torch.uint8).cuda()
    st = (N.PsItemState * n_items)()
    for i in range(n_items):
        st[i].t, st[i].beta1_pow, st[i].beta2_pow = 0, 1.0, 1.0
    state_t = torch.frombuffer(bytearray(bytes(st)), dtype=torch.uint8).cuda()
    next_seq = torch.ones(1, n_items, dtype=torch.int32, device=dev)
    consumed = torch.zeros(1, nslots, dtype=torch.int32, device=dev)
    ctrl = torch.zeros(64, dtype=torch.int32, device=dev)
    inbox = torch.zeros(2, dtype=torch.int32, device=dev)
    table = torch.tensor([inbox.data_ptr()], dtype=torch.int64, device=dev)
    P = N.PsServeParams()
    P.params, P.adam_m, P.adam_v = params.data_ptr(), m.data_ptr(), v.data_ptr()
    P.shadow_bf16 = shadow.data_ptr() if dt == N.DT_BF16 else None
    P.items, P.item_state = items_t.data_ptr(), state_t.data_ptr()
    P.n_items, P.n_workers, P.nslots = n_items, 1, nslots
    P.n_flags = n_items
    P.opt, P.apply_mode = (N.OPT_ADAM if args.opt == "adam" else N.OPT_SGD), N.APPLY_PER_PUSH
    P.lr, P.beta1, P.beta2, P.eps = 1e-4, 0.9, 0.999, 1e-8
    P.mailbox, P.arena_elems = mailbox.data_ptr(), arena
    P.flags, P.next_seq, P.consumed = flags.data_ptr(), next_seq.data_ptr(), consumed.data_ptr()
    P.global_step, P.host_stop, P.exit_counter = ctrl.data_ptr(), ctrl.data_ptr() + 4, ctrl.data_ptr() + 8
    P.worker_done, P.inbox_table = ctrl.data_ptr() + 64, table.data_ptr()
    done_view = ctrl[16:17]

    if args.phases:
        ts = torch.zeros(16 + 2 * 120, dtype=torch.int64, device=dev)
        names_ph = ["entry", "prologue done", "1st stage TMA issued", "1st full barrier", "last MMA committed",
                    "tmem_full seen", "-", "epilogue done", "exit"]
        for p_ in plans:
            if not hasattr(p_, "tm_a"):
                p_.params.debug_ts = ts.data_ptr()
                for _ in range(3):
                    p_.launch(N.current_stream_ptr())
                torch.cuda.synchronize()
                t = ts.tolist()
                lab = ["seq+ack", "staged (A)", "logits+softmax (B+C)", "grads (D)", "pushed+sync", "flags out"]
                print("head: " + "  ".join(f"{lab[i - 1]}=+{t[i] - t[0]}" for i in range(1, 7)) + " (SM cycles)")
                p_.params.debug_ts = None
                continue
            p_.params.debug_ts = ts.data_ptr()
            for _ in range(3):
                p_.launch(N.current_stream_ptr())
            torch.cuda.synchronize()
            t = ts.tolist()
            print(f"{p_.name}: grid={p_.grid} stages={p_.params.stages} " + "  ".join(
                f"{names_ph[i]}=+{t[i] - t[0]}" for i in (1, 2, 3, 4, 5, 7, 8)) + " (SM cycles)")
            ncta = min(120, p_.grid[0] * p_.grid[1] * p_.grid[2])
            ent = [t[16 + 2 * i] for i in range(ncta)]
            ext = [t[17 + 2 * i] for i in range(ncta)]
            base = min(ent)
            print("    per-CTA wall clock (ns since first entry): entry " + " ".join(str(e - base) for e in ent))
            print("                                               exit  " + " ".join(str(e - base) for e in ext))
            # two launches back to back: gap between the first kernel's last exit and the second kernel's first entry
            ts.zero_()
            p_.launch(N.current_stream_ptr())
            torch.cuda.synchronize()
            first_exit = max(ts.tolist()[17 + 2 * i] for i in range(ncta))
            ts.zero_()
            g = torch.cuda.CUDAGraph()
            s_ = torch.cuda.Stream()
            with torch.cuda.stream(s_):
                p_.launch(s_.cuda_stream)
                s_.synchronize()
                with torch.cuda.graph(g, stream=s_):
                    p_.launch(s_.cuda_stream)
                    p_.launch(s_.cuda_stream)
                    p_.launch(s_.cuda_stream)
                ts.zero_()
                s_.synchronize()
                g.replay()
                s_.synchronize()
            t2 = ts.tolist()
            ent = [t2[16 + 2 * i] for i in range(ncta)]
            ext = [t2[17 + 2 * i] for i in range(ncta)]
            print(f"    graph of 3 launches, last launch: first entry..last exit = {max(ext) - min(ent)} ns")
            p_.params.debug_ts = None
        return 0

    if args.graph_time:
        # warm-cache per-kernel time: R back-to-back launches of one plan inside a CUDA graph (no host launch
        # overhead, same-stream serialisation), timed with events around the replay.
        R = 20
        s = torch.cuda.Stream()
        done_view.fill_(2)
        results = []
        with torch.cuda.stream(s):
            for p in plans:
                p.launch(s.cuda_stream)  # warm-up + lazy load
            s.synchronize()
            for p in plans:
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g, stream=s):
                    for _ in range(R):
                        p.launch(s.cuda_stream)
                g.replay()
                s.synchronize()
                t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                t0.record(s)
                for _ in range(5):
                    g.replay()
                t1.record(s)
                t1.synchronize()
                results.append((p.name, t0.elapsed_time(t1) * 1e3 / (5 * R)))
            # whole step as one graph (what the executor replays), without the PS
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=s):
                for p in plans:
                    p.launch(s.cuda_stream)
            g.replay()
            s.synchronize()
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record(s)
            for _ in range(50):
                g.replay()
            t1.record(s)
            t1.synchronize()
            results.append(("step graph", t0.elapsed_time(t1) * 1e3 / 50))
        print(f"model={args.model} dtype={args.dtype} B={B} graph-replayed kernel times (warm caches, incl. ~1 us launch gap):")
        for name, us in results:
            print(f"  {name:12s} {us:8.2f} us")
        return 0

    stream = N.current_stream_ptr()
    evs = None
    if args.time:
        evs = [[torch.cuda.Event(enable_timing=True) for _ in range(len(plans) + 2)] for _ in range(args.iters)]
    for it in range(args.iters):
        done_view.fill_(it + 2)  # "the worker left after push it+1": the serve kernel exits once it is applied
        if evs:
            evs[it][0].record()
        for j, p in enumerate(plans):
            p.launch(stream)
            if evs:
                evs[it][j + 1].record()
        N.check(N.lib().dm_launch_ps_serve(C.addressof(P), min(32, n_items), 1, stream), "ps_serve")
        if evs:
            evs[it][len(plans) + 1].record()
    torch.cuda.synchronize()
    loss = res[:1].view(torch.float32).item()
    print(f"model={args.model} dtype={args.dtype} B={B}: {len(plans)} step kernels + ps_serve x {args.iters} iterations; "
          f"loss={loss:.5f} global_step={int(ctrl[0])} acked={int(inbox[0])}")
    if evs:
        labels = [p.name for p in plans] + ["ps_serve"]
        for j, lab in enumerate(labels):
            ts = sorted(evs[it][j].elapsed_time(evs[it][j + 1]) * 1e3 for it in range(2, args.iters))
            print(f"  {lab:10s} median {ts[len(ts) // 2]:8.2f} us   min {ts[0]:8.2f} us (event-to-event, includes launch gap)")
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
