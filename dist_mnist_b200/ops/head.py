"""Launch plan for the fused classifier head (csrc/head_sm90.cu): last dense layer + softmax + loss +
accuracy + small-variable gradients + their parameter-server push.

Reference parity: /root/reference/distributed_server-basic.py:52-53 (book loss), :35 (xent loss),
and the gradient ops `minimize` builds for them at :103.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Optional

import torch

from .. import _native as N
from .gemm import null_push

HEAD_SLICE = 128
MAX_CLASSES = 16
MAX_BATCH = 256


@dataclass
class HeadPlan:
    params: N.HeadParams
    name: str = "head"

    def launch(self, stream: Optional[int] = None) -> None:
        s = N.current_stream_ptr() if stream is None else stream
        N.ensure_prepared()
        N.check(N.lib().dm_launch_head(C.addressof(self.params), s), f"launch {self.name}")


def head_plan(*, h_ptr: int, labels_ptr: int, w_last_ptr: int, b_last_ptr: int, dpre_ptr: int, result_ptr: int,
              B: int, B_pad: int, H: int, num_classes: int, loss_kind: int, act_bf16: bool,
              push: Optional[N.PushTarget] = None, push_bh: Optional[N.PushTarget] = None,
              push_bl: Optional[N.PushTarget] = None,
              off_w_last: int = 0, off_b_last: int = 0, off_b_hidden: int = 0,
              item_w_last_base: int = 0, item_b_last: int = 0, item_b_hidden_base: int = 0,
              seq_ptr: int = 0, inbox_ptr: int = 0, n_inbox: int = 0, ps_global_step_ptr: int = 0,
              nslots: int = 1, compute_grads: bool = True, ldh: Optional[int] = None) -> HeadPlan:
    assert num_classes <= MAX_CLASSES and B <= B_pad <= MAX_BATCH
    p = N.HeadParams()
    p.B, p.B_pad, p.H, p.C = B, B_pad, H, num_classes
    p.loss_kind = loss_kind
    p.act_bf16 = int(act_bf16)
    p.ldh = H if ldh is None else ldh
    p.compute_grads = int(compute_grads)
    p.h, p.labels, p.w_last, p.b_last, p.dpre = h_ptr, labels_ptr, w_last_ptr, b_last_ptr, dpre_ptr
    p.push = push if push is not None else null_push()
    p.push_bh = push_bh if push_bh is not None else p.push
    p.push_bl = push_bl if push_bl is not None else p.push
    p.off_w_last, p.off_b_last, p.off_b_hidden = off_w_last, off_b_last, off_b_hidden
    p.item_w_last_base, p.item_b_last, p.item_b_hidden_base = item_w_last_base, item_b_last, item_b_hidden_base
    p.result = result_ptr
    p.seq_ptr = seq_ptr
    p.inbox = inbox_ptr
    p.n_inbox = n_inbox
    p.ps_global_step = ps_global_step_ptr
    p.nslots = nslots
    return HeadPlan(p)


def head_slices(H: int) -> int:
    return (H + HEAD_SLICE - 1) // HEAD_SLICE


def accuracy_count(logits: torch.Tensor, labels: torch.Tensor) -> torch.Tensor:
    """Hand-written argmax-compare-count reduction (SURVEY K12). Returns a 1-element uint32-as-int32 tensor."""
    assert logits.is_cuda and logits.dtype == torch.float32 and labels.dtype == torch.float32
    assert logits.is_contiguous() and labels.is_contiguous() and logits.shape == labels.shape
    out = torch.zeros(1, dtype=torch.int32, device=logits.device)
    B, Cn = logits.shape
    N.check(
        N.lib().dm_launch_accuracy(logits.data_ptr(), labels.data_ptr(), B, Cn, out.data_ptr(), N.current_stream_ptr()),
        "launch accuracy",
    )
    return out
