"""Python launch plans for the wgmma dense-layer GEMM (csrc/gemm_sm90.cu).

A `GemmPlan` freezes the TMA tensor maps and the parameter block of one launch; `plan.launch()` enqueues
it on the current CUDA stream, so plans can be replayed inside a CUDA graph. The three constructors map
the MLP's three GEMM roles onto the kernel's operand layouts (all tensors stay row-major):

    forward : out[b, o] = act(sum_i x[b, i] W[o, i] + bias[o])        W may be an NVLink peer pointer
    dW      : dW[o, i]  = sum_b dy[b, o] x[b, i]                      epilogue = gradient push
    dX      : dx[b, i]  = (sum_o dy[b, o] W[o, i]) * (h[b, i] > 0)    W may be an NVLink peer pointer

Reference parity: MatMul / BiasAdd / Relu and their gradients at
/root/reference/distributed_server-basic.py:49-52,103.
"""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import dataclass
from typing import Optional

from .. import _native as N

TILE_M = 128
SMEM_BUDGET = 200 * 1024
MAX_STAGES = 8


def elem_size(dtype: int) -> int:
    return 4 if dtype == N.DT_F32 else 2


def bke(dtype: int) -> int:
    """k elements per 128-byte stage chunk (32 for fp32/tf32, 64 for bf16)."""
    return 128 // elem_size(dtype)


def ceil_div(a: int, b: int) -> int:
    return (a + b - 1) // b


def round_up(a: int, b: int) -> int:
    return ceil_div(a, b) * b


def padded_ld(n: int) -> int:
    """Leading dimension for a row of n elements such that the row stride is a multiple of 16 bytes for
    both fp32 and bf16 (TMA requirement): round up to 8 elements."""
    return round_up(n, 8)


def local_push(base_ptr: int) -> N.PushTarget:
    t = N.PushTarget()
    t.mode = N.PUSH_LOCAL
    t.scale = 1.0
    t.base = base_ptr
    t.nslots = 1
    return t


def null_push() -> N.PushTarget:
    return local_push(0)


@dataclass
class GemmPlan:
    tm_a: object
    tm_b: object
    params: N.GemmParams
    dtype: int
    a_mn: bool
    b_mn: bool
    splits: int
    grid: tuple
    name: str = "gemm"
    scratch: object = None    # split-K partial tiles (kept alive with the plan)
    counters: object = None

    def launch(self, stream: Optional[int] = None) -> None:
        s = N.current_stream_ptr() if stream is None else stream
        N.ensure_prepared()
        N.check(
            N.lib().dm_launch_gemm(
                C.addressof(self.tm_a), C.addressof(self.tm_b), C.addressof(self.params), self.dtype,
                int(self.a_mn), int(self.b_mn), self.splits, s,
            ),
            f"launch {self.name}",
        )

    @property
    def smem_bytes(self) -> int:
        return N.lib().dm_gemm_smem_bytes(self.params.bn, self.params.stages, int(self.params.splitk_cluster))


def _pick_stages(bn: int, kc: int, budget: int = SMEM_BUDGET) -> int:
    stage = TILE_M * 128 + bn * 128
    return max(1, min(MAX_STAGES, kc, budget // stage))


def auto_splits(K: int, dtype: int, mtiles: int) -> int:
    """Split-K factor for the K-loop GEMMs (forward, dX). One CTA streams its K loop one 128-byte-wide TMA box
    per operand and k-chunk, so a long K loop on one SM is latency bound. The loop is therefore spread over up
    to 8 CTAs (~3-4 k-chunks each) whose fp32 partial tiles are summed by the last-arriving CTA in a single
    round of independent L2 loads."""
    kc = ceil_div(K, bke(dtype))
    return max(1, min(8, ceil_div(kc, 3), max(1, 96 // max(1, mtiles))))


def cluster_splits(K: int, dtype: int) -> int:
    """Cluster size (power of two <= 8) for the DSMEM split-K: ~3-4 k-chunks per CTA."""
    kc = ceil_div(K, bke(dtype))
    if kc >= 16:
        return 8
    if kc >= 8:
        return 4
    if kc >= 4:
        return 2
    return 1


def splitk_mode(bn: int) -> str:
    """'cluster' (thread-block cluster + distributed shared memory reduce-scatter, bn <= 64) or 'global'."""
    mode = os.environ.get("DM_SPLITK", "cluster")
    return mode if (mode != "cluster" or bn <= 64) else "global"


def _attach_splitk(plan: "GemmPlan", mtiles: int, splits: int, bn: int) -> None:
    if splits <= 1 or plan.params.splitk_cluster:
        return
    import torch

    dev = torch.device("cuda", torch.cuda.current_device())
    plan.scratch = torch.zeros(mtiles * splits * TILE_M * bn, dtype=torch.float32, device=dev)
    plan.counters = torch.zeros(mtiles, dtype=torch.int32, device=dev)
    plan.params.splitk_scratch = plan.scratch.data_ptr()
    plan.params.splitk_counter = plan.counters.data_ptr()


def _base_params(M, N_, K, bn, dtype, splits) -> N.GemmParams:
    p = N.GemmParams()
    p.M, p.N, p.K = M, N_, K
    p.bn = bn
    kc_total = ceil_div(K, bke(dtype))
    p.kc_per_split = ceil_div(kc_total, splits)
    p.stages = _pick_stages(bn, p.kc_per_split)
    p.colsum = null_push()
    p.push = null_push()
    p.has_colsum = 0
    return p


def forward_plan(*, w_ptr: int, x_ptr: int, out_ptr: int, bias_ptr: int, O: int, I: int, B: int, B_pad: int,
                 dtype: int, relu: bool, ldw: Optional[int] = None, ldx: Optional[int] = None,
                 ldo: Optional[int] = None, bump_seq_ptr: int = 0, seq_counter_ptr: int = 0, splits: Optional[int] = None,
                 name: str = "fwd") -> GemmPlan:
    """out[b, o] = act(x[b, :] . W[o, :] + bias[o]); A = W (K-major, may be peer), B = x (K-major)."""
    assert B_pad % 16 == 0 and B_pad <= 256 and B <= B_pad
    es = elem_size(dtype)
    ldw = I if ldw is None else ldw
    ldx = I if ldx is None else ldx
    ldo = O if ldo is None else ldo
    k = bke(dtype)
    tm_a = N.make_tensor_map(w_ptr, dtype, I, O, ldw * es, k, TILE_M)
    tm_b = N.make_tensor_map(x_ptr, dtype, I, B_pad, ldx * es, k, B_pad)
    mtiles = ceil_div(O, TILE_M)
    cluster = splitk_mode(B_pad) == "cluster"
    if splits is None:
        splits = cluster_splits(I, dtype) if cluster else auto_splits(I, dtype, mtiles)
    cluster = cluster and 1 < splits <= 8
    p = _base_params(O, B, I, B_pad, dtype, splits)
    if not cluster or os.environ.get("DM_CLUSTER_TRIM", "0") == "1":
        splits = ceil_div(ceil_div(I, k), p.kc_per_split)  # drop empty trailing splits
    p.splitk_cluster = int(cluster and splits > 1)
    p.epi = N.EPI_TRANSPOSED
    p.out = out_ptr
    p.out_bf16 = int(dtype == N.DT_BF16)
    p.ldo = ldo
    p.bias = bias_ptr
    p.relu = int(relu)
    p.bump_seq = bump_seq_ptr
    p.seq_counter = seq_counter_ptr or bump_seq_ptr
    grid = (mtiles, 1, splits)
    plan = GemmPlan(tm_a, tm_b, p, dtype, False, False, splits, grid, name)
    _attach_splitk(plan, mtiles, splits, B_pad)
    return plan


def dw_plan(*, dy_ptr: int, x_ptr: int, O: int, I: int, B_pad: int, dtype: int, push: N.PushTarget,
            push_offset: int, item_base: int = 0, bn: int = 64, lddy: Optional[int] = None,
            ldx: Optional[int] = None, ldw: Optional[int] = None, name: str = "dw") -> GemmPlan:
    """dW[o, i] = sum_b dy[b, o] x[b, i]; A = dy (MN-major), B = x (MN-major); epilogue pushes dW rows."""
    es = elem_size(dtype)
    k = bke(dtype)
    assert bn % k == 0 and bn <= 256, "MN-major B tile must be whole 128-byte slabs"
    lddy = O if lddy is None else lddy
    ldx = I if ldx is None else ldx
    tm_a = N.make_tensor_map(dy_ptr, dtype, O, B_pad, lddy * es, k, k)
    tm_b = N.make_tensor_map(x_ptr, dtype, I, B_pad, ldx * es, k, k)
    p = _base_params(O, I, B_pad, bn, dtype, 1)
    # the kernel keeps a K-major copy of the MN-major B tile (bn rows x 128 B, + 1 KB alignment) beside the ring
    p.stages = _pick_stages(bn, p.kc_per_split, SMEM_BUDGET - (bn * 128 + 1024))
    p.epi = N.EPI_ROWMAJOR_PUSH
    p.ldo = I if ldw is None else ldw
    p.push = push
    p.push_offset = push_offset
    p.push_item_base = item_base
    p.push_staged = int(os.environ.get("DM_PUSH_STAGED", "0") == "1")
    grid = (ceil_div(O, TILE_M), ceil_div(I, bn), 1)
    return GemmPlan(tm_a, tm_b, p, dtype, True, True, 1, grid, name)


def dw_tiles(O: int, I: int, bn: int = 64):
    """Tile decomposition the dW epilogue publishes flags for: list of (row0, rows, col0, cols)."""
    out = []
    for mt in range(ceil_div(O, TILE_M)):
        for nt in range(ceil_div(I, bn)):
            out.append((mt * TILE_M, min(TILE_M, O - mt * TILE_M), nt * bn, min(bn, I - nt * bn)))
    return out


def dx_plan(*, w_ptr: int, dy_ptr: int, out_ptr: int, mask_ptr: int, O: int, I: int, B: int, B_pad: int,
            dtype: int, ldw: Optional[int] = None, lddy: Optional[int] = None, ldo: Optional[int] = None,
            colsum: Optional[N.PushTarget] = None, colsum_offset: int = 0, colsum_item_base: int = 0,
            splits: Optional[int] = None, name: str = "dx") -> GemmPlan:
    """dx[b, i] = (dy[b, :] . W[:, i]) * (mask[b, i] > 0); A = W (MN-major, may be peer), B = dy (K-major)."""
    assert B_pad % 16 == 0 and B_pad <= 256
    es = elem_size(dtype)
    k = bke(dtype)
    ldw = I if ldw is None else ldw
    lddy = O if lddy is None else lddy
    ldo = I if ldo is None else ldo
    tm_a = N.make_tensor_map(w_ptr, dtype, I, O, ldw * es, k, k)
    tm_b = N.make_tensor_map(dy_ptr, dtype, O, B_pad, lddy * es, k, B_pad)
    mtiles = ceil_div(I, TILE_M)
    cluster = splitk_mode(B_pad) == "cluster"
    if splits is None:
        splits = cluster_splits(O, dtype) if cluster else auto_splits(O, dtype, mtiles)
    cluster = cluster and 1 < splits <= 8
    p = _base_params(I, B, O, B_pad, dtype, splits)
    if not cluster or os.environ.get("DM_CLUSTER_TRIM", "0") == "1":
        splits = ceil_div(ceil_div(O, k), p.kc_per_split)
    p.splitk_cluster = int(cluster and splits > 1)
    p.epi = N.EPI_TRANSPOSED
    p.out = out_ptr
    p.out_bf16 = int(dtype == N.DT_BF16)
    p.ldo = ldo
    p.mask = mask_ptr
    p.ldmask = ldo
    p.mask_bf16 = int(dtype == N.DT_BF16)
    if colsum is not None:
        p.colsum = colsum
        p.colsum_offset = colsum_offset
        p.colsum_item_base = colsum_item_base
        p.has_colsum = 1
    grid = (mtiles, 1, splits)
    plan = GemmPlan(tm_a, tm_b, p, dtype, True, False, splits, grid, name)
    _attach_splitk(plan, mtiles, splits, B_pad)
    return plan
