"""Variable -> parameter-server placement and the per-shard memory layout.

Reference parity: `tf.device(tf.train.replica_device_setter(worker_device=..., cluster=cluster))`
(/root/reference/distributed_server-basic.py:88-89) pins every Variable — `global_step` first (DS:91), then the
model variables in creation order (DS:41-47), with the Adam slots colocated — to ps tasks round-robin, whole
variables only. `strategy="round_robin"` reproduces that order exactly (2 ps: global_step->ps0, hid_w->ps1,
hid_b->ps0, sm_w->ps1, sm_b->ps0); `strategy="byte_balanced"` is the better sharding mode for this engine
(greedy largest-first by bytes), since hid_w alone is 98.6 % of the bytes.

`strategy="row_split"` additionally splits the hidden weight *inside* the variable: TF stores it `[in, out]`, so a
TF row split is a split along the input features — exactly the K-slices the CTAs of the fused step kernel own
(csrc/fused_step_sm90.cu). Slice r of the 8 goes to ps task r % num_ps: every ps shard then serves 1/num_ps of the
pull and push bytes of the big variable (the reference's `--ps_hosts` list, DS:73-77, finally balances the flagship
model); the small variables stay round-robin.

A shard's *arena* is one flat fp32 buffer; every variable sits at a 64-element (256-byte) aligned offset,
2-D weights of hidden layers use a padded leading dimension so TMA row strides are 16-byte multiples. The
unit of push hand-off is a *flag* (one per pushed tile), the unit of apply work is an *item* (2-D block of the
arena, announced by one flag; several items may share a flag so that several ps CTAs apply one tile) — see
csrc/protocol.h.

Two tilings exist: `engine="graph"` (per-layer kernels: 128 x dw_tile_n dW tiles, one item per tile) and
`engine="fused"` (fused step kernel, 784-H-10 models: 8 column slices of the hidden weight, one flag each, every slice
cut into `ps_row_blocks` row blocks = items).
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List, Tuple

from ..models.mlp import MLPSpec, VarSpec

FUSED_CLUSTER = 8     # CTAs per cluster of the fused step kernel == column slices of the hidden weight
FUSED_MAX_CHUNKS = 4  # 32-feature k-chunks per CTA
FUSED_MAX_HIDDEN = 128
FUSED_MAX_BATCH = 32
FUSED_MAX_CLASSES = 11
PS_ROW_BLOCKS = 4     # fused tiling: ps items (CTAs) per pushed column slice
TILE_M = 128          # rows of a dW tile / width of a bias or head slice
DW_TILE_N = 64        # columns of a dW tile (bn of the dW GEMM)
ALIGN_ELEMS = 64      # 256-byte alignment of every variable inside the arena
GLOBAL_STEP = "global_step"


def _round_up(a: int, b: int) -> int:
    return (a + b - 1) // b * b


def padded_ld(n: int) -> int:
    return _round_up(n, 8)


def place_variables(spec: MLPSpec, num_ps: int, strategy: str = "round_robin") -> Dict[str, int]:
    """Map variable name (incl. `global_step`) -> ps task index."""
    names = [GLOBAL_STEP] + [v.name for v in spec.variables()]
    if num_ps <= 0:
        raise ValueError("need at least one ps task")
    if strategy in ("round_robin", "row_split"):   # row_split: whole-variable owners stay round-robin
        return {n: i % num_ps for i, n in enumerate(names)}
    if strategy == "byte_balanced":
        sizes = {v.name: v.numel * 4 for v in spec.variables()}
        sizes[GLOBAL_STEP] = 4
        load = [0] * num_ps
        out: Dict[str, int] = {GLOBAL_STEP: 0}  # the step counter stays on ps 0 (workers read it from there)
        load[0] += 4
        for n in sorted((n for n in names if n != GLOBAL_STEP), key=lambda k: -sizes[k]):
            k = min(range(num_ps), key=lambda j: (load[j], j))
            out[n] = k
            load[k] += sizes[n]
        return out
    raise ValueError(f"unknown sharding strategy {strategy!r} (round_robin | byte_balanced | row_split)")


@dataclass(frozen=True)
class Item:
    offset: int   # element offset in the arena
    rows: int
    cols: int
    ld: int
    shadow: bool  # refresh the bf16 shadow copy of this block on apply
    flag: int = -1  # index of the per-push flag announcing this block (-1: assigned = own item index)


@dataclass(frozen=True)
class Piece:
    """Column range [c0, c1) of a variable owned by ps task `ps` (whole-variable placement: one piece)."""
    ps: int
    c0: int
    c1: int
    offset: int   # element offset of the *variable* (column 0) inside that shard's arena


@dataclass(frozen=True)
class FusedSliceLayout:
    """What CTA `rank` of the fused step kernel's cluster owns (csrc/protocol.h FusedSlice)."""
    rank: int
    kc_begin: int
    kc_count: int
    ps: int
    flag: int
    w_offset: int


@dataclass
class VarLayout:
    spec: VarSpec
    ps: int
    offset: int          # element offset of the variable inside its shard's arena
    ld: int              # leading dimension (== cols for vectors / the classifier weight)
    item_base: int       # index of this variable's first item in the shard's item table
    n_items: int
    role: str            # "hidden_w" | "hidden_b" | "last_w" | "last_b"
    flag_base: int = 0   # index of this variable's first flag on its (primary) shard
    pieces: Tuple[Piece, ...] = ()   # who owns which columns (row_split: several shards)

    @property
    def rows(self) -> int:
        return self.spec.shape[0] if len(self.spec.shape) == 2 else 1

    @property
    def cols(self) -> int:
        return self.spec.shape[-1]

    @property
    def span(self) -> int:
        """Elements the variable occupies in the arena (with row padding)."""
        return self.rows * self.ld if len(self.spec.shape) == 2 else self.cols


@dataclass
class ShardLayout:
    ps: int
    variables: List[VarLayout] = field(default_factory=list)
    items: List[Item] = field(default_factory=list)
    arena_elems: int = 0
    owns_global_step: bool = False
    n_flags: int = 0

    @property
    def n_items(self) -> int:
        return len(self.items)


@dataclass
class ModelLayout:
    spec: MLPSpec
    placement: Dict[str, int]
    shards: List[ShardLayout]
    by_name: Dict[str, VarLayout]
    dw_tile_n: int = DW_TILE_N     # columns of a dW tile == bn of the dW GEMMs == width of a hidden-weight item
    engine: str = "graph"          # "graph" | "fused" (which kernels push into this layout)
    fused_slices: Tuple[FusedSliceLayout, ...] = ()
    strategy: str = "round_robin"

    def shard_of(self, name: str) -> ShardLayout:
        return self.shards[self.by_name[name].ps]


def dw_tile_n_for(dtype: str) -> int:
    """dW tile width per compute dtype. fp32 (tf32 MMA, 32-element = 128-byte slabs) uses 32-column tiles: twice
    the tiles of the 64-column layout, i.e. twice the worker CTAs pushing and twice the ps CTAs applying a push
    (the per-item apply is what bounds a shard's push rate). bf16 slabs are 64 elements wide."""
    return 32 if dtype == "fp32" else 64


def _items_for(role: str, offset: int, rows: int, cols: int, ld: int, dw_tile_n: int = DW_TILE_N) -> List[Item]:
    items: List[Item] = []
    if role == "hidden_w":
        # tile order == gridDim of the dW GEMM: mtile-major, then ntile (tile = mtile * ntiles + ntile)
        for r0 in range(0, rows, TILE_M):
            for c0 in range(0, cols, dw_tile_n):
                items.append(Item(offset + r0 * ld + c0, min(TILE_M, rows - r0), min(dw_tile_n, cols - c0), ld, True))
    elif role == "hidden_b":
        for c0 in range(0, cols, TILE_M):
            items.append(Item(offset + c0, 1, min(TILE_M, cols - c0), cols, False))
    elif role == "last_w":
        # head kernel: CTA j pushes columns [128 j, 128 j + 128) of every class row
        for c0 in range(0, cols, TILE_M):
            items.append(Item(offset + c0, rows, min(TILE_M, cols - c0), ld, False))
    elif role == "last_b":
        items.append(Item(offset, 1, cols, cols, False))
    else:
        raise ValueError(role)
    return items


def fused_eligible(spec: MLPSpec, batch_size: int, dtype: str = "fp32") -> bool:
    """Can the fused step kernel (csrc/fused_step_sm90.cu) run this model? One hidden layer of <= 128 units, <= 11
    classes, batch <= 32, fp32 storage (tf32 MMA), 8 <= ceil(in / 32) <= 32 and in % 4 == 0."""
    sizes = spec.layer_sizes
    if len(sizes) != 2 or dtype != "fp32":
        return False
    fin, hid = sizes[0]
    nchunks = (fin + 31) // 32
    return (hid <= FUSED_MAX_HIDDEN and spec.num_classes <= FUSED_MAX_CLASSES and 1 <= batch_size <= FUSED_MAX_BATCH
            and fin % 4 == 0 and FUSED_CLUSTER <= nchunks <= FUSED_CLUSTER * FUSED_MAX_CHUNKS)


def fused_chunk_split(in_features: int) -> List[Tuple[int, int]]:
    """(first k-chunk, k-chunks) of each of the 8 cluster CTAs: 32-feature chunks dealt as evenly as possible."""
    nchunks = (in_features + 31) // 32
    base, rem = divmod(nchunks, FUSED_CLUSTER)
    out, k = [], 0
    for r in range(FUSED_CLUSTER):
        n = base + (1 if r < rem else 0)
        out.append((k, n))
        k += n
    return out


def build_layout(spec: MLPSpec, num_ps: int, strategy: str = "round_robin", dw_tile_n: int = DW_TILE_N,
                 engine: str = "graph", ps_row_blocks: int = PS_ROW_BLOCKS) -> ModelLayout:
    if engine not in ("graph", "fused"):
        raise ValueError(f"unknown engine {engine!r}")
    if strategy == "row_split" and engine != "fused":
        raise ValueError("sharding 'row_split' splits the hidden weight along the K-slices of the fused step kernel; "
                         "it needs the fused engine (one hidden layer <= 128 units, batch <= 32, fp32)")
    placement = place_variables(spec, num_ps, strategy)
    shards = [ShardLayout(ps=k) for k in range(num_ps)]
    shards[placement[GLOBAL_STEP]].owns_global_step = True
    by_name: Dict[str, VarLayout] = {}
    n_layers = len(spec.layer_sizes)
    fused_slices: List[FusedSliceLayout] = []

    def alloc(k: int, span: int) -> int:
        sh = shards[k]
        off = _round_up(sh.arena_elems, ALIGN_ELEMS)
        sh.arena_elems = off + span
        return off

    for v in spec.variables():
        k = placement[v.name]
        last = v.layer == n_layers - 1
        if v.kind == "weight":
            role = "last_w" if last else "hidden_w"
            rows, cols = v.shape
            ld = cols if last else padded_ld(cols)
            if engine == "fused" and not last:
                # Fused tiling: rows are padded to whole 128-byte lines (32 floats). Every 128-byte row segment of a
                # pulled W tile / pushed dW tile is then ONE aligned line on the ps shard instead of two half lines:
                # half the NVLink packets and no partial-line writes into the mailbox (with ld = 784 the ps ingress
                # took 10-25 us to acknowledge a tile once three workers pushed concurrently).
                ld = _round_up(cols, 32)
            span = rows * ld
        else:
            role = "last_b" if last else "hidden_b"
            rows, cols = 1, v.shape[0]
            ld = cols
            span = cols
        if engine == "fused" and role == "hidden_w":
            # 8 column slices (one per cluster CTA, one flag each), every slice cut into row blocks (= ps items)
            split = fused_chunk_split(cols)
            owners = [(r % num_ps) if strategy == "row_split" else k for r in range(FUSED_CLUSTER)]
            offsets = {o: alloc(o, span) for o in dict.fromkeys(owners)}   # the full span on every owning shard
            blk = -(-rows // max(1, ps_row_blocks))
            pieces = []
            first_item = {o: None for o in offsets}
            n_items_primary = 0
            for r, (kb, kn) in enumerate(split):
                o = owners[r]
                sh = shards[o]
                c0, c1 = min(kb * 32, cols), min((kb + kn) * 32, cols)
                flag = sh.n_flags
                sh.n_flags += 1
                if first_item[o] is None:
                    first_item[o] = len(sh.items)
                if c1 > c0:
                    for r0 in range(0, rows, blk):
                        sh.items.append(Item(offsets[o] + r0 * ld + c0, min(blk, rows - r0), c1 - c0, ld, False, flag))
                        if o == owners[0]:
                            n_items_primary += 1
                pieces.append(Piece(o, c0, c1, offsets[o]))
                fused_slices.append(FusedSliceLayout(r, kb, kn if c1 > c0 else 0, o, flag, offsets[o]))
            prim = owners[0]
            vl = VarLayout(spec=v, ps=prim, offset=offsets[prim], ld=ld, item_base=first_item[prim] or 0,
                           n_items=n_items_primary, role=role, flag_base=fused_slices[0].flag, pieces=tuple(pieces))
            for o in offsets:
                shards[o].variables.append(vl)
            by_name[v.name] = vl
            continue
        sh = shards[k]
        offset = alloc(k, span)
        if engine == "fused":
            # small variables: one item, one flag each (the fused kernel pushes them whole)
            raw = [Item(offset, rows, cols, ld, False)]
        else:
            raw = _items_for(role, offset, rows, cols, ld, dw_tile_n)
        flag_base = sh.n_flags
        items = [Item(it.offset, it.rows, it.cols, it.ld, it.shadow, sh.n_flags + i) for i, it in enumerate(raw)]
        sh.n_flags += len(items)
        vl = VarLayout(spec=v, ps=k, offset=offset, ld=ld, item_base=len(sh.items), n_items=len(items), role=role,
                       flag_base=flag_base, pieces=(Piece(k, 0, cols, offset),))
        sh.items.extend(items)
        sh.variables.append(vl)
        by_name[v.name] = vl
    for sh in shards:
        sh.arena_elems = max(_round_up(sh.arena_elems, ALIGN_ELEMS), ALIGN_ELEMS)
    return ModelLayout(spec=spec, placement=placement, shards=shards, by_name=by_name, dw_tile_n=dw_tile_n,
                       engine=engine, fused_slices=tuple(fused_slices), strategy=strategy)


def shard_bytes_summary(layout: ModelLayout) -> List[Tuple[int, int, int]]:
    """[(ps index, parameter bytes, number of items)] — for logs and tests."""
    out = []
    for sh in layout.shards:
        nbytes = 0
        for v in sh.variables:
            rows = v.rows
            nbytes += sum((pc.c1 - pc.c0) * rows * 4 for pc in v.pieces if pc.ps == sh.ps)
        out.append((sh.ps, nbytes, sh.n_items))
    return out
