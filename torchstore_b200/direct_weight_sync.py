"""Direct weight sync over NVLink -- one hop, one kernel launch per destination GPU.

Same caller-facing surface as the reference's ``torchstore/direct_weight_sync.py``
(RDMAWeightHandle :46-58, DirectWeightSyncSource :82-176, DirectWeightSyncDest :209-350) with
the data plane replaced:

* the ``rdma_buffer`` inside a handle is an :class:`NvlinkBuffer` (exported HBM region + layout;
  picklable; ``read_into`` / ``write_from`` / ``drop`` like ``monarch.rdma.RDMABuffer``);
* the destination does **not** read whole source shards into temporaries and slice afterwards
  (reference :280-286, 3.1x read amplification and 4.8 GB of scratch per rank for Llama-3-8B
  FSDP(8)->TP(8)); every plan op becomes one source-rectangle -> destination-rectangle
  descriptor and the whole plan runs as a single persistent ``copy_rects`` launch that loads
  over NVLink (peer-mapped addresses) and stores coalesced into the destination shard;
* ``transfer_dtype`` staging is refreshed by one batched fused-cast launch instead of one
  ``staging.copy_(src)`` per parameter (reference :158-169); if a handle's dtype differs from the
  destination's, the cast is fused into the gather itself.  Pairs the fused cast does not cover
  (an int64 buffer, float64 staging, ...) keep the reference's ``staging.copy_(src)``.

Typical usage is unchanged::

    source = DirectWeightSyncSource()
    handles = source.register(model.state_dict(), rank=dist.get_rank())
    await ts.put(f"{RDMA_KEY_PREFIX}/rank_{rank}", handles)
    ...
    dest = DirectWeightSyncDest()
    await dest.pull(all_handles, model.state_dict())
"""

from __future__ import annotations

import itertools
import logging
import math
import re
from collections import defaultdict
from dataclasses import dataclass

import torch

from torchstore_b200 import _native
from torchstore_b200.launch import Plans, copy_once, wait_copy_stream
from torchstore_b200.planner import HbmDescriptor, StridedMem
from torchstore_b200.transport.types import Request, TensorSlice
from torchstore_b200.utils import get_slice_intersection, to_byte_view

logger = logging.getLogger(__name__)

RDMA_KEY_PREFIX = "policy_rdma"
BLOCK = 128  # edge of a block-scaled fp8 block (elements)
# scale granularity -> native code; register() and pull() take one f"{granularity}_scales" dict for each
GRANULARITIES = {"block": _native.TSB_SCALE_PER_BLOCK, "channel": _native.TSB_SCALE_PER_CHANNEL,
                 "tensor": _native.TSB_SCALE_PER_TENSOR}
UNQUANTISED_DTYPES = {torch.bfloat16, torch.float16, torch.float32}  # what quantising routes read and dequantising writes
SCALE_FORMATS = (None, "ue8m0")  # scale_fmt of the quantising routes: float32 amax / 448, or its power of two up
SCALED_DTYPES = (torch.float8_e4m3fn, torch.int8)  # what a scaled handle holds, and quant_dtype's choices


def scale_fmt_flags(scale_fmt: str | None) -> int:
    """The native quantising plans' ``flags`` for ``scale_fmt`` (ValueError for an unknown format)."""
    if scale_fmt is not None and (not isinstance(scale_fmt, str) or scale_fmt not in SCALE_FORMATS):
        raise ValueError(f"scale_fmt must be None or 'ue8m0', not {scale_fmt!r}")
    return _native.TSB_QUANT_UE8M0 if scale_fmt == "ue8m0" else 0


# ---------------------------------------------------------------------------------------------
# the rdma_buffer duck-type
# ---------------------------------------------------------------------------------------------
class NvlinkBuffer:
    """Handle to a contiguous tensor in some GPU's HBM, readable/writable from any GPU on the box.

    Drop-in for the ``rdma_buffer`` field of :class:`RDMAWeightHandle` (reference call sites
    direct_weight_sync.py:143,174,339; monarch_rdma.py:121,146,177).  Pickles to plain bytes.
    """

    def __init__(self, tensor: torch.Tensor | None = None, *, descriptor: HbmDescriptor | None = None):
        if descriptor is None:
            if tensor is None:
                raise ValueError("NvlinkBuffer needs a tensor or a descriptor")
            if not tensor.is_contiguous():
                raise ValueError("NvlinkBuffer registers contiguous memory (stage non-contiguous tensors first)")
            descriptor = HbmDescriptor.from_tensor(tensor)
        self.descriptor = descriptor
        # keep the exporter's tensor alive as long as the handle object lives in its process
        self._keepalive = tensor

    # -- metadata --------------------------------------------------------------------------------
    @property
    def dtype(self) -> torch.dtype:
        return self.descriptor.dtype

    @property
    def shape(self) -> tuple:
        return self.descriptor.shape

    @property
    def nbytes(self) -> int:
        return self.descriptor.nbytes

    @property
    def device(self) -> int:
        return self.descriptor.device

    def __getstate__(self):
        return {"descriptor": self.descriptor}

    def __setstate__(self, state):
        self.descriptor = state["descriptor"]
        self._keepalive = None

    def window(self, device: int) -> StridedMem:
        """The registered tensor as seen from ``device`` (imports + caches the mapping)."""
        return self.descriptor.resolve(device)

    # -- one-sided ops (API parity; the batched plan below is the fast path) ---------------------
    async def read_into(self, dest_byte_view: torch.Tensor) -> None:
        await self._move(dest_byte_view, read=True)

    async def write_from(self, src_byte_view: torch.Tensor) -> None:
        await self._move(src_byte_view, read=False)

    async def _move(self, local_bytes: torch.Tensor, read: bool) -> None:
        if not local_bytes.is_cuda:
            raise RuntimeError("NvlinkBuffer moves bytes between GPUs; got a CPU tensor")
        if local_bytes.dtype != torch.uint8 or local_bytes.dim() != 1 or not local_bytes.is_contiguous():
            raise ValueError("expected a flat contiguous uint8 view (see to_byte_view)")
        if local_bytes.numel() != self.nbytes:
            raise RuntimeError(f"size mismatch: buffer has {self.nbytes} bytes, view has {local_bytes.numel()}")
        device = local_bytes.device.index
        remote = self.window(device).flat_bytes()
        local = StridedMem.from_tensor(local_bytes)
        copy_once({device: [(remote, local) if read else (local, remote)]})
        await wait_copy_stream(device)

    async def drop(self) -> None:
        try:
            self.descriptor.release()
        except Exception as e:  # cleanup failures are logged, not raised (reference monarch_rdma.py:176-179)
            logger.warning("NvlinkBuffer.drop failed: %s", e)
        self._keepalive = None


class ScaledNvlinkBuffer(NvlinkBuffer):
    """An :class:`NvlinkBuffer` over a scaled ``float8_e4m3fn`` or ``int8`` weight shard (its descriptor's dtype
    says which) that also carries its float32 scale (the dequantisation multiplier: ``weight_scale_inv`` per
    128x128 block, ``weight_scale`` per channel or per tensor), the granularity, and the shard's global offset ``(row0, col0)`` in the last
    two dims, which anchors the blocks at the global origin.  Pickles to plain data.  ``read_into`` /
    ``write_from`` move the raw fp8 (or int8) bytes; a pull into a bf16/f16/f32 destination dequantises."""

    def __init__(self, tensor: torch.Tensor | None = None, scale: torch.Tensor | None = None, granularity: str = "",
                 row0: int = 0, col0: int = 0, *, descriptor: HbmDescriptor | None = None,
                 scale_descriptor: HbmDescriptor | None = None):
        super().__init__(tensor, descriptor=descriptor)
        if granularity not in GRANULARITIES:
            raise ValueError(f"granularity must be one of {sorted(GRANULARITIES)}, not {granularity!r}")
        self.scale_descriptor = scale_descriptor if scale_descriptor is not None else HbmDescriptor.from_tensor(scale)
        self.granularity = granularity
        self.row0, self.col0 = int(row0), int(col0)
        self._scale_keepalive = scale

    def __getstate__(self):
        return {"descriptor": self.descriptor, "scale_descriptor": self.scale_descriptor,
                "granularity": self.granularity, "row0": self.row0, "col0": self.col0}

    def __setstate__(self, state):
        super().__setstate__(state)
        self.scale_descriptor = state["scale_descriptor"]
        self.granularity = state["granularity"]
        self.row0, self.col0 = state["row0"], state["col0"]
        self._scale_keepalive = None

    def scale_window(self, device: int) -> StridedMem:
        """The scale tensor as seen from ``device``."""
        return self.scale_descriptor.resolve(device)

    async def drop(self) -> None:
        await super().drop()
        try:
            self.scale_descriptor.release()
        except Exception as e:
            logger.warning("ScaledNvlinkBuffer.drop failed to release the scale: %s", e)
        self._scale_keepalive = None


def source_scale_shapes(granularity: str, shape: tuple, row0: int, col0: int) -> list[tuple]:
    """Accepted shapes of the scale of a ``shape`` fp8 shard at global offset (row0, col0) in its last
    two dims: exactly the groups the shard touches, anchored at the global origin."""
    lead, (n, k) = tuple(shape[:-2]), tuple(shape[-2:])
    if granularity == "block":
        return [lead + (-(-(row0 + n) // BLOCK) - row0 // BLOCK, -(-(col0 + k) // BLOCK) - col0 // BLOCK)]
    if granularity == "channel":
        return [lead + (n, 1)]
    return [lead, lead + (1,)]


def scale_grid(granularity: str, shape: tuple, row0: int, col0: int) -> tuple:
    """The scale of a ``shape`` fp8 shard at global offset (row0, col0) viewed as ``lead + (group rows, group
    cols)``: one of :func:`source_scale_shapes`, with ``lead + (1, 1)`` per tensor."""
    if granularity == "tensor":
        return tuple(shape[:-2]) + (1, 1)
    return source_scale_shapes(granularity, shape, row0, col0)[0]


def verbatim_scale_rects(granularity: str, shape: tuple, offset: tuple, ops: list, *,
                         src_starts: list | None = None, src_rows: list | None = None) -> tuple[list, tuple | None]:
    """Map the scales of a verbatim pull: fp8 bytes and scales of same-granularity sources moved as they are.

    ``shape`` and ``offset`` are the destination's local shape and global offset (all dims); each op is
    ``(source shard shape, source shard global offset, (global offset, extent) of the op's rectangle)``.
    Destination groups are anchored at the destination's local origin (128x128 blocks, rows, or the matrix
    per leading index); source groups at the global origin, cut by the source shard.  ``src_starts`` (packed
    destinations) gives, per op, the source's global coordinates of the rectangle's first element, where they
    differ from the destination's; without it the two coordinate systems are the same.  ``src_rows`` (rotary packed
    parts, with ``src_starts``) gives, per op, None or ``(hd, heads, halves, rows)``: the op's rows in the destination's
    dim -2 are (heads, halves, rows) whose source rows step by (hd, 1, 2) from its first (:class:`PackedPart`).

    Returns ``(rects, None)`` when every destination group lies inside one source group of one op:
    ``rects[i] = (op index, source index, destination index)``, unit-step slices into the :func:`scale_grid`
    views of the op's source scale and of the destination scale, together writing every destination scale
    once.  Otherwise ``([], group)``: the first (lexicographically smallest) offending destination group as
    ``lead + (group row, group col)``.  ValueError when a destination element lies in no op's rectangle or in
    two."""
    nd = len(shape)
    lead = nd - 2
    rows, cols = shape[-2:]
    # per dim: destination group size and source group size (None: the whole dim, as far as the shard reaches)
    size, src_size = [1] * lead, [1] * lead
    if granularity == "block":
        size, src_size = size + [BLOCK, BLOCK], src_size + [BLOCK, BLOCK]
    elif granularity == "channel":
        size, src_size = size + [1, cols], src_size + [1, None]
    else:
        size, src_size = size + [rows, cols], src_size + [None, None]
    starts = src_starts if src_starts is not None else [g_off for _, _, (g_off, _) in ops]
    row_maps = src_rows if src_rows is not None else [None] * len(ops)
    local = []  # op rectangles in destination-local coordinates: [(start, stop) per dim]
    volume = 0
    for (src_shape, src_off, (g_off, ext)), sg, rm in zip(ops, starts, row_maps):
        box = [(g - o, g - o + e) for g, o, e in zip(g_off, offset, ext)]
        sext = list(ext)
        if rm is not None:  # the source rows the op reads: whole heads, or one head half of step 2
            sext[-2] = rm[1] * rm[0] if rm[2] == 2 else 2 * rm[3] - 1
        if any(s < 0 or t > n or s >= t for (s, t), n in zip(box, shape)) or \
                any(g < so or g + e > so + n for g, e, so, n in zip(sg, sext, src_off, src_shape)):
            raise ValueError(f"op rectangle at {tuple(g_off)} extent {tuple(ext)} is empty or leaves its source shard "
                             "or the destination")
        local.append(box)
        volume += math.prod(ext)
    for i, a in enumerate(local):
        for b in local[:i]:
            if all(max(sa, sb) < min(ta, tb) for (sa, ta), (sb, tb) in zip(a, b)):
                first = tuple(o + max(sa, sb) for o, (sa, _), (sb, _) in zip(offset, a, b))
                raise ValueError(f"global element {first} is covered by two handles")
    if volume != math.prod(shape):
        raise ValueError(f"{math.prod(shape) - volume} of its {math.prod(shape)} elements are covered by no handle")

    def groups(d, s, t):  # destination groups [first, last + 1) meeting local [s, t) in dim d
        return s // size[d], (t - 1) // size[d] + 1

    bad = []  # low corners of boxes of offending groups
    for box in local:
        low = [groups(d, s, t)[0] for d, (s, t) in enumerate(box)]
        for d, (s, t) in enumerate(box):  # an op edge inside a group: the group straddles two handles
            if s % size[d]:
                bad.append(tuple(low))
            if t % size[d] and t != shape[d]:
                bad.append(tuple(low[:d] + [(t - 1) // size[d]] + low[d + 1:]))
    for d in range(lead, nd):  # a group across a source group edge (only 128-blocks have such edges)
        if src_size[d] is None:
            continue
        if src_starts is None:
            for j in range(-(-shape[d] // size[d])):
                s, t = offset[d] + j * size[d], offset[d] + min((j + 1) * size[d], shape[d])
                if s // src_size[d] != (t - 1) // src_size[d]:
                    bad.append(tuple(j if e == d else 0 for e in range(nd)))
                    break
            continue
        for box, sg, rm in zip(local, starts, row_maps):  # packed: each op's own shift between the two coordinate systems
            s0, t0 = box[d]
            for j in range(*groups(d, s0, t0)):
                lo, hi = max(s0, j * size[d]) - s0, min(t0, (j + 1) * size[d]) - s0
                if rm is not None and d == nd - 2:  # the rows' image under the rotary order: its first and last
                    lo, hi = _rotary_image(rm, lo, hi)
                s, t = sg[d] + lo, sg[d] + hi
                if s // src_size[d] != (t - 1) // src_size[d]:
                    bad.append(tuple(j if e == d else groups(e, *box[e])[0] for e in range(nd)))
                    break
    if bad:
        return [], min(bad)
    rects = []
    for i, (box, (_, src_off, _), sg, rm) in enumerate(zip(local, ops, starts, row_maps)):
        src_idx, dst_idx = [], []
        for d, (s, t) in enumerate(box):
            j0, j1 = groups(d, s, t)
            g0 = sg[d] - s + j0 * size[d]  # global start of the first group, in the source's coordinates
            k0 = 0 if src_size[d] is None else g0 // src_size[d] - src_off[d] // src_size[d]
            src_idx.append(slice(k0, k0 + j1 - j0))
            dst_idx.append(slice(j0, j1))
        if rm is None or src_size[nd - 2] is None:
            rects.append((i, tuple(src_idx), tuple(dst_idx)))
            continue
        # rotary rows: per destination row group, the source group holding its image (one source row per channel)
        s, t = box[nd - 2]
        pieces = []  # (source start, step, destination start, count) along the rows
        if granularity == "channel":
            hd, heads, halves, rows = rm
            for a in range(heads):
                for b in range(halves):
                    pieces.append((sg[nd - 2] - src_off[nd - 2] + a * hd + b, 2, s + (a * halves + b) * rows, rows))
        else:
            for j in range(*groups(nd - 2, s, t)):
                lo, _ = _rotary_image(rm, max(s, j * BLOCK) - s, min(t, (j + 1) * BLOCK) - s)
                k = (sg[nd - 2] + lo) // BLOCK - src_off[nd - 2] // BLOCK
                if pieces and pieces[-1][0] + pieces[-1][3] == k and pieces[-1][2] + pieces[-1][3] == j:
                    pieces[-1] = pieces[-1][:3] + (pieces[-1][3] + 1,)
                else:
                    pieces.append((k, 1, j, 1))
        for k, step, j, n in pieces:
            src_idx[nd - 2], dst_idx[nd - 2] = slice(k, k + step * (n - 1) + 1, step), slice(j, j + n)
            rects.append((i, tuple(src_idx), tuple(dst_idx)))
    return rects, None


def _rotary_image(rm: tuple, lo: int, hi: int) -> tuple[int, int]:
    """``(first, last + 1)`` of the source rows (relative to the op's first) that the op's destination rows
    ``[lo, hi)`` read, for the rotary row map ``rm = (hd, heads, halves, rows)`` (:func:`verbatim_scale_rects`)."""
    hd, _, halves, rows = rm
    def src(i):
        a, r = divmod(i, halves * rows)
        b, c = divmod(r, rows)
        return a * hd + b + 2 * c
    first = last = src(lo)
    i = lo
    while i < hi:  # per head half, the rows of [lo, hi) are one progression of step 2
        end = min(hi, (i // rows + 1) * rows)
        first, last = min(first, src(i)), max(last, src(end - 1))
        i = end
    return first, last + 1


@dataclass(frozen=True)
class PackedPart:
    """One part of a packed (fused) destination, such as vLLM's ``qkv_proj`` or an expert of ``w13_weight``.

    ``dest_index`` is a tuple of ints and unit-step slices into the destination's *local* tensor, one entry per
    dim; the box it selects is what the part fills, and an int entry drops its dim.  The box is read from the
    handles named ``source``, starting at global offsets ``source_offsets`` of the source tensor (one per source
    dim: the box's rank after the int entries are dropped).  Each element at local index ``i`` of the box takes
    the source's value at ``source_offsets + (i - box start)``, through the route the destination's dtype and
    scale dicts select (DESIGN.md section 4, "Packed destinations").

    ``rotary_head_dim = hd`` reorders the rows of every head, as a torchtitan (Meta) Llama's ``wq`` / ``wk`` need
    on their way into a Hugging Face / vLLM ``qkv_proj``: the source holds each head's ``hd`` rows (its dim -2) in
    interleaved rotary order, pairs ``(2j, 2j + 1)``, and the destination receives them in half-split order, pairs
    ``(j, j + hd / 2)``.  A box element whose component along the source's dim -2 is ``h * hd + t * hd / 2 + j``
    (``t`` in {0, 1}) reads source row ``source_offsets[-2] + h * hd + 2 * j + t``; every other dim is as above.
    ``None`` keeps the rows in order.

    ``transpose = True`` reads an input-major source into an output-major destination, as a grouped-GEMM trainer's
    MoE experts (``w1`` / ``w3`` ``[E, dim, hidden]``, ``w2`` ``[E, hidden, dim]``) need on their way into vLLM's
    ``w13_weight`` / ``w2_weight``: the box, after its int dims are dropped, has shape ``(..., a, b)`` and reads the
    source box of shape ``(..., b, a)`` at ``source_offsets`` (in the source's own coordinates), its last two dims
    swapped.  A box element at ``(..., i, j)`` reads source index ``source_offsets + (..., j, i)``.  The swapped dims
    must be the destination's last two (no int index on them), the source needs at least 2 dims, and it does not
    combine with ``rotary_head_dim``.  Transposed parts take the element-wise routes only (byte copies, fused casts,
    ``transfer_dtype`` staging): a quantised destination (a scale dict names it) and scaled source handles are
    refused (DESIGN.md section 4, "Transposed packed parts")."""

    source: str
    dest_index: tuple
    source_offsets: tuple
    rotary_head_dim: int | None = None
    transpose: bool = False


@dataclass
class RDMAWeightHandle:
    """Serializable handle to one weight shard (same fields as the reference)."""

    rdma_buffer: object  # NvlinkBuffer
    tensor_slice: TensorSlice  # shard position in the global tensor
    source_rank: int


def _last_two_offsets(tslice: TensorSlice) -> tuple[int, int]:
    """Global (row, column) offset of a shard in its last two dims."""
    return int(tslice.offsets[-2]), int(tslice.offsets[-1])


def _request_to_slice(req: Request, param: torch.Tensor) -> TensorSlice:
    """TensorSlice of a request; plain tensors cover their whole (own) global shape at offset 0."""
    if req.tensor_slice is not None:
        return req.tensor_slice
    shape = tuple(param.shape)
    zeros = tuple(0 for _ in shape)
    return TensorSlice(offsets=zeros, coordinates=zeros, global_shape=shape, local_shape=shape,
                       mesh_shape=tuple(1 for _ in shape))


# ---------------------------------------------------------------------------------------------
# source side (trainer)
# ---------------------------------------------------------------------------------------------
class DirectWeightSyncSource:
    """Registers live parameter memory (zero-copy) or dtype-cast staging buffers.

    With ``transfer_dtype`` every param gets an HBM staging buffer in that dtype; ``refresh()``
    re-casts all of them with ONE fused-cast kernel launch per device.  A param whose dtype has no
    fused cast to ``transfer_dtype`` is refreshed like the reference does it, with
    ``staging.copy_(source)`` on the caller's stream.
    """

    def __init__(self) -> None:
        self._handles: dict[str, RDMAWeightHandle] = {}
        # name -> (staging_buffer, source_local_tensor)
        self._staging: dict[str, tuple[torch.Tensor, torch.Tensor]] = {}
        self._refresh_plans = Plans()
        self._copied: list[tuple[torch.Tensor, torch.Tensor]] = []  # (staging, source) refreshed with copy_
        self._devices: tuple[int, ...] = ()  # devices holding registered memory (fence targets)
        # quantize= names: name -> (fp8 or int8 staging, float32 scale, source local tensor), refreshed by _quant_plans
        self._quantized: dict[str, tuple[torch.Tensor, torch.Tensor, torch.Tensor]] = {}
        self._quant_plans = Plans()

    def register(self, state_dict: dict[str, torch.Tensor], rank: int,
                 transfer_dtype: torch.dtype | None = None,
                 tensor_slices: dict[str, TensorSlice] | None = None, *,
                 block_scales: dict[str, torch.Tensor] | None = None,
                 channel_scales: dict[str, torch.Tensor] | None = None,
                 tensor_scales: dict[str, torch.Tensor] | None = None,
                 quantize: dict[str, str] | None = None,
                 scale_fmt: str | None = None,
                 quant_dtype: torch.dtype | None = None) -> dict[str, RDMAWeightHandle]:
        """Create a handle for every entry of ``state_dict`` (tensors or DTensors).

        ``tensor_slices`` (extension) gives the global rectangle of *plain* local shards for
        callers that do not wrap them in DTensors.

        Scaled fp8 sources (extension): a ``float8_e4m3fn`` weight named in one of ``block_scales``
        (float32 ``weight_scale_inv`` per 128x128 block), ``channel_scales`` (``weight_scale`` per row)
        or ``tensor_scales`` (one per matrix) is published with its scale, so that a pull into a bf16, f16
        or f32 destination dequantises it (DESIGN.md section 4).  Scales are anchored at the global
        origin: a shard at global offset (r0, c0) of its last two dims carries exactly the groups it
        touches (:func:`source_scale_shapes`).  Such weights are registered zero-copy.  An ``int8`` weight
        (W8A8-INT8 ``weight_scale`` per channel or per tensor, block-INT8 ``weight_scale_inv``) is published the
        same way: a pull dequantises it into bf16/f16/f32 as ``(q.float() * scale).to(dst)``, moves it verbatim
        into a scaled int8 destination, or moves its bytes into an unscaled int8 one.

        Source-side quantisation (extension): ``quantize={name: "block" | "channel" | "tensor"}`` publishes a
        bf16, f16 or f32 weight (at least 2 dims, contiguous, on CUDA) as float8_e4m3fn staging plus a float32
        scale, a scaled handle exactly like one registered with a scale dict, so every pull that reads scaled
        handles reads it.  Groups are shard-local and anchored at the global origin: per block the part of a
        global 128x128 block inside the shard, per channel the shard's part of a row, per tensor the shard's
        [rows, cols] matrix.  Each group gets the quantising formula of DESIGN.md section 4.  ``refresh()``
        requantises the staging from the live weights; ``transfer_dtype`` does not apply to these names.
        ``scale_fmt="ue8m0"`` rounds every such scale up to a power of two (DESIGN.md section 4, "UE8M0 scales");
        the scales stay float32, so every consumer of scaled handles reads them unchanged.
        ``quant_dtype=torch.int8`` publishes int8 staging instead (``None`` or ``torch.float8_e4m3fn``: fp8): per
        group ``scale_inv = max(amax, 1e-4) / 127`` and ``q = round_half_even(x * (127 / max(amax, 1e-4)))``
        saturated to [-128, 127], NaN -> 0 (DESIGN.md section 4, "INT8 sources").  ValueError without
        ``quantize``, for another dtype, and together with ``scale_fmt``.

        Everything is validated before anything is exported, so a failed call registers nothing."""
        scale_dicts = {"block_scales": block_scales, "channel_scales": channel_scales, "tensor_scales": tensor_scales}
        quant_flags = scale_fmt_flags(scale_fmt)
        if scale_fmt is not None and not quantize:
            raise ValueError("scale_fmt applies to source-side quantisation: it needs quantize")
        if quant_dtype is not None:
            if not quantize:
                raise ValueError("quant_dtype applies to source-side quantisation: it needs quantize")
            if not isinstance(quant_dtype, torch.dtype) or quant_dtype not in SCALED_DTYPES:
                raise ValueError(f"quant_dtype must be None, torch.float8_e4m3fn or torch.int8, not {quant_dtype!r}")
            if quant_dtype == torch.int8 and scale_fmt is not None:
                raise ValueError("scale_fmt='ue8m0' does not apply to int8 staging: its scales are float32 amax / 127 "
                                 "(power-of-two int8 scales are not offered)")
        staging_dtype = quant_dtype or torch.float8_e4m3fn
        quantize = self._check_quantize(state_dict, tensor_slices, quantize or {}, scale_dicts)
        scaled = self._check_source_scales(state_dict, transfer_dtype, tensor_slices, scale_dicts)
        handles: dict[str, RDMAWeightHandle] = {}
        self._refresh_plans.close()
        self._quant_plans.close()
        self._staging = {}
        self._copied = []
        self._quantized = {}
        casts: dict[int, list] = defaultdict(list)  # device -> (source, staging) windows of the refresh
        quant_targets: dict[int, list] = defaultdict(list)  # device -> SourceQuantTarget of the refresh
        devices = set()
        for name, param in state_dict.items():
            req = Request.from_any(name, param, tensor_slices.get(name) if tensor_slices else None)
            local = req.tensor_val
            tslice = _request_to_slice(req, param)
            if not local.is_cuda:
                raise RuntimeError(f"direct weight sync registers GPU memory; '{name}' is on {local.device}")
            devices.add(local.device.index)
            if any(name in (d or {}) for d in scale_dicts.values()):
                granularity, scale = scaled[name]
                handles[name] = RDMAWeightHandle(
                    rdma_buffer=ScaledNvlinkBuffer(local, scale, granularity, *_last_two_offsets(tslice)),
                    tensor_slice=tslice, source_rank=rank)
                continue
            if name in quantize:
                granularity = quantize[name]
                r0, c0 = _last_two_offsets(tslice)
                qbuf = torch.empty(local.shape, dtype=staging_dtype, device=local.device)
                scale = torch.empty(source_scale_shapes(granularity, tuple(local.shape), r0, c0)[0], dtype=torch.float32,
                                    device=local.device)
                rows, cols = local.shape[-2:]
                quant_targets[local.device.index].append(_native.SourceQuantTarget(
                    local.data_ptr(), qbuf.data_ptr(), scale.data_ptr(), local.numel() // (rows * cols), rows, cols, r0, c0,
                    _native.cast_code(local.dtype), GRANULARITIES[granularity]))
                self._quantized[name] = (qbuf, scale, local)
                handles[name] = RDMAWeightHandle(rdma_buffer=ScaledNvlinkBuffer(qbuf, scale, granularity, r0, c0),
                                                 tensor_slice=tslice, source_rank=rank)
                continue
            if transfer_dtype is not None:
                staging = torch.empty(local.shape, dtype=transfer_dtype, device=local.device)
                self._staging[name] = (staging, local)
                if fused_refresh(local.dtype, transfer_dtype):
                    casts[local.device.index].append((StridedMem.from_tensor(local), StridedMem.from_tensor(staging)))
                else:
                    self._copied.append((staging, local))
                buf = staging
            else:
                assert local.is_contiguous(), f"Expected contiguous tensor for key={name}, strides={local.stride()}"
                buf = local
            handles[name] = RDMAWeightHandle(rdma_buffer=NvlinkBuffer(buf), tensor_slice=tslice, source_rank=rank)
        self._handles = handles
        self._devices = tuple(sorted(devices))
        if self._staging or self._quantized:
            if casts:
                self._refresh_plans = Plans.build(casts)
            if quant_targets:
                self._quant_plans = Plans.build_source_quant(
                    quant_targets, quant_flags, _native.TSB_I8 if staging_dtype == torch.int8 else _native.TSB_F8E4M3)
            self.refresh()
        else:
            # make sure the weights the handles point at are materialised before anyone reads them
            for dev in devices:
                torch.cuda.current_stream(dev).synchronize()
        staged = len(self._staging) + len(self._quantized)
        logger.info("Registered %d NVLink handles (%d staged, %d quantised into scaled %s, %d direct)", len(handles),
                    staged, len(self._quantized), "int8" if staging_dtype == torch.int8 else "fp8", len(handles) - staged)
        return handles

    @staticmethod
    def _check_source_scales(state_dict, transfer_dtype, tensor_slices, scales: dict[str, dict | None]) -> dict[str, tuple]:
        """Validate the scale dicts of :meth:`register` -> ``{name: (granularity, scale)}``.  Raises before
        anything is exported."""
        from torch.distributed.tensor import DTensor

        seen: set[str] = set()
        for kw, by_name in scales.items():
            for name in by_name or {}:
                if name not in state_dict:
                    raise ValueError(f"{kw} names '{name}', which is not in the state dict")
                if name in seen:
                    raise ValueError(f"'{name}' is in more than one of block_scales, channel_scales and tensor_scales")
                seen.add(name)
        if seen and transfer_dtype is not None:
            raise ValueError("scaled fp8 weights are published as they are: block_scales, channel_scales and "
                             "tensor_scales cannot be combined with transfer_dtype")
        out: dict[str, tuple] = {}
        for kw, by_name in scales.items():
            granularity = kw.removesuffix("_scales")
            for name, scale in (by_name or {}).items():
                req = Request.from_any(name, state_dict[name], tensor_slices.get(name) if tensor_slices else None)
                w = req.tensor_val
                if w.dtype not in SCALED_DTYPES:
                    raise TypeError(f"scaled weight '{name}' ({kw}) must be float8_e4m3fn or int8, not {w.dtype}")
                if w.dim() < 2 or w.numel() == 0 or not w.is_contiguous() or not w.is_cuda:
                    raise ValueError(f"scaled weight '{name}' must be a non-empty contiguous CUDA tensor with at least "
                                     f"2 dims; got shape {tuple(w.shape)}, strides {w.stride()} on {w.device}")
                if isinstance(scale, DTensor):
                    raise TypeError(
                        f"the scale of '{name}' ({kw}) is a DTensor; pass the local scale of this shard as a plain "
                        "tensor.  Scales are anchored at the global origin and must hold exactly the groups the "
                        "local weight shard touches; sharding a scale tensor on its own gives local shapes that can "
                        "match while covering the wrong groups")
                if not isinstance(scale, torch.Tensor) or scale.dtype != torch.float32:
                    what = type(scale).__name__ if not isinstance(scale, torch.Tensor) else str(scale.dtype)
                    raise TypeError(f"the scale of '{name}' ({kw}) must be a plain float32 tensor, not {what}")
                r0, c0 = _last_two_offsets(_request_to_slice(req, state_dict[name]))
                wants = source_scale_shapes(granularity, tuple(w.shape), r0, c0)
                if tuple(scale.shape) not in wants or not scale.is_contiguous() or scale.device != w.device:
                    want = " or ".join(map(str, wants))
                    raise ValueError(f"the scale of '{name}' ({kw}, shard at global offset ({r0}, {c0})) must be a "
                                     f"contiguous {want} tensor on {w.device}; got {tuple(scale.shape)}, strides "
                                     f"{scale.stride()} on {scale.device}")
                out[name] = (granularity, scale)
        return out

    @staticmethod
    def _check_quantize(state_dict, tensor_slices, quantize: dict, scale_dicts: dict[str, dict | None]) -> dict[str, str]:
        """Validate the ``quantize`` dict of :meth:`register` -> ``{name: granularity}``.  Raises before anything
        is exported or allocated."""
        for name, granularity in quantize.items():
            if name not in state_dict:
                raise ValueError(f"quantize names '{name}', which is not in the state dict")
            if any(name in (d or {}) for d in scale_dicts.values()):
                raise ValueError(f"'{name}' is in quantize and in one of block_scales, channel_scales and tensor_scales: "
                                 "a weight is either published with its scale or quantised on refresh")
            if granularity not in GRANULARITIES:
                raise ValueError(f"quantize['{name}'] must be one of {sorted(GRANULARITIES)}, not {granularity!r}")
            w = Request.from_any(name, state_dict[name], tensor_slices.get(name) if tensor_slices else None).tensor_val
            if w.dtype not in UNQUANTISED_DTYPES:
                raise TypeError(f"quantised weight '{name}' must be bfloat16, float16 or float32, not {w.dtype}")
            if w.dim() < 2:
                raise ValueError(f"quantised weight '{name}' needs at least 2 dims; got shape {tuple(w.shape)}")
            if w.numel() == 0:
                raise ValueError(f"quantised weight '{name}' is empty (shape {tuple(w.shape)})")
            if not w.is_contiguous():
                raise ValueError(f"quantised weight '{name}' is not contiguous (shape {tuple(w.shape)}, strides {w.stride()})")
            if not w.is_cuda:
                raise ValueError(f"quantised weight '{name}' must live on a CUDA device, not {w.device}")
        return dict(quantize)

    def refresh(self) -> int:
        """Re-cast the source params into their staging buffers and requantise the ``quantize`` names into
        their scaled fp8 (or int8) staging (no-op without either).  Returns the number of staging buffers refreshed.
        Blocks until everything has landed so the caller may publish/notify right after, like the
        reference's synchronous copy loop."""
        if not self._staging and not self._quantized:
            return 0
        self._quant_plans.launch()
        self._refresh_plans.launch()
        for staging, local in self._copied:
            staging.copy_(local)
        self._quant_plans.synchronize()
        self._refresh_plans.synchronize()
        for dev in {local.device.index for _, local in self._copied}:
            torch.cuda.current_stream(dev).synchronize()
        return len(self._staging) + len(self._quantized)

    def fence(self) -> None:
        """Make every write queued on the caller's streams (optimizer step, staging refresh) land in
        HBM before readers are told to pull.  The reference has no such fence (its RDMA reads race
        with in-flight kernels); on one box it costs a stream sync."""
        for dev in self._devices:
            torch.cuda.current_stream(dev).synchronize()

    async def cleanup(self) -> None:
        for handle in self._handles.values():
            await handle.rdma_buffer.drop()
        self._handles.clear()
        self._staging.clear()
        self._copied.clear()
        self._quantized.clear()
        self._refresh_plans.close()
        self._quant_plans.close()


def fused_refresh(src_dtype: torch.dtype, transfer_dtype: torch.dtype) -> bool:
    """Does a ``src_dtype`` param's ``transfer_dtype`` staging refresh in the batched fused-cast
    launch?  Otherwise :meth:`DirectWeightSyncSource.refresh` uses ``staging.copy_(source)``."""
    return _native.cast_supported(src_dtype, transfer_dtype)


# ---------------------------------------------------------------------------------------------
# destination side (generator)
# ---------------------------------------------------------------------------------------------
@dataclass
class _TransferOp:
    """One planned read.  Field names follow the reference (:184-206); ``recv_buffer`` is always
    None here because the kernel reads the overlap rectangle straight from the source shard."""

    rdma_buffer: object
    dest_byte_view: torch.Tensor | None
    dest_tensor: torch.Tensor | None = None  # None <=> exact match (whole shard -> whole param)
    recv_buffer: torch.Tensor | None = None
    src_slices: tuple[slice, ...] | None = None
    dest_slices: tuple[slice, ...] | None = None
    # planner metadata
    name: str = ""
    dest_local: torch.Tensor | None = None
    dest_offsets: tuple = ()  # global offsets of the destination shard and of the source shard
    src_offsets: tuple = ()
    # packed parts: the source's global coordinates of the op's first element (None: the destination's global
    # coordinates are the source's), and the destination dims an int index dropped (unit slices in dest_slices)
    src_start: tuple | None = None
    dest_dropped: tuple = ()
    # rotary parts: (destination dim of the source's rows, head dim hd, heads, halves, rows per half).  The op's rows
    # are (heads, halves, rows) with source row steps (hd, 1, 2) and destination row steps (hd, hd / 2, 1) from its
    # first row; src_slices then bound the source rows it reads
    rotary: tuple | None = None
    # transposed parts: src_slices index the source in its own order; op_windows swaps its last two dims
    transpose: bool = False


class DirectWeightSyncDest:
    """Pulls weights from source handles with one persistent-kernel launch per local GPU.

    The transfer plan (ops, then the compiled native tile table) is built on the first
    :meth:`pull` and cached, like the reference (:334-335).
    """

    def __init__(self) -> None:
        self._plan: list[_TransferOp] | None = None
        self._plan_signature: tuple | None = None
        self._plan_ids: tuple | None = None  # id() of the destination objects the plan was built for
        self._plan_refs: list | None = None  # ...kept alive, so those ids cannot be recycled
        self._plan_dict: dict | None = None  # the dict object they came in (identity short-cut of the next pull)
        self._native_plans = Plans()  # the compiled plan, one native plan per destination device
        self._block_plans = Plans()  # block-scaled fp8 names: one quantising plan per destination device
        self._scaled_plans = Plans()  # per-channel / per-tensor scaled fp8 names: likewise
        self._dequant_plans = Plans()  # names read from scaled fp8 handles into bf16/f16/f32: one dequantising plan per device
        self._requant_plans = Plans()  # scaled fp8 destinations read from scaled fp8 handles: one requantising plan per device
        self._int8_block_plans = Plans()  # block-scaled int8 names: one quantising plan per destination device
        self._int8_scaled_plans = Plans()  # per-channel / per-tensor scaled int8 names: likewise
        self._int8_dequant_plans = Plans()  # names read from scaled int8 handles into bf16/f16/f32: one plan per device
        self._transpose_plans = Plans()  # transposed packed parts: one transposing plan per destination device
        # ({(name, scale keyword)}, requantize, scale_fmt, verbatim, {int8 names}, packed spec)
        self._plan_key: tuple | None = None
        self._packed_last: tuple | None = None  # (packed dict, its items, its key) of the last pull (_packed_spec)
        self._plan_scale_dicts: tuple | None = None  # the three scale dict objects of the last pull
        self.last_pull_ms: dict[int, float] = {}  # device -> kernel time of the last pull

    # -- planning (host, metadata only) ----------------------------------------------------------
    def _build_plan(self, all_handles: dict[str, list[RDMAWeightHandle]],
                    dest_state_dict: dict[str, torch.Tensor],
                    dest_slices: dict[str, TensorSlice] | None = None, *,
                    packed: dict[str, tuple[PackedPart, ...]] | None = None) -> list[_TransferOp]:
        """Per destination param x per source handle: intersect, dedup replicated regions, classify
        exact / partial (same rules and op order as the reference, :221-317).

        ``dest_slices`` (extension) names the rectangle a *plain* local tensor holds, for callers
        that keep raw shards instead of DTensors (e.g. torchrun ranks).  ``packed`` (extension) fills the
        named destinations part by part (:meth:`_check_packed`): per part x per handle of its source, the
        intersection with the part's source box becomes one partial op in the destination's local
        coordinates."""
        parts = self._check_packed(all_handles, dest_state_dict, packed)
        ops: list[_TransferOp] = []
        for name, param in dest_state_dict.items():
            if name in parts:
                dest_req = Request.from_any(name, param, dest_slices.get(name) if dest_slices else None)
                ops += _packed_ops(name, dest_req.tensor_val, tuple(_request_to_slice(dest_req, param).offsets),
                                   parts[name])
                continue
            handles = all_handles.get(name)
            if not handles:
                continue
            override = dest_slices.get(name) if dest_slices else None
            dest_req = Request.from_any(name, param, override)
            dest_tensor = dest_req.tensor_val
            dest_slice = _request_to_slice(dest_req, param)
            seen: set[tuple] = set()  # replicated sources: read each region once
            for handle in handles:
                inter = get_slice_intersection(handle.tensor_slice, dest_slice)
                if inter is None:
                    continue
                region = (inter.offsets, inter.local_shape)
                if region in seen:
                    continue
                seen.add(region)
                src_slice = handle.tensor_slice
                exact = src_slice.offsets == dest_slice.offsets and src_slice.local_shape == dest_slice.local_shape
                if exact:
                    assert dest_tensor.is_contiguous(), (
                        f"Expected contiguous dest tensor for key={name}, strides={dest_tensor.stride()}"
                    )
                    ops.append(_TransferOp(rdma_buffer=handle.rdma_buffer, dest_byte_view=to_byte_view(dest_tensor),
                                           name=name, dest_local=dest_tensor, dest_offsets=tuple(dest_slice.offsets),
                                           src_offsets=tuple(src_slice.offsets)))
                else:
                    ndim = len(inter.offsets)
                    src_idx = tuple(
                        slice(inter.offsets[d] - src_slice.offsets[d],
                              inter.offsets[d] - src_slice.offsets[d] + inter.local_shape[d])
                        for d in range(ndim)
                    )
                    dst_idx = tuple(
                        slice(inter.offsets[d] - dest_slice.offsets[d],
                              inter.offsets[d] - dest_slice.offsets[d] + inter.local_shape[d])
                        for d in range(ndim)
                    )
                    ops.append(_TransferOp(rdma_buffer=handle.rdma_buffer, dest_byte_view=None, dest_tensor=dest_tensor,
                                           src_slices=src_idx, dest_slices=dst_idx, name=name, dest_local=dest_tensor,
                                           dest_offsets=tuple(dest_slice.offsets), src_offsets=tuple(src_slice.offsets)))
        logger.info("Built transfer plan with %d NVLink ops", len(ops))
        return ops

    @staticmethod
    def op_windows(op: _TransferOp, src_window: StridedMem) -> tuple[StridedMem, StridedMem]:
        """(source rectangle, destination rectangle) of one op given the mapped source shard."""
        dst_full = StridedMem.from_tensor(op.dest_local)
        if op.dest_tensor is None:
            # exact: whole shard onto whole param (reshape of the source is irrelevant: same numel)
            src = src_window
            if tuple(src.shape) != tuple(dst_full.shape):
                src = StridedMem(src.ptr, dst_full.shape, _contig(dst_full.shape), src.dtype, src.device)
            return src, dst_full
        src, dst = src_window.sub(op.src_slices), dst_full.sub(op.dest_slices)
        if getattr(op, "transpose", False):  # the source box in the destination's order: its last two dims swapped
            src = StridedMem(src.ptr, _swap_last(src.shape), _swap_last(src.stride), src.dtype, src.device)
        if op.dest_dropped:  # a packed part whose int index dropped destination dims: unit dims on the source side
            src = StridedMem(src.ptr, dst.shape, _lift(src.stride, op.dest_dropped, 0), src.dtype, src.device)
        if getattr(op, "rotary", None) is not None:
            k, hd, heads, halves, rows = op.rotary
            src = _split_rows(src, k, (heads, halves, rows), (hd, 1, 2))
            dst = _split_rows(dst, k, (heads, halves, rows), (hd, hd // 2, 1))
        return src, dst

    @staticmethod
    def _check_packed(all_handles, dest_state_dict, packed: dict | None) -> dict[str, list]:
        """Validate the ``packed`` spec of a pull -> ``{name: [(part index, part, box, dropped dims, handles)]}``,
        ``box`` the part's ``(start, stop)`` in every destination-local dim (``(i, i + 1)`` where an int index
        drops the dim).  Raises ValueError naming the destination and the part before anything is compiled."""
        out: dict[str, list] = {}
        for name, spec in (packed or {}).items():
            if name not in dest_state_dict:
                raise ValueError(f"packed names '{name}', which is not in the destination state dict")
            if all_handles.get(name):
                raise ValueError(f"packed destination '{name}' also has handles of its own name: a packed destination "
                                 "is filled from its parts only")
            dest = getattr(dest_state_dict[name], "_local_tensor", dest_state_dict[name])
            entries = []
            for k, part in enumerate(spec):
                what = f"packed destination '{name}' part {k} (source '{part.source}')"
                handles = all_handles.get(part.source) or []
                if not handles:
                    raise ValueError(f"{what}: the source has no handles")
                box, dropped = _index_box(what, part.dest_index, tuple(dest.shape))
                ext = [t - s for d, (s, t) in enumerate(box) if d not in dropped]
                gshape = tuple(handles[0].tensor_slice.global_shape)
                offs = tuple(part.source_offsets)
                if len(ext) != len(gshape) or len(offs) != len(gshape):
                    raise ValueError(f"{what}: a {len(ext)}-dim box with {len(offs)} source offsets does not match "
                                     f"the source's {len(gshape)}-dim global shape {gshape}")
                if not all(isinstance(o, int) and not isinstance(o, bool) for o in offs):
                    raise ValueError(f"{what}: source_offsets {offs} must be ints")
                if not isinstance(part.transpose, bool):
                    raise ValueError(f"{what}: transpose must be a bool, not {part.transpose!r}")
                if part.transpose:
                    if len(gshape) < 2:
                        raise ValueError(f"{what}: transpose swaps the source's last two dims, and the source has "
                                         f"{len(gshape)} dim")
                    if part.rotary_head_dim is not None:
                        raise ValueError(f"{what}: transpose and rotary_head_dim do not combine")
                    if any(d >= len(box) - 2 for d in dropped):
                        raise ValueError(f"{what}: its int index drops one of the destination's last two dims, which "
                                         "transpose swaps (they must be slices)")
                    ext = _swap_last(ext)  # the source box's extents, in the source's order
                if any(o < 0 or o + e > g for o, e, g in zip(offs, ext, gshape)):
                    raise ValueError(f"{what}: the source box at {offs} with extent {tuple(ext)} leaves the source's "
                                     f"global shape {gshape}")
                hd = part.rotary_head_dim
                if hd is not None:
                    if not isinstance(hd, int) or isinstance(hd, bool) or hd <= 0 or hd % 2:
                        raise ValueError(f"{what}: rotary_head_dim must be None or a positive even int, not {hd!r}")
                    if len(gshape) < 2:
                        raise ValueError(f"{what}: rotary_head_dim reorders the rows (dim -2) of each head, and the "
                                         f"source has {len(gshape)} dim")
                    if ext[-2] % hd:
                        raise ValueError(f"{what}: its extent {ext[-2]} along the source's dim -2 is not a multiple of "
                                         f"rotary_head_dim {hd}")
                    if offs[-2] % hd:
                        raise ValueError(f"{what}: source_offsets[-2] ({offs[-2]}) is not a multiple of rotary_head_dim "
                                         f"{hd} (heads start at source row 0)")
                for j, _, other, _, _ in entries:
                    if all(max(s, a) < min(t, b) for (s, t), (a, b) in zip(box, other)):
                        raise ValueError(f"{what}: its box overlaps part {j}'s")
                hole = _first_uncovered(offs, ext, [(tuple(h.tensor_slice.offsets), tuple(h.tensor_slice.local_shape))
                                                    for h in handles])
                if hole is not None:
                    raise ValueError(f"{what}: no handle covers global element {hole} of the source")
                entries.append((k, part, box, dropped, handles))
            out[name] = entries
        return out

    @staticmethod
    def _signature(dest_state_dict, scales: tuple = ()) -> tuple:
        # data pointers only: ~35 us for 291 tensors; a new state_dict() wrapper around the same
        # memory keeps the plan, new memory invalidates it
        sig = tuple(getattr(p, "_local_tensor", p).data_ptr() for p in dest_state_dict.values())
        for d in scales:
            if d:
                sig += tuple(s.data_ptr() for s in d.values())
        return sig

    @staticmethod
    def _ids(dest_state_dict, scales: tuple = ()) -> tuple:
        ids = tuple(map(id, dest_state_dict.values()))
        for d in scales:
            if d:
                ids += tuple(map(id, d.values()))
        return ids

    @staticmethod
    def _check_scales(all_handles, dest_state_dict, scales: dict[str, dict | None], *,
                      requantize: bool = False, verbatim: bool = False) -> dict[str, tuple]:
        """Validate the scale dicts of a pull (``{keyword: {name: scale}}``, keyword ``f"{granularity}_scales"``) ->
        ``{name: (keyword, destination, scale, route)}``, route ``"quantise"``, ``"requantise"`` or
        ``"verbatim"``.  With ``requantize``, a name whose handles are all scaled fp8 sources of one granularity is
        accepted too, and requantised; with ``verbatim``, such a name of the destination's granularity is moved as
        it is.  A float8_e4m3fn destination takes every route; an int8 destination ``"quantise"`` from bf16/f16/f32
        handles, and ``"verbatim"`` (``verbatim=True`` only) from scaled int8 handles, which no other route reads.
        Raises before anything is compiled or launched."""
        if requantize and verbatim:
            raise ValueError("requantize=True and verbatim=True are exclusive: verbatim=True moves scaled fp8 bytes and "
                             "scales as they are (same granularity, groups that line up), requantize=True re-rounds "
                             "them into any destination layout")
        out = {}
        for kw, by_name in scales.items():
            granularity = kw.removesuffix("_scales")
            what, kind = f"{granularity} scale", f"{granularity}-scaled"
            for name, scale in (by_name or {}).items():
                if name not in dest_state_dict:
                    raise ValueError(f"{kw} names '{name}', which is not in the destination state dict")
                if name in out:
                    raise ValueError(f"'{name}' is in both {out[name][0]} and {kw}: a destination has one scale layout")
                dest = getattr(dest_state_dict[name], "_local_tensor", dest_state_dict[name])
                if not isinstance(scale, torch.Tensor):
                    raise TypeError(f"{what} of '{name}' is a {type(scale).__name__}, not a tensor")
                if dest.dtype not in (torch.float8_e4m3fn, torch.int8):
                    raise TypeError(f"{kind} destination '{name}' must be float8_e4m3fn or int8, not {dest.dtype}")
                if dest.dim() < 2 or dest.numel() == 0 or not dest.is_contiguous() or not dest.is_cuda:
                    raise ValueError(f"{kind} destination '{name}' must be a non-empty contiguous CUDA tensor with at "
                                     f"least 2 dims; got shape {tuple(dest.shape)}, strides {dest.stride()} on {dest.device}")
                if scale.dtype != torch.float32:
                    raise TypeError(f"{what} of '{name}' must be float32, not {scale.dtype}")
                wants = source_scale_shapes(granularity, tuple(dest.shape), 0, 0)
                if tuple(scale.shape) not in wants or not scale.is_contiguous() or scale.device != dest.device:
                    want = " or ".join(map(str, wants))
                    raise ValueError(f"{what} of '{name}' must be a contiguous {want} tensor on {dest.device}; got "
                                     f"{tuple(scale.shape)}, strides {scale.stride()} on {scale.device}")
                handles = all_handles.get(name) or []
                if not handles:
                    raise ValueError(f"no source handles for {kind} destination '{name}': its groups would not be covered")
                kinds = {getattr(h.rdma_buffer, "granularity", None) for h in handles}
                int8 = dest.dtype == torch.int8
                if torch.int8 in _scaled_dtypes(handles):
                    out[name] = (kw, dest, scale, _int8_source_route(name, kind, granularity, dest, handles, kinds,
                                                                     requantize, verbatim))
                    continue
                route = "quantise"
                if int8 and kinds != {None}:
                    raise TypeError(f"{kind} int8 destination '{name}' has scaled fp8 handles: int8 destinations are "
                                    "quantised from bf16, f16 or f32 handles (scaled fp8 handles are neither "
                                    "requantised nor moved verbatim into int8)")
                if requantize and kinds != {None} and not int8:
                    route = "requantise"
                    if None in kinds:
                        raise ValueError(f"the handles of {kind} destination '{name}' mix scaled fp8 and unscaled sources "
                                         "(requantize=True)")
                    if len(kinds) > 1:
                        raise ValueError(f"the handles of {kind} destination '{name}' mix scale granularities "
                                         f"{sorted(kinds)} (requantize=True)")
                elif verbatim and kinds != {None} and not int8:
                    route = "verbatim"
                    if None in kinds:
                        raise TypeError(f"the handles of {kind} destination '{name}' mix scaled fp8 and unscaled sources "
                                        "(verbatim=True)")
                    if kinds != {granularity}:
                        raise ValueError(f"{kind} destination '{name}' has {'/'.join(sorted(kinds))}-scaled handles: a "
                                         "verbatim pull moves scales of the destination's granularity only; use "
                                         "requantize=True to convert them")
                else:
                    dtypes = {h.rdma_buffer.dtype for h in handles}
                    if not dtypes <= UNQUANTISED_DTYPES or len(dtypes) != 1:
                        hint = ""
                        if kinds - {None}:
                            hint = "; scaled fp8 handles are requantised only with requantize=True"
                        elif (requantize or verbatim) and not int8:
                            flag = "requantize" if requantize else "verbatim"
                            hint = f"; {flag}=True reads scaled fp8 handles (registered with a scale), not unscaled fp8"
                        raise TypeError(f"{kind} pulls of '{name}' read bf16, f16 or f32 handles of one dtype; "
                                        f"got {sorted(map(str, dtypes))}{hint}")
                out[name] = (kw, dest, scale, route)
        return out

    @staticmethod
    def _verbatim_rects(plan: list[_TransferOp], scaled: dict) -> dict[str, list]:
        """The scale rectangles of every verbatim name of ``scaled`` (:meth:`_check_scales`' verdict) ->
        ``{name: [(op, source scale index, destination scale index)]}`` (:func:`verbatim_scale_rects`).  Raises
        ValueError naming the weight before anything is compiled or launched."""
        ops: dict[str, list] = {n: [] for n, (*_, route) in scaled.items() if route == "verbatim"}
        for op in plan:
            if op.name in ops:
                ops[op.name].append(op)
        out = {}
        for name, mine in ops.items():
            kw, dest, _, _ = scaled[name]
            granularity = kw.removesuffix("_scales")
            if not mine:
                raise ValueError(f"verbatim pull of '{name}' ({kw}): no handle covers its destination")
            shape, offset = tuple(dest.shape), mine[0].dest_offsets
            rects, starts = [], []
            rows = [op.rotary[1:] if getattr(op, "rotary", None) is not None else None for op in mine]
            for op in mine:
                start = [0] * len(shape) if op.dest_slices is None else [s.start for s in op.dest_slices]
                ext = shape if op.dest_slices is None else [s.stop - s.start for s in op.dest_slices]
                src_shape, src_off = tuple(op.rdma_buffer.shape), op.src_offsets
                if op.src_start is not None:  # a packed part: the source in the destination's rank
                    if any(d >= len(shape) - 2 for d in op.dest_dropped):
                        raise ValueError(f"verbatim pull of '{name}' ({kw}): a packed part whose int index drops one "
                                         "of the destination's last two dims cannot keep its source's scale groups")
                    src_shape, src_off = _lift(src_shape, op.dest_dropped, 1), _lift(src_off, op.dest_dropped, 0)
                    starts.append(_lift(op.src_start, op.dest_dropped, 0))
                rects.append((src_shape, src_off, (tuple(o + s for o, s in zip(offset, start)), tuple(ext))))
            try:
                mapped, group = verbatim_scale_rects(granularity, shape, offset, rects, src_starts=starts or None,
                                                     src_rows=rows if any(rows) else None)
            except ValueError as e:
                raise ValueError(f"verbatim pull of '{name}' ({kw}): {e}") from None
            if group is not None:
                what, idx, legend = {"block": ("block", group, "leading indices, block row, block column"),
                                     "channel": ("row", group[:-1], "leading indices, row"),
                                     "tensor": ("matrix", group[:-2], "leading indices")}[granularity]
                raise ValueError(f"verbatim pull of '{name}' ({kw}): destination {what} {idx} ({legend}) does not lie "
                                 "inside one source group of one handle; requantize=True pulls it into these groups (the "
                                 "usual cause is a TP shard whose global column offset is not a multiple of 128)")
            out[name] = [(mine[i], src, dst) for i, src, dst in mapped]
        return out

    @staticmethod
    def _check_dequant(all_handles, dest_state_dict, scaled_dests) -> set[str]:
        """Names whose handles are scaled fp8 (or scaled int8) sources and whose destination is bf16/f16/f32: the
        dequantising plans.  A float8_e4m3fn destination of fp8 handles, or an int8 destination of int8 handles,
        gets the plain byte move.  Raises before anything is compiled or launched."""
        out = set()
        for name, param in dest_state_dict.items():
            handles = all_handles.get(name) or []
            kinds = {getattr(h.rdma_buffer, "granularity", None) for h in handles}
            if not handles or kinds == {None}:
                continue
            dtypes = _scaled_dtypes(handles)
            if len(dtypes) > 1:
                raise ValueError(f"the handles of '{name}' mix scaled int8 and scaled fp8 sources")
            fmt = "int8" if torch.int8 in dtypes else "fp8"
            if None in kinds:
                raise ValueError(f"the handles of '{name}' mix scaled {fmt} and unscaled sources")
            if len(kinds) > 1:
                raise ValueError(f"the handles of '{name}' mix scale granularities {sorted(kinds)}")
            if name in scaled_dests:
                continue  # a scaled destination: _check_scales refuses fp8 handles with its TypeError
            dest = getattr(param, "_local_tensor", param)
            if fmt == "int8":
                if dest.dtype == torch.int8:
                    continue
                if dest.dtype not in UNQUANTISED_DTYPES:
                    raise TypeError(f"'{name}' has {kinds.pop()}-scaled int8 handles: its destination must be bfloat16, "
                                    f"float16, float32 (dequantised) or int8 (bytes moved), not {dest.dtype}; int8 is not "
                                    "converted to fp8")
            elif dest.dtype == torch.float8_e4m3fn:
                continue
            if dest.dtype not in UNQUANTISED_DTYPES:
                raise TypeError(f"'{name}' has {kinds.pop()}-scaled fp8 handles: its destination must be bfloat16, "
                                f"float16, float32 (dequantised) or float8_e4m3fn (bytes moved), not {dest.dtype}")
            if dest.dim() < 2 or not dest.is_contiguous():
                raise ValueError(f"dequantised destination '{name}' must be contiguous with at least 2 dims; got shape "
                                 f"{tuple(dest.shape)}, strides {dest.stride()}")
            out.add(name)
        return out

    @staticmethod
    def _check_packed_rows(parts: dict, dequant: set, requant: set) -> None:
        """Refuse a packed part whose int index drops the destination's last dim on a route that reads scaled handles
        (``dequant`` and ``requant`` names): those kernels move whole rows of a scaled source shard into whole
        destination rows, and such a part gives each destination row one element of a source row.  ValueError naming the
        destination and the part, before anything is compiled (verbatim parts are refused by :meth:`_verbatim_rects`;
        quantising and element-wise routes take such parts)."""
        for name, entries in parts.items():
            if name not in dequant and name not in requant:
                continue
            for k, part, box, dropped, _ in entries:
                if dropped and dropped[-1] == len(box) - 1:
                    what = "dequantising" if name in dequant else "requantising"
                    raise ValueError(f"packed destination '{name}' part {k} (source '{part.source}'): its int index drops "
                                     f"the destination's last dim, which a {what} pull cannot fill (it moves whole rows of "
                                     "its scaled handles into whole destination rows); quantising and element-wise pulls "
                                     "take such parts")

    @staticmethod
    def _check_transposed_routes(parts: dict, scaled: dict) -> None:
        """Refuse a transposed packed part on any route but the element-wise ones: its destination in a scale dict
        (quantised, requantised or verbatim), or scaled handles feeding it (dequantised, or fp8 bytes moved with
        their scales elsewhere).  ValueError naming the destination and the part, before anything is compiled."""
        for name, entries in parts.items():
            for k, part, _, _, handles in entries:
                if not part.transpose:
                    continue
                what = f"packed destination '{name}' part {k} (source '{part.source}')"
                if name in scaled:
                    raise ValueError(f"{what}: a transposed part takes element-wise routes only (copies and fused casts), "
                                     f"and '{name}' is in {scaled[name][0]}: quantising transposed sources is not "
                                     "supported")
                if any(getattr(h.rdma_buffer, "granularity", None) is not None for h in handles):
                    raise ValueError(f"{what}: a transposed part takes element-wise routes only (copies and fused casts), "
                                     "and its source handles are scaled: dequantising transposed sources is not supported")

    def _compile(self, scaled: dict | None = None, dequant: set | None = None, requant: set | None = None,
                 flags: int = 0, verbatim: dict | None = None) -> None:
        """Compile the cached transfer plan along the routes :meth:`_check_scales` chose: ``scaled`` is its
        ``{name: (keyword, destination, scale, ...)}``, ``requant`` the names it requantises and ``verbatim``
        :meth:`_verbatim_rects` of the names it moves as they are; ``dequant`` is what :meth:`_check_dequant`
        returned.  ``flags`` go to the quantising and requantising plans."""
        scaled, requant, verbatim = scaled or {}, requant or set(), verbatim or {}
        # the plan kind of each quantised or requantised name, in build order: 0 requantises, 1 quantises into fp8
        # blocks, 2 into fp8 channels or tensors, 3 and 4 the same into int8 (a plan writes one destination dtype)
        kind = {n: 0 if n in requant else (1 if kw == "block_scales" else 2) + (2 if _is_int8(d) else 0)
                for n, (kw, d, *_) in scaled.items() if n not in verbatim}
        per_device: dict[int, list] = defaultdict(list)
        # verbatim names: their fp8 bytes go with the plain copies below, their scales as float32 rectangles
        for n, rects in verbatim.items():
            kw, dest_q, dest_s, *_ = scaled[n]
            dev, granularity = dest_q.device.index, kw.removesuffix("_scales")
            dst = StridedMem.from_tensor(dest_s)
            dst = _as_grid(dst, scale_grid(granularity, tuple(dest_q.shape), 0, 0))
            for op, src_idx, dst_idx in rects:
                buf = op.rdma_buffer
                grid = _lift(scale_grid(granularity, tuple(buf.shape), buf.row0, buf.col0), op.dest_dropped, 1)
                src = _as_grid(buf.scale_window(dev), grid)
                per_device[dev].append((_stepped_sub(src, src_idx), dst.sub(dst_idx)))
        # (int8 sources, device) -> (windows, {source buffer id: (name, DqSource)}): a plan reads one source format
        dq: dict[tuple, tuple[list, dict]] = {}
        quant: dict[tuple, tuple] = defaultdict(lambda: ([], {}, [], []))  # (kind, device) -> the same, names, targets
        transposed: dict[int, tuple] = defaultdict(lambda: ([], []))  # device -> (windows, the name of each)
        for op in self._plan:
            dest = op.dest_local
            if not dest.is_cuda:
                raise RuntimeError(
                    f"direct weight sync writes GPU memory; destination '{op.name}' is on {dest.device} "
                    "(torchstore_b200 has no CPU data path)"
                )
            if not isinstance(op.rdma_buffer, NvlinkBuffer):
                raise TypeError(
                    f"handle for '{op.name}' carries a {type(op.rdma_buffer).__name__}; the direct path needs NvlinkBuffer handles"
                )
            dev = dest.device.index
            window = self.op_windows(op, op.rdma_buffer.window(dev))
            if getattr(op, "transpose", False):
                pairs, names = transposed[dev]
                pairs.append(window)
                names.append(op.name)
                continue
            rotary = getattr(op, "rotary", None)  # plan ops built by hand (tests) may lack it
            grid = op.name in kind or (dequant and op.name in dequant)
            windows = _head_halves(window, rotary) if grid and rotary is not None else [window]
            if op.name in kind:
                pairs, sources, _, _ = quant[(kind[op.name], dev)]
                pairs += windows
                if kind[op.name] == 0:
                    _add_dq_source(sources, op, dev)
            elif dequant and op.name in dequant:
                pairs, sources = dq.setdefault((op.rdma_buffer.dtype == torch.int8, dev), ([], {}))
                pairs += windows
                _add_dq_source(sources, op, dev)
            else:
                per_device[dev].append(window)
        self._native_plans = Plans.build(per_device)
        try:
            for dev, (pairs, names) in sorted(transposed.items()):
                _build_named(self._transpose_plans, Plans.build_transpose, {dev: pairs}, {"rect": names},
                             lambda n: f"transposed pull of '{n}'", (_native.TSB_ERR_INVALID, _native.TSB_ERR_UNSUPPORTED))
            for (int8_src, dev), (pairs, sources) in sorted(dq.items()):
                names = [n for n, _ in sources.values()]
                _build_named(self._int8_dequant_plans if int8_src else self._dequant_plans, Plans.build_dequant_fp8,
                             {dev: (pairs, [s for _, s in sources.values()])}, {"source": names},
                             lambda n: f"dequantising pull of '{n}'")
            for n, (kw, d, s, *_) in scaled.items():
                if n not in kind:
                    continue
                _, _, names, targets = quant[(kind[n], d.device.index)]
                names.append(n)
                targets.append(_quant_target(kw.removesuffix("_scales"), d, s, n in requant))

            def pull_of(n):
                kw, d = scaled[n][:2]
                what = "requantising" if n in requant else f"{kw.removesuffix('_scales')}-scaled"
                return f"{what}{' int8' if _is_int8(d) else ''} pull of '{n}' ({kw})"

            builds = ((self._requant_plans, Plans.build_requant_fp8), (self._block_plans, Plans.build_block_fp8),
                      (self._scaled_plans, Plans.build_scaled_fp8), (self._int8_block_plans, Plans.build_block_fp8),
                      (self._int8_scaled_plans, Plans.build_scaled_fp8))
            for (k, dev), (pairs, sources, names, targets) in sorted(quant.items()):
                plans, build = builds[k]
                args, by_index = (pairs, targets), {"target": names}
                if k == 0:
                    args = (pairs, [s for _, s in sources.values()], targets)
                    by_index["source"] = [n for n, _ in sources.values()]
                _build_named(plans, lambda per_device, build=build: build(per_device, flags), {dev: args}, by_index,
                             pull_of)
        except BaseException:
            for plans in self._fp8_plans:
                plans.close()
            self._native_plans.close()
            raise

    @property
    def _fp8_plans(self) -> tuple:
        """The plans launched after the copy plan on each device's copy stream, in launch order: the transposing plans,
        then the scaled fp8 and int8 plans."""
        return (self._transpose_plans, self._block_plans, self._scaled_plans, self._dequant_plans, self._requant_plans, self._int8_block_plans,
                self._int8_scaled_plans, self._int8_dequant_plans)

    def plan_info(self) -> dict[int, dict]:
        return self._native_plans.info()

    # -- execution ---------------------------------------------------------------------------------
    async def pull(self, all_handles: dict[str, list[RDMAWeightHandle]],
                   dest_state_dict: dict[str, torch.Tensor],
                   dest_slices: dict[str, TensorSlice] | None = None, *,
                   block_scales: dict[str, torch.Tensor] | None = None,
                   channel_scales: dict[str, torch.Tensor] | None = None,
                   tensor_scales: dict[str, torch.Tensor] | None = None, requantize: bool = False,
                   scale_fmt: str | None = None, verbatim: bool = False,
                   packed: dict[str, tuple[PackedPart, ...]] | None = None) -> None:
        """Pull every overlapping region into ``dest_state_dict`` (in place).  Returns when the
        bytes are in destination HBM (so the caller may tell the source it is done reading).

        Packed destinations (extension): ``packed={name: (PackedPart, ...)}`` fills a fused generator parameter
        (``qkv_proj``, ``gate_up_proj``, a stacked MoE ``w13_weight``) from handles of other names, part by part
        (:class:`PackedPart`); values must be tuples (TypeError otherwise).  A packed name takes no handles of its
        own name.  Every route below applies unchanged: element-wise routes per element, with the scale of the
        handle each byte is read from; grouped routes (quantising, requantising, verbatim) over the destination's
        local groups whichever part an element came from, and their route checks over the union of the parts'
        handles.  ValueError naming the destination and part, before anything is compiled, for an unknown name,
        a source without handles, a name with handles of its own, a bad index, a source box outside the source,
        overlapping parts, a part the handles do not cover, and a part whose int index drops the destination's last
        dim on a dequantising or requantising route (DESIGN.md section 4, "Packed destinations").
        Elements outside every part are left alone.  Changing the spec rebuilds the plan.  A transposed part
        (``PackedPart(transpose=True)``) is moved by its own transposing plan after the copy plan; it takes the byte
        copy and fused casts only, and a ValueError naming the destination and the part refuses it for a name in the
        scale dicts or fed by scaled handles (DESIGN.md section 4, "Transposed packed parts").

        Scaled fp8 destinations (extension): float8_e4m3fn weights quantised during the pull from
        bf16/f16/f32 handles, each name in at most one of
        * ``block_scales``: float32 ``scale_inv`` per 128x128 block, the layout of DeepSeek-V3 / vLLM
          ``weight_block_size=[128, 128]`` (shape ``lead + (ceil(N/128), ceil(K/128))``);
        * ``channel_scales``: one float32 scale per output row, compressed-tensors FP8 / fbgemm-fp8
          ``weight_scale`` (shape ``lead + (N, 1)``);
        * ``tensor_scales``: one float32 scale per [N, K] matrix, vLLM ``quantization="fp8"`` (shape
          ``lead`` or ``lead + (1,)``).
        ``lead`` is the destination's dims before the last two (MoE stacks quantise every matrix on its
        own).  The formula is in DESIGN.md section 4.  Every element of such a destination must be
        covered by the handles.  The other names are pulled as without scales.

        Scaled int8 destinations (extension): a name of the three scale dicts whose destination is ``torch.int8``
        is quantised the same way into symmetric int8 (W8A8-INT8 ``weight_scale`` per channel, one scale per
        tensor, block-INT8 ``weight_scale_inv`` per 128x128 block): ``scale_inv = max(amax, 1e-4) / 127`` and
        ``q = round_half_even(x * (127 / max(amax, 1e-4)))`` saturated to [-128, 127], NaN -> 0 (DESIGN.md
        section 4, "INT8 destinations").  Only bf16/f16/f32 handles feed it: scaled fp8 handles raise TypeError
        (with or without ``requantize`` / ``verbatim``), and ``scale_fmt`` raises ValueError.  An int8
        destination outside the scale dicts is still moved as bytes.

        Scaled fp8 sources (extension): a name whose handles were registered with scales
        (``DirectWeightSyncSource.register(block_scales= / channel_scales= / tensor_scales=)``) and whose
        destination is bf16, f16 or f32 is dequantised during the pull, each element with the scale of
        the handle its bytes are read from: ``(q.float() * scale).to(dst)``.  Elements the handles do not
        cover are left alone.  A float8_e4m3fn destination not named in a scale dict gets the raw fp8
        bytes; the caller moves the scales separately (for example as their own state-dict entries).

        Requantising (extension, ``requantize=True``): a name in one of the scale dicts may then be fed by
        scaled fp8 handles of one granularity.  Each element is dequantised exactly as a pull into float32
        would write it (``f32(q) * scale`` of the handle it is read from), then quantised with the
        destination's formula: the result equals a dequantising pull into a float32 temporary followed by a
        quantising pull from it, byte for byte.  This re-rounds, so it is refused (TypeError) by default.

        Power-of-two scales (extension, ``scale_fmt="ue8m0"``): every name of the three scale dicts, quantised or
        requantised, gets its float32 ``amax_c / 448`` rounded up to a power of two (DESIGN.md section 4, "UE8M0
        scales"), the scales of DeepSeek-V3.1 checkpoints (``"scale_fmt": "ue8m0"``) and of FP8 recipes that round
        scales to powers of two.  ``None`` keeps the plain float32 formula.  ValueError for another value, or for a
        ``scale_fmt`` without a name in the scale dicts.  Changing it rebuilds the plan.

        Verbatim (extension, ``verbatim=True``): a name in one of the scale dicts whose handles are all scaled fp8
        sources of the destination's granularity is moved as it is: its fp8 bytes and the float32 scales of the
        source groups holding its groups go into the copy plan, with no arithmetic, so ``f32(q) * scale`` is the
        source's bit for bit (NaN and Inf groups, UE8M0 and any checkpoint scale included).  Every destination group
        must lie inside one source group of one handle (:func:`verbatim_scale_rects`); ValueError naming the first
        group that does not, for handles of another granularity, for an element covered by no handle or by two,
        with ``requantize=True``, and for a ``scale_fmt`` when every scaled name is verbatim.  Names fed by
        bf16/f16/f32 handles are still quantised.  Changing it rebuilds the plan.

        Scaled int8 sources (extension): handles registered as int8 with a scale (``register(block_scales= /
        channel_scales= / tensor_scales=)`` of an int8 weight, or ``quantize=`` with ``quant_dtype=torch.int8``)
        are dequantised into a bf16/f16/f32 destination, ``(q.float() * scale).to(dst)``, and moved as raw bytes
        into an int8 destination outside the scale dicts.  An int8 destination in a scale dict takes them only with
        ``verbatim=True`` (the verbatim rule above, bytes and scales as they are); without it, with
        ``requantize=True`` (int8 handles are not requantised), and into any float8_e4m3fn destination they raise
        TypeError.  A name whose handles mix scaled int8 and scaled fp8 sources raises ValueError (DESIGN.md section
        4, "INT8 sources").

        Steady state costs one native call to launch and a poll loop: the cached plan is checked
        against the destination OBJECTS first (their ids; the plan keeps them alive), the kernel
        is enqueued, and the data-pointer signature -- which catches ``param.data = new`` under an
        unchanged object -- is recomputed while the kernel runs."""
        scales = (block_scales, channel_scales, tensor_scales)
        scale_dicts = {f"{g}_scales": d for g, d in zip(GRANULARITIES, scales)}
        scaled_names = frozenset((n, kw) for kw, d in scale_dicts.items() for n in (d or ()))
        flags = scale_fmt_flags(scale_fmt)
        if scale_fmt is not None and not scaled_names:
            raise ValueError("scale_fmt applies to quantised and requantised names: block_scales, channel_scales or "
                             "tensor_scales must name at least one")
        # a name whose destination turns from float8_e4m3fn into int8 (or back) at the same address needs other kernels
        int8_names = frozenset(n for n, _ in scaled_names
                               if _is_int8(getattr(dest_state_dict.get(n), "_local_tensor", dest_state_dict.get(n))))
        key = (scaled_names, bool(requantize), scale_fmt, bool(verbatim), int8_names, self._packed_spec(packed))
        if self._plan is not None and key != self._plan_key:
            logger.info("scaled names or their granularity changed; rebuilding the transfer plan")
            self.close()
        if self._plan is not None and dest_state_dict is self._plan_dict and \
                all(a is b for a, b in zip(scales, self._plan_scale_dicts)):
            # the very dict object of the last pull: launch first, validate it (object ids, then data pointers)
            # while the kernel runs -- a stale launch only fills memory the plan still references
            self.launch()
            same = self._ids(dest_state_dict, scales) == self._plan_ids and \
                self._signature(dest_state_dict, scales) == self._plan_signature
            await self.wait()
            if same:
                return
            logger.info("destination dict was edited in place; rebuilding the transfer plan")
            self.close()
        ids = self._ids(dest_state_dict, scales)
        refs = list(dest_state_dict.values()) + [t for d in scales if d for t in d.values()]
        verified = False
        if self._plan is not None and ids != self._plan_ids:
            # other wrapper objects: fine if they alias the same memory (e.g. a fresh state_dict())
            if self._signature(dest_state_dict, scales) != self._plan_signature:
                logger.info("destination tensors changed; rebuilding the transfer plan")
                self.close()
            else:
                self._plan_ids, self._plan_refs, self._plan_dict = ids, refs, dest_state_dict
                self._plan_scale_dicts = scales
            verified = True
        if self._plan is None:
            parts = self._check_packed(all_handles, dest_state_dict, packed)
            route_handles = _route_handles(all_handles, parts)
            scaled = self._check_scales(route_handles, dest_state_dict, scale_dicts, requantize=requantize,
                                        verbatim=verbatim)
            if scale_fmt is not None and any(_is_int8(d) for _, d, *_ in scaled.values()):
                raise ValueError("scale_fmt='ue8m0' does not apply to int8 destinations: their scales are float32 "
                                 "amax / 127 (power-of-two int8 scales are not offered)")
            if scale_fmt is not None and all(route == "verbatim" for *_, route in scaled.values()):
                raise ValueError("scale_fmt does nothing here: every name of block_scales, channel_scales and "
                                 "tensor_scales is moved verbatim and keeps its source's scales")
            dequant = self._check_dequant(route_handles, dest_state_dict, scaled)
            requant = {n for n, (*_, route) in scaled.items() if route == "requantise"}
            self._check_packed_rows(parts, dequant, requant)
            self._check_transposed_routes(parts, scaled)
            self._plan = self._build_plan(all_handles, dest_state_dict, dest_slices, packed=packed)
            try:
                verbatim_rects = self._verbatim_rects(self._plan, scaled)
                self._compile(scaled, dequant, requant, flags, verbatim_rects)
            except BaseException:
                self._plan = None
                raise
            self._plan_key = key
            self._plan_signature = self._signature(dest_state_dict, scales)
            self._plan_ids, self._plan_refs, self._plan_dict = ids, refs, dest_state_dict
            self._plan_scale_dicts = scales
            verified = True
        self.launch()
        stale = not verified and self._signature(dest_state_dict, scales) != self._plan_signature
        await self.wait()
        if stale:
            # the launch above filled the OLD memory (still referenced by the plan, so harmless)
            logger.info("destination storage changed under the same tensors; rebuilding the transfer plan")
            self.close()
            await self.pull(all_handles, dest_state_dict, dest_slices, block_scales=block_scales,
                            channel_scales=channel_scales, tensor_scales=tensor_scales, requantize=requantize,
                            scale_fmt=scale_fmt, verbatim=verbatim, packed=packed)

    def _packed_spec(self, packed: dict | None) -> frozenset | None:
        """The plan-key entry of ``packed`` (:func:`_packed_key`).  The dict object of the previous pull, with the same
        names mapped to the very same tuples, reuses its key without looking at a single part (the tuples are kept
        alive, so their ids cannot be recycled)."""
        last = self._packed_last
        if packed and last is not None and packed is last[0] and len(packed) == len(last[1]) and \
                all(n == m and v is w for (n, v), (m, w) in zip(packed.items(), last[1])):
            return last[2]
        key = _packed_key(packed)
        self._packed_last = (packed, tuple(packed.items()), key) if packed else None
        return key

    def launch(self) -> None:
        """Enqueue the cached plan on each device's copy stream, fenced against the caller's current
        stream on both sides (later work on that stream sees the new weights without a host wait)."""
        if self._plan is None:
            raise RuntimeError("pull() must build the plan first")
        self._native_plans.launch()
        for plans in self._fp8_plans:
            if plans:
                plans.launch()

    async def wait(self) -> None:
        await self._native_plans.wait()
        ms = self._native_plans.elapsed_ms()
        # the plans of a device run back to back on its copy stream
        for plans in self._fp8_plans:
            if plans:
                await plans.wait()
                for dev, t in plans.elapsed_ms().items():
                    ms[dev] = ms.get(dev, 0.0) + t
        self.last_pull_ms.update(ms)

    def close(self) -> None:
        self._native_plans.close()
        for plans in self._fp8_plans:
            plans.close()
        self._plan = None
        self._plan_key = self._plan_ids = self._plan_refs = self._plan_dict = self._plan_scale_dicts = None


def _build_named(plans: Plans, build, per_device: dict, names: dict[str, list[str]], pull_of,
                 codes: tuple = (_native.TSB_ERR_INVALID,)) -> None:
    """Add ``build(per_device)`` (a ``Plans.build_*`` call) to ``plans``.  A TsbError of one of ``codes`` naming
    "target N" (or else "source N", or "rect N") becomes a ValueError naming the weight ``names[noun][N]``, whose pull
    ``pull_of(name)`` describes."""
    try:
        plans.update(build(per_device))
    except _native.TsbError as e:
        if e.code in codes:
            for noun, by_index in names.items():
                m = re.search(noun + r" (\d+)", str(e))
                if m:
                    raise ValueError(f"{pull_of(by_index[int(m.group(1))])}: {e}") from e
        raise


def _scaled_dtypes(handles) -> set:
    """The dtypes of the scaled handles (:class:`ScaledNvlinkBuffer`) among ``handles``."""
    return {h.rdma_buffer.dtype for h in handles if getattr(h.rdma_buffer, "granularity", None) is not None}


def _int8_source_route(name: str, kind: str, granularity: str, dest, handles, kinds: set, requantize: bool,
                       verbatim: bool) -> str:
    """:meth:`DirectWeightSyncDest._check_scales`' verdict on a scaled destination fed by scaled int8 handles: only
    ``"verbatim"`` into int8 of the destination's granularity; every other case raises."""
    if len(_scaled_dtypes(handles)) > 1:
        raise ValueError(f"the handles of {kind} destination '{name}' mix scaled int8 and scaled fp8 sources")
    if None in kinds:
        raise ValueError(f"the handles of {kind} destination '{name}' mix scaled int8 and unscaled sources")
    if dest.dtype != torch.int8:
        raise TypeError(f"{kind} {dest.dtype} destination '{name}' has scaled int8 handles: int8 is not converted to "
                        "fp8 (int8 handles are dequantised into bf16, f16 or f32, or moved into int8)")
    if requantize:
        raise TypeError(f"{kind} int8 destination '{name}' has scaled int8 handles: int8 handles are not requantised; "
                        "verbatim=True moves their bytes and scales as they are")
    if not verbatim:
        raise TypeError(f"{kind} int8 destination '{name}' has scaled int8 handles: pass verbatim=True to move their "
                        "bytes and scales as they are (int8 destinations are quantised from bf16, f16 or f32 handles)")
    if kinds != {granularity}:
        raise ValueError(f"{kind} destination '{name}' has {'/'.join(sorted(kinds))}-scaled int8 handles: a verbatim "
                         "pull moves scales of the destination's granularity only")
    return "verbatim"


def _is_int8(dest) -> bool:
    """Whether a scaled destination (or None for a name the dict lacks) is quantised into int8."""
    return getattr(dest, "dtype", None) == torch.int8


def _add_dq_source(sources: dict, op: _TransferOp, dev: int) -> None:
    """Describe the scaled fp8 shard behind ``op`` once per buffer: ``{id(buffer): (name, DqSource)}``."""
    buf = op.rdma_buffer
    if id(buf) not in sources:
        w, s = buf.window(dev), buf.scale_window(dev)
        rows, cols = w.shape[-2:]
        sources[id(buf)] = (op.name, _native.DqSource(w.ptr, s.ptr, w.numel // (rows * cols), rows, cols,
                                                      buf.row0, buf.col0, GRANULARITIES[buf.granularity], 0))


def _quant_target(granularity: str, dest: torch.Tensor, scale: torch.Tensor, requant: bool):
    """The native target of a scaled fp8 destination: a BqTarget for a block-quantising pull, else an SqTarget (the
    requantising plan takes SqTargets of every granularity)."""
    rows, cols = dest.shape[-2:]
    args = (dest.data_ptr(), scale.data_ptr(), dest.numel() // (rows * cols), rows, cols)
    if granularity == "block" and not requant:
        return _native.BqTarget(*args)
    return _native.SqTarget(*args, GRANULARITIES[granularity], 0)


def _packed_key(packed: dict | None) -> frozenset | None:
    """The content of a ``packed`` spec as a plan-key entry (None without packed names).  TypeError unless every
    value is a tuple of :class:`PackedPart` whose index and offsets are tuples: immutable values are what lets a
    later pull with the same dict trust the ids of its values."""
    if not packed:
        return None
    if not isinstance(packed, dict):
        raise TypeError(f"packed must be a dict of name -> tuple of PackedPart, not {type(packed).__name__}")
    out = []
    for name, parts in packed.items():
        if not isinstance(parts, tuple) or not all(isinstance(p, PackedPart) for p in parts):
            raise TypeError(f"packed['{name}'] must be a tuple of PackedPart, not {type(parts).__name__}: the cached "
                            "plan recognises an unchanged spec by the identity of these (immutable) tuples")
        for p in parts:
            if not isinstance(p.dest_index, tuple) or not isinstance(p.source_offsets, tuple):
                raise TypeError(f"packed['{name}']: dest_index and source_offsets of a PackedPart must be tuples")
        out.append((name, tuple((p.source, tuple((e.start, e.stop, e.step) if isinstance(e, slice) else e
                                                 for e in p.dest_index), p.source_offsets, p.rotary_head_dim,
                                    p.transpose)
                                for p in parts)))
    return frozenset(out)


def _index_box(what: str, index: tuple, shape: tuple) -> tuple[list, tuple]:
    """``(box, dropped dims)`` of a packed part's ``dest_index`` into a destination of local ``shape``."""
    if len(index) != len(shape):
        raise ValueError(f"{what}: dest_index has {len(index)} entries for a {len(shape)}-dim destination")
    box, dropped = [], []
    for d, (e, n) in enumerate(zip(index, shape)):
        if isinstance(e, int) and not isinstance(e, bool):
            if not 0 <= e < n:
                raise ValueError(f"{what}: dest_index entry {d} ({e}) is out of range for extent {n}")
            box.append((e, e + 1))
            dropped.append(d)
        elif isinstance(e, slice):
            if e.step not in (None, 1):
                raise ValueError(f"{what}: dest_index entry {d} ({e}) has a non-unit step")
            s, t = 0 if e.start is None else e.start, n if e.stop is None else e.stop
            if not (isinstance(s, int) and isinstance(t, int) and 0 <= s < t <= n):
                raise ValueError(f"{what}: dest_index entry {d} ({e}) is out of range (or empty) for extent {n}")
            box.append((s, t))
        else:
            raise ValueError(f"{what}: dest_index entry {d} is a {type(e).__name__}, not an int or a slice")
    return box, tuple(dropped)


def _first_uncovered(lo: tuple, ext: list, boxes: list) -> tuple | None:
    """The lexicographically first global element of the box ``lo + [0, ext)`` outside every ``(offsets, shape)``
    box, or None.  The boxes' edges cut it into cells that are covered or not as a whole, so that element is the
    low corner of the first uncovered cell."""
    hi = [a + e for a, e in zip(lo, ext)]
    cuts = [sorted({a, b} | {min(max(v, a), b) for bo, bs in boxes for v in (bo[d], bo[d] + bs[d])})
            for d, (a, b) in enumerate(zip(lo, hi))]
    for corner in itertools.product(*(c[:-1] for c in cuts)):
        if not any(all(o <= c < o + s for c, o, s in zip(corner, bo, bs)) for bo, bs in boxes):
            return tuple(corner)
    return None


def _packed_ops(name: str, dest: torch.Tensor, dest_offsets: tuple, entries: list) -> list[_TransferOp]:
    """The ops of one packed destination (:meth:`DirectWeightSyncDest._check_packed` ``entries``): per part, per
    handle of its source (replicated regions read once), the intersection of the handle with the part's source
    box, placed in the destination's local coordinates."""
    ops = []
    nd = dest.dim()
    for _, part, box, dropped, handles in entries:
        kept = [d for d in range(nd) if d not in dropped]
        so = part.source_offsets
        flip = _swap_last if part.transpose else tuple  # destination order <-> source order of the kept dims
        ext = flip([box[d][1] - box[d][0] for d in kept])
        seen: set[tuple] = set()
        for h in handles:
            ho, hs = h.tensor_slice.offsets, h.tensor_slice.local_shape
            lo = tuple(max(a, b) for a, b in zip(ho, so))
            hi = tuple(min(a + x, b + e) for a, x, b, e in zip(ho, hs, so, ext))
            if any(t <= s for s, t in zip(lo, hi)) or (lo, hi) in seen:
                continue
            seen.add((lo, hi))
            # rotary parts: (first source row, first destination row of the box, row spans) of the handle's rows
            pieces = [(None, None, None)] if part.rotary_head_dim is None else \
                _rotary_pieces(so[-2], part.rotary_head_dim, lo[-2], hi[-2])
            for srow, drow, rotary in pieces:
                slo, shi, dlo, dhi = list(lo), list(hi), [a - b for a, b in zip(lo, so)], [a - b for a, b in zip(hi, so)]
                if rotary is not None:
                    heads, halves, rows = rotary
                    n_dst = heads * halves * rows
                    n_src = heads * part.rotary_head_dim if halves == 2 else 2 * rows - 1
                    slo[-2], shi[-2], dlo[-2], dhi[-2] = srow, srow + n_src, drow, drow + n_dst
                    rotary = (kept[-2], part.rotary_head_dim) + rotary
                dlo, dhi = flip(dlo), flip(dhi)
                dst_idx = [slice(s, t) for s, t in box]
                for i, d in enumerate(kept):
                    dst_idx[d] = slice(box[d][0] + dlo[i], box[d][0] + dhi[i])
                ops.append(_TransferOp(rdma_buffer=h.rdma_buffer, dest_byte_view=None, dest_tensor=dest,
                                       src_slices=tuple(slice(s - o, t - o) for s, t, o in zip(slo, shi, ho)),
                                       dest_slices=tuple(dst_idx), name=name, dest_local=dest, dest_offsets=dest_offsets,
                                       src_offsets=tuple(ho), src_start=tuple(slo), dest_dropped=dropped, rotary=rotary,
                                       transpose=part.transpose))
    return ops


def _rotary_pieces(r0: int, hd: int, a: int, b: int) -> list[tuple]:
    """The source rows ``[a, b)`` of a rotary part whose heads start at source row ``r0`` (a multiple of ``hd``
    rows before ``a``), as ``(first source row, its row in the part's box, (heads, halves, rows))`` pieces: one
    piece for the whole heads, and one per head half that the handle's edges cut (one arithmetic progression of
    step 2 each)."""
    h2 = hd // 2
    first, last = -(-(a - r0) // hd), (b - r0) // hd  # whole heads [first, last)
    if first >= last:
        return [p for h in range((a - r0) // hd, -(-(b - r0) // hd)) for p in _half_pieces(r0, hd, h, a, b)]
    lead = [p for h in range((a - r0) // hd, first) for p in _half_pieces(r0, hd, h, a, b)]
    tail = _half_pieces(r0, hd, last, a, b) if last * hd + r0 < b else []
    return lead + [(r0 + first * hd, first * hd, (last - first, 2, h2))] + tail


def _half_pieces(r0: int, hd: int, h: int, a: int, b: int) -> list[tuple]:
    """The pieces of head ``h`` inside source rows ``[a, b)``: per half ``t``, rows ``r0 + h * hd + t + 2j``."""
    h2, out = hd // 2, []
    for t in (0, 1):
        base = r0 + h * hd + t
        j0, j1 = max(0, -(-(a - base) // 2)), min(h2, -(-(b - base) // 2))
        if j0 < j1:
            out.append((base + 2 * j0, h * hd + t * h2 + j0, (1, 1, j1 - j0)))
    return out


def _swap_last(values) -> tuple:
    """``values`` with its last two entries swapped (a transposed part's box between destination and source order)."""
    v = tuple(values)
    return v[:-2] + (v[-1], v[-2])


def _split_rows(win: StridedMem, k: int, shape: tuple, steps: tuple) -> StridedMem:
    """``win`` with its dim ``k`` replaced by dims of extents ``shape`` and strides ``steps`` times its row stride."""
    st = win.stride[k]
    return StridedMem(win.ptr, win.shape[:k] + shape + win.shape[k + 1:],
                      win.stride[:k] + tuple(s * st for s in steps) + win.stride[k + 1:], win.dtype, win.device)


def _head_halves(window: tuple, rotary: tuple) -> list[tuple]:
    """The (source, destination) windows of a rotary op (:meth:`DirectWeightSyncDest.op_windows`) cut into one pair per
    head half, each a plain box of destination rows whose source rows step by 2: the kernels that map a rect onto a
    scale grid take one row dim."""
    k = rotary[0]
    src, dst = window
    heads, halves, rows = src.shape[k:k + 3]
    out = []
    for h in range(heads):
        for t in range(halves):
            pair = []
            for w in (src, dst):
                off = (h * w.stride[k] + t * w.stride[k + 1]) * w.itemsize
                pair.append(StridedMem(w.ptr + off, w.shape[:k] + (rows,) + w.shape[k + 3:],
                                       w.stride[:k] + (w.stride[k + 2],) + w.stride[k + 3:], w.dtype, w.device))
            out.append(tuple(pair))
    return out


def _stepped_sub(win: StridedMem, index: tuple) -> StridedMem:
    """``win[index]`` for slices of positive step (:meth:`StridedMem.sub` takes unit steps only)."""
    base = win.sub(tuple(slice(s.start, s.stop) for s in index))
    shape = tuple(len(range(s.start, s.stop, s.step or 1)) for s in index)
    stride = tuple(st * (s.step or 1) for st, s in zip(win.stride, index))
    return StridedMem(base.ptr, shape, stride, win.dtype, win.device)


def _route_handles(all_handles: dict, parts: dict) -> dict:
    """``all_handles`` with every packed name mapped to the handles of all its parts: the route checks
    (:meth:`DirectWeightSyncDest._check_scales`, :meth:`~DirectWeightSyncDest._check_dequant`) apply to them."""
    if not parts:
        return all_handles
    out = dict(all_handles)
    for name, entries in parts.items():
        out[name] = list({id(h): h for *_, handles in entries for h in handles}.values())
    return out


def _lift(values: tuple, dims: tuple, fill) -> tuple:
    """``values`` (one per source dim) with ``fill`` inserted at each destination dim of ``dims`` (ascending)."""
    out = list(values)
    for d in dims:
        out.insert(d, fill)
    return tuple(out)


def _as_grid(scale: StridedMem, grid: tuple) -> StridedMem:
    """A contiguous scale window viewed with the shape of its :func:`scale_grid`."""
    return StridedMem(scale.ptr, grid, _contig(grid), scale.dtype, scale.device)


def _contig(shape) -> tuple:
    out, s = [], 1
    for e in reversed(shape):
        out.append(s)
        s *= e
    return tuple(reversed(out))
