"""Differential harness for the store path: drives the product store (sharded puts, ts.get, get_batch,
put_batch over several volumes) and ``oracle.reshard_oracle.OracleStore`` in lockstep and compares
every result, guard bytes of in-place destinations included.

The oracle only moves bytes, so it holds every tensor as a signed-integer view of the same itemsize;
the harness keeps each key's dtype and reinterprets.  A failure message carries the seed and the full
layout, so ``Layout.describe()`` is enough to replay it."""

from __future__ import annotations

import itertools
import os
import random
from collections import Counter
from dataclasses import dataclass

import numpy as np
import torch

import torchstore_b200 as ts
from oracle import reshard_oracle as ro
from tests.helpers import CAST_PAIRS, assert_equal_modulo_nan, bytes_of, random_bits
from tests.test_random_layouts import rand_layout, to_ts
from torchstore_b200 import _native
from torchstore_b200.rpc import ActorError
from torchstore_b200.transport import create_transport_buffer
from torchstore_b200.transport.types import Request

DTYPES = [torch.float32, torch.bfloat16, torch.float16, torch.float64, torch.int64, torch.int32, torch.int16,
          torch.uint8, torch.bool, torch.float8_e4m3fn, torch.complex64]
# pairs a CUDA destination converts through torch's copy_ because the fused cast has no kernel for them
TORCH_CAST_PAIRS = [
    (torch.bfloat16, torch.float64), (torch.float16, torch.float64), (torch.float64, torch.bfloat16),
    (torch.int32, torch.int64), (torch.float32, torch.int32), (torch.int16, torch.bfloat16),
    (torch.bfloat16, torch.float8_e4m3fn),
]
# shapes whose innermost run crosses 16-byte alignment and copy-tile boundaries
MEDIUM = [((257, 1030), torch.bfloat16), ((33, 7, 4099), torch.uint8), ((130, 517), torch.float32)]
EXTENTS = [1, 2, 3, 5, 7, 8, 9, 13]
_BITS = {1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}


def to_np(t: torch.Tensor) -> np.ndarray:
    """Bit pattern of a CPU tensor as a numpy integer array (what the oracle stores)."""
    return t.contiguous().view(_BITS[t.dtype.itemsize]).numpy().copy()


def from_np(a: np.ndarray, dtype: torch.dtype) -> torch.Tensor:
    return torch.from_numpy(np.array(a, order="C")).view(dtype)


def fill(shape, dtype: torch.dtype, gen: torch.Generator, finite: bool = False) -> torch.Tensor:
    """CPU tensor of `dtype`: random bit patterns (NaN payloads, signed zeros, denormals), or for
    `finite` small values that every destination dtype of the conversion tables holds exactly enough."""
    if dtype == torch.bool:
        return torch.randint(0, 2, shape, generator=gen).bool()
    if not finite:
        return random_bits(shape, dtype, gen)
    if dtype.is_floating_point:
        return (torch.randn(shape, generator=gen, dtype=torch.float64) * 8).to(dtype)
    lo = 0 if dtype == torch.uint8 else -100
    return torch.randint(lo, 100, shape, generator=gen).to(dtype)


@dataclass
class Layout:
    seed: int
    key: str
    shape: tuple
    dtype: torch.dtype
    smesh: tuple
    spl: list
    dmesh: tuple
    dpl: list
    cast_to: torch.dtype | None = None   # a conversion leg's destination dtype (values finite, in range)
    strided_src: bool = False

    @property
    def plain(self) -> bool:
        """All-replicated sources are plain puts into several volumes."""
        return all(p[0] == "R" for p in self.spl)

    @property
    def cast_class(self) -> str | None:
        if self.cast_to is None:
            return None
        return "fused" if _native.cast_supported(self.dtype, self.cast_to) else "torch"

    def describe(self) -> str:
        return (f"seed={self.seed} key={self.key} shape={self.shape} dtype={self.dtype} src_mesh={self.smesh} "
                f"src_placements={self.spl} dst_mesh={self.dmesh} dst_placements={self.dpl} cast_to={self.cast_to} "
                f"strided_src={self.strided_src}")


def store_layout(rng: random.Random, seed: int, key: str, medium: bool = False, cast: str | None = None,
                 dtype: torch.dtype | None = None) -> Layout:
    """One random layout.  cast: None (random), "none", "fused" or "torch" forces the conversion leg;
    `dtype` forces the stored dtype of a layout without one."""
    if medium:
        shape, dtype = rng.choice(MEDIUM)
    else:
        ndim = rng.choice([0, 1, 1, 2, 2, 3])
        shape, dtype = tuple(rng.choice(EXTENTS) for _ in range(ndim)), dtype or rng.choice(DTYPES)
    smesh, spl = rand_layout(rng, len(shape))
    dmesh, dpl = rand_layout(rng, len(shape))
    if cast is None and not medium:
        cast = rng.choice(["none", "none", "fused", "torch"])
    cast_to = None
    if cast in ("fused", "torch"):
        dtype, cast_to = rng.choice(CAST_PAIRS if cast == "fused" else TORCH_CAST_PAIRS)
    return Layout(seed, key, shape, dtype, smesh, spl, dmesh, dpl, cast_to, rng.random() < 0.4)


def _box(sl) -> tuple:
    return tuple(slice(o, o + s) for o, s in zip(sl.offsets, sl.local_shape))


def _window(shape, rng: random.Random):
    """(padded base shape, index of a `shape` window in it): non-contiguous unless every padded dim is
    outermost or of extent 1; a 0-d window is one element at an offset in a 1-D base."""
    pads = [rng.randint(1, 3) for _ in shape]
    starts = [rng.randint(0, p) for p in pads]
    idx = tuple(slice(a, a + s) for a, s in zip(starts, shape)) or (1,)
    return [s + p for s, p in zip(shape, pads)] or [3], idx


def _strided_copy(t: torch.Tensor, rng: random.Random, device: str) -> torch.Tensor:
    """The values of CPU tensor `t` as a strided view inside a padded buffer on `device`."""
    shape, idx = _window(tuple(t.shape), rng)
    base = torch.zeros(shape, dtype=t.dtype)
    base[idx] = t
    return base.to(device)[idx]


def _guarded(shape, dtype, gen, rng, strided: bool):
    """(CPU base buffer filled with guard values, index of the destination window in it)."""
    if not strided:
        return fill(shape, dtype, gen), ...
    base_shape, idx = _window(shape, rng)
    return fill(base_shape, dtype, gen), idx


class StoreHarness:
    """One product store (already initialised by the caller) and one OracleStore over `nvol` volumes.
    Rank r's shard goes to volume r % nvol, so one volume holds several shards of a key."""

    def __init__(self, nvol: int, devices: tuple, source_device: str, result_device: str = "cpu"):
        self.nvol = nvol
        self.devices = devices                # where in-place destinations live
        self.source_device = source_device
        self.result_device = result_device    # device of a fresh result
        self.oracle = ro.OracleStore(nvol)
        self.dtypes: dict[str, torch.dtype] = {}
        self.sources: dict[str, list] = {}    # key -> [(volume, Slice or None for a plain key, product source)]
        self.coverage: Counter = Counter()

    # ---- put ------------------------------------------------------------------------------------
    async def put_layout(self, lay: Layout, gen: torch.Generator, rng: random.Random):
        """Put every source shard of `lay`, rank r into volume r % nvol, into product and oracle."""
        full = fill(lay.shape, lay.dtype, gen, finite=lay.cast_to is not None)
        self.dtypes[lay.key] = lay.dtype
        self.sources[lay.key] = []
        regions = Counter()
        per_volume = Counter()
        coords = list(itertools.product(*(range(m) for m in lay.smesh)))
        if lay.plain:
            coords = coords[:self.nvol]  # one put per volume; more ranks only repeat the same bytes
        for rank, coord in enumerate(coords):
            sl = ro.make_slice(lay.shape, lay.smesh, coord, lay.spl)
            local = full[_box(sl)].contiguous()
            src = _strided_copy(local, rng, self.source_device) if lay.strided_src else local.to(self.source_device)
            vol = rank % self.nvol
            await self.put(vol, lay.key, src, local, None if lay.plain else sl)
            regions[(sl.offsets, sl.local_shape)] += 1
            per_volume[vol] += 1
            if 0 in sl.local_shape:
                self.coverage["empty_shard"] += 1
        if not lay.plain and any(n > 1 for n in per_volume.values()):
            self.coverage["several_shards_in_one_volume"] += 1
        if not lay.plain and any(n > 1 for n in regions.values()):
            self.coverage["replicated_dedup"] += 1
        self.coverage[f"dtype:{lay.dtype}"] += 1
        if not lay.shape:
            self.coverage["zero_dim"] += 1

    async def put(self, vol: int, key: str, src: torch.Tensor, cpu_values: torch.Tensor, tslice=None) -> None:
        """One put of `src` (values `cpu_values`) into volume `vol`: ts.put of a plain key, or what
        ts.put(key, dtensor) does on the mesh member whose LOCAL_RANK selects `vol`."""
        self.dtypes[key] = src.dtype
        self.sources.setdefault(key, []).append((vol, tslice, src))
        os.environ["LOCAL_RANK"] = str(vol)
        try:
            if tslice is None:
                await ts.put(key, src)
            else:
                c = await ts.client()
                req = Request(key=key, tensor_val=src, tensor_slice=to_ts(tslice))
                ref = c.strategy.select_storage_volume()
                await create_transport_buffer(ref).put_to_storage_volume([req])
                await c._controller.notify_put_batch.call([req.meta_only()], ref.volume_id)
        finally:
            os.environ["LOCAL_RANK"] = "0"
        self.oracle.put(vol, key, to_np(cpu_values), tslice)

    async def overwrite(self, key: str, gen: torch.Generator, dtype: torch.dtype | None = None, finite: bool = True):
        """Re-put every source of `key` with new values: into the same source tensors (an in-place
        overwrite in the volume) when `dtype` is unchanged, else from new tensors of `dtype`.  The new
        values are cut from one new global tensor, so replicas of a region stay equal."""
        dtype = dtype or self.dtypes[key]
        puts, self.sources[key] = self.sources[key], []
        vol, sl, src = puts[0]
        full = fill(tuple(src.shape) if sl is None else tuple(sl.global_shape), dtype, gen, finite)
        for vol, sl, src in puts:
            new = full if sl is None else full[_box(sl)].contiguous()
            if dtype == src.dtype:
                src.copy_(new.to(src.device))
            else:
                src = new.to(src.device)
            await self.put(vol, key, src, new, sl)

    # ---- get ------------------------------------------------------------------------------------
    def expected(self, key: str, want):
        """(expected CPU tensor in the stored dtype, None) or (None, the oracle's exception)."""
        try:
            return from_np(self.oracle.get(key, None, want), self.dtypes[key]), None
        except (RuntimeError, KeyError) as e:
            return None, e

    def make_dest(self, shape, dtype, kind: str, device: str, gen, rng):
        """kind: "contig" or "strided" -> (CPU copy of the base, device base, destination view)."""
        base, idx = _guarded(tuple(shape), dtype, gen, rng, kind == "strided")
        dev_base = base.clone().to(device)
        return base, dev_base, dev_base[idx], idx

    async def check_get(self, lay: Layout, want, kind: str, device: str | None, gen, rng):
        """One ts.get of `lay.key` (wanted slice `want`, None for the whole key) into a destination of
        `kind` ("none", "contig", "strided", "cast") on `device`; compared with the oracle."""
        sharded = "plain" if lay.plain else "sharded"
        ctx = f"{lay.describe()} want={want} dest={kind}/{device}"
        exp, err = self.expected(lay.key, want)
        stored = self.dtypes[lay.key]
        shape = tuple(want.local_shape) if want is not None else tuple(lay.shape)
        dtype = lay.cast_to if kind == "cast" else stored
        dest = None
        if kind != "none":
            strided = kind == "strided" or (kind == "cast" and rng.random() < 0.5)
            base, dev_base, dest, idx = self.make_dest(shape, dtype, "strided" if strided else "contig", device, gen, rng)
        try:
            got = await ts.get(lay.key, dest, to_ts(want) if want is not None else None)
        except Exception as e:
            if err is None:
                raise AssertionError(f"product raised {type(e).__name__}: {e} where the oracle did not; {ctx}") from e
            # the oracle restates the reference and raises client-side; the product raises the same
            # condition inside the volume's get endpoint, which the RPC layer re-raises as ActorError
            # (a RuntimeError), or client-side as RuntimeError when no stored rectangle intersects
            assert isinstance(e, RuntimeError), f"{type(e).__name__}: {e}; oracle raised {err!r}; {ctx}"
            if "not found in any stored shards" in str(err):
                assert isinstance(e, ActorError), f"{type(e).__name__}: {e}; {ctx}"
            self.coverage["error_parity"] += 1
            return
        assert err is None, f"oracle raised {err!r} but the product returned; {ctx}"
        if kind == "none":
            assert tuple(got.shape) == tuple(exp.shape) and got.dtype == exp.dtype, (tuple(got.shape), got.dtype, ctx)
            assert got.device.type == self.result_device, (got.device, ctx)
            assert np.array_equal(bytes_of(got), bytes_of(exp)), ctx
            self.coverage[f"dest:none:{sharded}"] += 1
            return
        assert got is dest, f"in-place get did not return the caller's tensor; {ctx}"
        self.assert_landed(lay.key, want, base, dev_base, idx, ctx)
        if kind == "cast":
            self.coverage[f"cast:{lay.cast_class}:{device}"] += 1
        self.coverage[f"dest:{kind}:{device}:{sharded}"] += 1

    def assert_landed(self, key: str, want, base: torch.Tensor, dev_base: torch.Tensor, idx, ctx: str) -> None:
        """The whole destination buffer `dev_base` equals its guard-filled CPU copy `base` with the
        oracle's result (converted to the buffer's dtype) in window `idx`: bit for bit when no
        conversion happened, else with every NaN encoding equal."""
        exp, err = self.expected(key, want)
        assert err is None, f"oracle raised {err!r}; {ctx}"
        want_base = base.clone()
        want_base[idx] = exp.to(base.dtype)
        try:
            assert_equal_modulo_nan(dev_base, want_base, cast=base.dtype != self.dtypes[key])
        except AssertionError as e:
            raise AssertionError(f"destination buffer differs from the oracle; {ctx}") from e

    def wanted(self, lay: Layout, rng: random.Random, n: int):
        """The whole key plus up to `n` destination-mesh slices."""
        coords = list(itertools.product(*(range(m) for m in lay.dmesh)))
        picked = rng.sample(coords, min(n, len(coords)))
        return [None] + [ro.make_slice(lay.shape, lay.dmesh, c, lay.dpl) for c in picked]

    def kinds(self, lay: Layout):
        out = [("none", None)] + [(k, d) for d in self.devices for k in ("contig", "strided")]
        if lay.cast_to is not None:
            out += [("cast", d) for d in self.devices]
        return out

    async def run_layout(self, lay: Layout, gen, rng, n_wanted: int = 3, gets_per_slice: int = 3):
        await self.put_layout(lay, gen, rng)
        for want in self.wanted(lay, rng, n_wanted):
            kinds = self.kinds(lay)
            picks = rng.sample(kinds, min(gets_per_slice, len(kinds)))
            if lay.cast_to is not None and not any(k == "cast" for k, _ in picks):
                picks[-1] = rng.choice([k for k in kinds if k[0] == "cast"])
            for kind, device in picks:
                await self.check_get(lay, want, kind, device, gen, rng)

    def required(self, cast_classes=("fused", "torch")) -> set:
        """Every bucket a run over this harness's devices must reach."""
        req = {"empty_shard", "several_shards_in_one_volume", "replicated_dedup", "error_parity", "zero_dim"}
        req |= {f"dtype:{d}" for d in DTYPES}
        for s in ("plain", "sharded"):
            req.add(f"dest:none:{s}")
            req |= {f"dest:{k}:{d}:{s}" for k in ("contig", "strided", "cast") for d in self.devices}
        req |= {f"cast:{c}:{d}" for c in cast_classes for d in self.devices}
        return req

    def assert_coverage(self, required: set | None = None) -> None:
        missing = sorted((required or self.required()) - set(self.coverage))
        assert not missing, f"differential run never reached {missing}; reached {dict(self.coverage)}"


async def run_differential(seed: int, n_layouts: int, devices: tuple, source_device: str, nvol: int = 3,
                           n_medium: int = 0, result_device: str = "cpu") -> StoreHarness:
    """`n_layouts` small random layouts (plus `n_medium` medium ones) through a store the caller has
    initialised with `nvol` LocalRankStrategy volumes."""
    rng = random.Random(seed)
    gen = torch.Generator().manual_seed(seed)
    h = StoreHarness(nvol, devices, source_device, result_device)
    order = rng.sample(DTYPES, len(DTYPES))
    for i in range(n_layouts + n_medium):
        # every fourth layout converts through the fused cast, every fourth through torch; the others
        # cycle through every dtype with random bit patterns
        medium = i >= n_layouts
        cast = "none" if medium else ("none", "fused", "none", "torch")[i % 4]
        lay = store_layout(rng, seed, f"k{i}", medium=medium, cast=cast, dtype=order[(i // 2) % len(order)])
        try:
            await h.run_layout(lay, gen, rng, n_wanted=2 if medium else 3)
        except AssertionError:
            raise
        except Exception as e:
            raise AssertionError(f"{type(e).__name__}: {e} -- {lay.describe()}") from e
    return h
