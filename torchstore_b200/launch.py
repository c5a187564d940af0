"""Work on the library's per-device copy stream: fencing it behind the caller's stream, one-shot
copies, host<->device staging copies, compiled plans and their lifetime, and awaiting completion
from an event loop.  The rest of the package calls these instead of the plan and copy entry points
of ``_native``."""

from __future__ import annotations

import asyncio
import functools
import logging
import threading

from torchstore_b200 import _native
from torchstore_b200.planner import build_rects, build_transpose_rects

logger = logging.getLogger(__name__)


async def _poll(done) -> None:
    """Await ``done()`` without blocking the actor's event loop (the reference awaits RDMA
    completions the same way: everything on the path is a coroutine).  Every poll goes through the
    loop's selector, which drops the GIL, so actor-server threads keep running.  (Polling the last
    stretch without yielding was tried and measured no gain: 0.048 vs 0.049 ms of host time per sync.)"""
    spins = 0
    while not done():
        spins += 1
        await asyncio.sleep(0 if spins < 4000 else 0.0002)


_fence_events = threading.local()


def fence_in(device: int) -> None:
    """Copy stream waits for whatever torch has queued on the caller's current stream.  One reusable
    event per (thread, device): cudaStreamWaitEvent snapshots the record it follows, so a later
    record on the same event does not disturb earlier waits."""
    cache = getattr(_fence_events, "by_device", None)
    if cache is None:
        cache = _fence_events.by_device = {}
    ev = cache.get(device)
    if ev is None:
        ev = cache[device] = _native.Event(device)
    ev.record(_native.torch_stream(device))
    ev.wait_on(device, None)


def staging_copy(device: int, dst: int, src: int, nbytes: int, kind: int) -> None:
    """Async host<->device copy of ``nbytes`` (``kind``: ``_native.TSB_H2D`` or ``TSB_D2H``) on
    ``device``'s copy stream, fenced in behind the caller's stream: it reads what the caller queued
    before it, and a write the caller queued on the destination cannot land after it.  A copy of zero
    bytes (an empty tensor, whose data pointer torch reports as null) is not issued."""
    if nbytes == 0:
        return
    fence_in(device)
    _native.memcpy_async(device, dst, src, nbytes, kind)


async def wait_copy_stream(device: int) -> None:
    """Await everything queued so far on ``device``'s copy stream."""
    done = _native.Event(device).record(None)
    await _poll(done.query)
    done.close()


def copy_once(per_device: dict[int, list], fence: bool = True) -> set[int]:
    """One copy_rects launch per device of ``{device: [(src, dst) StridedMem windows]}``, fenced
    behind the caller's stream unless ``fence=False``.  Returns the devices to wait on."""
    for dev, pairs in per_device.items():
        rects, n = build_rects(pairs)
        if fence:
            fence_in(dev)
        _native.copy_rects(dev, rects, n)
    return set(per_device)


class Plans(dict):
    """Compiled native plans, one per device: ``{device: plan id}``.  Closed explicitly, never by a
    finalizer: destroying a plan frees device memory, which must not happen at an arbitrary
    garbage-collection point."""

    @classmethod
    def build(cls, per_device: dict[int, list]) -> "Plans":
        """Compile ``{device: [(src, dst) StridedMem windows]}``."""
        plans = cls()
        try:
            for dev, pairs in per_device.items():
                rects, n = build_rects(pairs)
                plans[dev] = _native.plan_create(dev, rects, n)
        except BaseException:
            plans.close()
            raise
        return plans

    @classmethod
    def build_fp8(cls, create, per_device: dict[int, tuple], flags: int = 0) -> "Plans":
        """Compile scaled fp8 plans: ``create(device, *args, flags=flags)`` for each ``{device: args}``, ``create``
        being one of the ``_native.*_plan_create`` calls (``flags``: ``_native.TSB_QUANT_UE8M0`` or 0)."""
        plans = cls()
        try:
            for dev, args in per_device.items():
                plans[dev] = create(dev, *args, flags=flags)
        except BaseException:
            plans.close()
            raise
        return plans

    @classmethod
    def _build_pulls(cls, create, per_device: dict[int, tuple], flags: int = 0, quantise: bool = False,
                     dequantise: bool = False) -> "Plans":
        """build_fp8 of pulls: ``{device: ([(src, dst) StridedMem windows], *tables)}``, the windows as rects
        (``quantise``: an int8 destination window is quantised; ``dequantise``: an int8 source window is
        dequantised; see :func:`build_rects`)."""
        return cls.build_fp8(create, {dev: (*build_rects(pairs, quantise, dequantise), *tables) for dev, (pairs, *tables) in
                                      per_device.items()}, flags)

    @classmethod
    def build_block_fp8(cls, per_device: dict[int, tuple[list, list]], flags: int = 0) -> "Plans":
        """Compile block-scaled fp8 pulls: ``{device: ([(src, dst) StridedMem windows], [BqTarget])}``; ``flags``:
        ``_native.TSB_QUANT_UE8M0`` for power-of-two scales, here and in the other quantising builders.  Windows
        into int8 destinations quantise into int8 (one plan writes one destination dtype), here and in
        :meth:`build_scaled_fp8`."""
        return cls._build_pulls(_native.block_fp8_plan_create, per_device, flags, quantise=True)

    @classmethod
    def build_scaled_fp8(cls, per_device: dict[int, tuple[list, list]], flags: int = 0) -> "Plans":
        """Compile per-channel / per-tensor scaled fp8 pulls: ``{device: ([(src, dst) StridedMem windows],
        [SqTarget])}``."""
        return cls._build_pulls(_native.scaled_fp8_plan_create, per_device, flags, quantise=True)

    @classmethod
    def build_dequant_fp8(cls, per_device: dict[int, tuple[list, list]]) -> "Plans":
        """Compile dequantising pulls of scaled fp8 (or int8) sources: ``{device: ([(src, dst) StridedMem windows],
        [DqSource])}``; one plan reads one source format."""
        return cls._build_pulls(_native.dequant_fp8_plan_create, per_device, dequantise=True)

    @classmethod
    def build_requant_fp8(cls, per_device: dict[int, tuple[list, list, list]], flags: int = 0) -> "Plans":
        """Compile requantising pulls of scaled fp8 sources into scaled fp8 destinations: ``{device:
        ([(src, dst) StridedMem windows], [DqSource], [SqTarget])}``."""
        return cls._build_pulls(_native.requant_fp8_plan_create, per_device, flags)

    @classmethod
    def build_transpose(cls, per_device: dict[int, list]) -> "Plans":
        """Compile transposing pulls: ``{device: [(src, dst) StridedMem windows]}``, each window's destination
        contiguous along its dim -1 and its source along dim -2 (:func:`build_transpose_rects`)."""
        return cls.build_fp8(lambda dev, rects, n, flags: _native.transpose_plan_create(dev, rects, n, flags),
                             {dev: build_transpose_rects(pairs) for dev, pairs in per_device.items()})

    @classmethod
    def build_source_quant(cls, per_device: dict[int, list], flags: int = 0,
                           dst_dtype: int = _native.TSB_F8E4M3) -> "Plans":
        """Compile source-side quantisations: ``{device: [SourceQuantTarget]}`` into ``dst_dtype`` staging
        (``_native.TSB_F8E4M3`` or ``_native.TSB_I8``)."""
        def create(dev, targets, flags):
            return _native.source_quant_plan_create(dev, targets, flags, dst_dtype)

        return cls.build_fp8(create, {dev: (targets,) for dev, targets in per_device.items()}, flags)

    def launch(self, fence_out: bool = True) -> None:
        """Enqueue every plan on its device's copy stream, fenced in against the caller's current
        stream of that device.  ``fence_out=False``: the caller's stream is not made to wait for the
        copy (puts: the source is only read, and completion is observed on the host)."""
        for dev, plan in self.items():
            _native.plan_launch(plan, _native.torch_stream(dev), fence_out=fence_out)

    async def wait(self) -> None:
        for plan in self.values():
            await _poll(functools.partial(_native.plan_poll, plan))

    def synchronize(self) -> None:
        """Block the calling thread until the last launch of every plan has finished."""
        for plan in self.values():
            _native.plan_wait(plan)

    def elapsed_ms(self) -> dict[int, float]:
        """Device time of each plan's last launch."""
        return {dev: _native.plan_elapsed_ms(plan) for dev, plan in self.items()}

    def info(self) -> dict[int, dict]:
        return {dev: _native.plan_info(plan).as_dict() for dev, plan in self.items()}

    def close(self) -> None:
        for plan in self.values():
            try:
                _native.plan_destroy(plan)
            except Exception as e:
                logger.warning("plan_destroy failed: %s", e)
        self.clear()
