"""The store path on HBM volumes against the oracle store (tests/store_harness.py): random layouts with
uneven, empty and replicated shards over three volumes, CUDA sources, fresh / contiguous / strided /
converting destinations on the CPU and on the GPU, medium shapes that reach both copy modes of the
kernel, TORCHSTORE_B200_GET_DEVICE=cuda, and fast-lane replays after in-place overwrites and layout
changes."""

import random

import pytest
import torch

import torchstore_b200 as ts
from tests.helpers import DEV, run
from tests.store_harness import (DTYPES, TORCH_CAST_PAIRS, Layout, StoreHarness, _strided_copy, fill, run_differential,
                                 store_layout, to_np)
from tests.test_random_layouts import to_ts

pytestmark = pytest.mark.gpu
NVOL = 3


@pytest.fixture(autouse=True)
def _env(monkeypatch):
    monkeypatch.delenv("RANK", raising=False)
    monkeypatch.setenv("LOCAL_RANK", "0")
    monkeypatch.delenv("TORCHSTORE_B200_GET_DEVICE", raising=False)
    yield


async def _store(body):
    await ts.initialize(num_storage_volumes=NVOL, strategy=ts.LocalRankStrategy())
    try:
        return await body()
    finally:
        await ts.shutdown()


@pytest.mark.parametrize("seed", range(3))
def test_store_matches_oracle_across_random_layouts_on_hbm_volumes(seed):
    h = run(_store(lambda: run_differential(2000 + seed, 36, devices=("cpu", "cuda"), source_device=DEV, n_medium=3)))
    h.assert_coverage()


def test_fresh_results_on_the_gpu_match_oracle(monkeypatch):
    """TORCHSTORE_B200_GET_DEVICE=cuda: a get without a destination returns a CUDA tensor."""
    monkeypatch.setenv("TORCHSTORE_B200_GET_DEVICE", "cuda")
    h = run(_store(lambda: run_differential(3000, 24, devices=("cuda",), source_device=DEV, result_device="cuda")))
    h.assert_coverage({"dest:none:plain", "dest:none:sharded", "dest:strided:cuda:sharded", "error_parity"})


def test_cuda_destinations_without_a_fused_cast_are_converted_like_copy_():
    """A CUDA destination whose dtype pair has no fused-cast kernel gets the stored values converted by
    torch (the reference's client_tensor.copy_), for plain and sharded keys, contiguous and strided."""
    async def body():
        rng, gen = random.Random(11), torch.Generator().manual_seed(11)
        h = StoreHarness(NVOL, ("cuda",), DEV)
        for i, (src, dst) in enumerate(TORCH_CAST_PAIRS):
            for j, placements in enumerate(([("R",)], [("S", 0)], [("S", 1)])):
                lay = Layout(11, f"c{i}_{j}", (9, 13), src, (3,), placements, (2,), [("S", 1)], dst)
                await h.put_layout(lay, gen, rng)
                for want in h.wanted(lay, rng, 2):
                    for kind in ("contig", "strided"):
                        base, dev_base, dest, idx = h.make_dest(want.local_shape if want else lay.shape, dst, kind, DEV,
                                                                gen, rng)
                        got = await ts.get(lay.key, dest, None if want is None else to_ts(want))
                        assert got is dest
                        h.assert_landed(lay.key, want, base, dev_base, idx, f"{lay.describe()} want={want} {kind}")

    run(_store(body))


async def _replay_set(h: StoreHarness, rng, gen, n_plain: int, n_sharded: int, dtypes):
    """Keys whose whole-key get succeeds (no empty shard): plain keys each in one volume, and sharded
    keys across volumes; every key with an in-place CUDA destination (contiguous or strided, of the
    stored dtype or of a dtype the fused cast converts to)."""
    lays, i = [], 0
    while sum(lay.plain for lay in lays) < n_plain or sum(not lay.plain for lay in lays) < n_sharded:
        lay = store_layout(rng, 0, f"f{i}", cast=rng.choice(["none", "fused"]), dtype=rng.choice(dtypes))
        i += 1
        if lay.dtype not in dtypes or (lay.cast_to is not None and lay.cast_to not in dtypes) or not lay.shape:
            continue
        if lay.plain and sum(x.plain for x in lays) >= n_plain or not lay.plain and sum(not x.plain for x in lays) >= n_sharded:
            continue
        if lay.plain:
            # each plain key lives in one volume, so a layout change moves one volume's epoch only
            lay.smesh = (1,)
            full = fill(lay.shape, lay.dtype, gen, finite=True)
            src = _strided_copy(full, rng, DEV) if lay.strided_src else full.to(DEV)
            await h.put(sum(x.plain for x in lays) % NVOL, lay.key, src, full)
        else:
            await h.put_layout(lay, gen, rng)
            if h.expected(lay.key, None)[1] is not None:
                continue
        lays.append(lay)
    dests = {}
    for lay in lays:
        dests[lay.key] = h.make_dest(lay.shape, lay.cast_to or lay.dtype, rng.choice(["contig", "strided"]), DEV, gen, rng)
    return lays, dests


async def _get_batch_and_check(h: StoreHarness, dests: dict, ctx: str):
    out = await ts.get_batch({k: d[2] for k, d in dests.items()})
    for key, (base, dev_base, dest, idx) in dests.items():
        assert out[key] is dest, f"{key}: not the caller's tensor; {ctx}"
        h.assert_landed(key, None, base, dev_base, idx, f"{key} {ctx}")


def test_get_batch_replays_after_in_place_overwrites_and_not_after_a_layout_change():
    floats = [torch.float32, torch.bfloat16, torch.float16]

    async def body():
        rng, gen = random.Random(21), torch.Generator().manual_seed(21)
        h = StoreHarness(NVOL, ("cuda",), DEV)
        lane = (await ts.client()).fast_lane
        lays, dests = await _replay_set(h, rng, gen, n_plain=NVOL, n_sharded=4, dtypes=floats)
        await _get_batch_and_check(h, dests, "recording get_batch")
        assert len(lane.get_sessions) == 1
        # 1. every source overwritten in place (same shapes and dtypes: no epoch moves) -> replay
        for lay in lays:
            await h.overwrite(lay.key, gen)
        hits = lane.get_hits
        await _get_batch_and_check(h, dests, "replay after in-place overwrites")
        assert lane.get_hits == hits + 1
        # 2. one volume at a time, re-put a key that lives only there in another dtype: the volume
        # reallocates and its layout epoch moves, so the next get_batch must not replay
        for vol in range(NVOL):
            lay = next(x for x in lays if x.plain and h.sources[x.key][0][0] == vol)
            new = next(d for d in floats if d != h.dtypes[lay.key])
            await h.overwrite(lay.key, gen, dtype=new)
            hits = lane.get_hits
            await _get_batch_and_check(h, dests, f"after {lay.key} in volume {vol} became {new}")
            assert lane.get_hits == hits, f"replayed a session recorded before volume {vol} reallocated {lay.key}"
            await _get_batch_and_check(h, dests, "re-recorded get_batch")
            assert lane.get_hits == hits + 1

    run(_store(body))


def test_get_batch_with_a_torch_converted_destination_is_not_replayed():
    """Its result depends on a torch copy_ after the plan, so the batch records no session; repeated
    after an in-place overwrite it still equals the oracle."""
    async def body():
        rng, gen = random.Random(31), torch.Generator().manual_seed(31)
        h = StoreHarness(NVOL, ("cuda",), DEV)
        lane = (await ts.client()).fast_lane
        lays, dests = await _replay_set(h, rng, gen, n_plain=2, n_sharded=2, dtypes=[torch.float32, torch.bfloat16])
        src, dst = torch.bfloat16, torch.float64
        lay = Layout(31, "torch_cast", (6, 10), src, (2,), [("S", 0)], (1,), [("R",)], dst)
        await h.put_layout(lay, gen, rng)
        dests[lay.key] = h.make_dest(lay.shape, dst, "strided", DEV, gen, rng)
        for _ in range(2):
            sessions, hits = len(lane.get_sessions), lane.get_hits
            await _get_batch_and_check(h, dests, "batch with a bf16 -> f64 destination")
            assert len(lane.get_sessions) == sessions and lane.get_hits == hits
            for x in lays + [lay]:
                await h.overwrite(x.key, gen)

    run(_store(body))


def test_put_batch_of_strided_sources_replays_and_reads_back():
    """An identical put_batch of plain keys (random dtypes, non-contiguous CUDA sources) replays; what
    later gets return equals the oracle."""
    async def body():
        rng, gen = random.Random(41), torch.Generator().manual_seed(41)
        h = StoreHarness(NVOL, ("cpu", "cuda"), DEV)
        lane = (await ts.client()).fast_lane
        shapes = {f"p{i}": tuple(rng.choice([3, 7, 16, 33]) for _ in range(rng.choice([1, 2, 3]))) for i in range(11)}
        dtypes = {k: DTYPES[i % len(DTYPES)] for i, k in enumerate(shapes)}
        values = {k: fill(s, dtypes[k], gen) for k, s in shapes.items()}
        srcs = {}
        for k, v in values.items():  # every other element of a buffer twice the size
            buf = torch.zeros(*v.shape, 2, dtype=v.dtype)
            buf[..., 0] = v
            srcs[k] = buf.to(DEV)[..., 0]
        assert not any(s.is_contiguous() for s in srcs.values())
        for round_ in range(2):
            misses, hits = lane.put_misses, lane.put_hits
            await ts.put_batch(srcs)
            for k in srcs:
                h.oracle.put(0, k, to_np(values[k]))
                h.dtypes[k] = dtypes[k]
            assert (lane.put_misses, lane.put_hits) == ((misses + 1, hits) if round_ == 0 else (misses, hits + 1))
            for k, s in shapes.items():
                lay = Layout(41, k, s, dtypes[k], (1,), [("R",)], (2,), [("S", 0)])
                for kind, dev in (("none", None), ("strided", "cuda"), ("contig", "cpu")):
                    await h.check_get(lay, None, kind, dev, gen, rng)
            for k in srcs:
                values[k] = fill(shapes[k], dtypes[k], gen)
                srcs[k].copy_(values[k].to(DEV))

    run(_store(body))
