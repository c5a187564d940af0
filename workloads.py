"""Synthetic weight-sync workloads shared by bench.py, tools/ and the tests: Llama-3 state-dict
layouts (shapes + the torchtitan TP plan of SURVEY.md section 8) and their FSDP/TP rectangles, the
same model under its Hugging Face names, a small Qwen3-MoE-style model, and the vLLM tensor-parallel
layout a generator holds for either (fused qkv_proj / gate_up_proj, stacked experts) as packed parts
of the Hugging Face tensors.  Metadata only -- no tensors are created here."""

from __future__ import annotations

import math

LLAMA3_8B = dict(name="llama3-8b", dim=4096, n_layers=32, n_heads=32, n_kv_heads=8, vocab=128256, ffn=14336)
LLAMA3_70B = dict(name="llama3-70b", dim=8192, n_layers=80, n_heads=64, n_kv_heads=8, vocab=128256, ffn=28672)
# Qwen3-30B-A3B's shapes (head_dim 128, so the q rows are 32 * 128 = 4096 against a hidden size of 2048)
QWEN3_MOE = dict(name="qwen3-moe", dim=2048, n_layers=48, n_heads=32, n_kv_heads=4, head_dim=128, vocab=151936,
                 n_experts=128, moe_ffn=768)


def llama_layout(cfg=LLAMA3_8B, n_layers: int | None = None, scale: int = 1, with_embeddings: bool = True):
    """name -> (global shape, TP placement) with placement ("S", dim) or ("R",).

    ColwiseParallel (Shard(0)): wq wk wv w1 w3, output; RowwiseParallel embedding: Shard(0);
    RowwiseParallel linear (Shard(1)): wo w2; norms replicated.  `scale` divides every dimension."""
    d = cfg["dim"] // scale
    kv = cfg["dim"] // cfg["n_heads"] * cfg["n_kv_heads"] // scale
    ffn = cfg["ffn"] // scale
    vocab = cfg["vocab"] // scale
    layers = cfg["n_layers"] if n_layers is None else n_layers
    out = {}
    if with_embeddings:
        out["tok_embeddings.weight"] = ((vocab, d), ("S", 0))
    for i in range(layers):
        p = f"layers.{i}."
        out[p + "attention.wq.weight"] = ((d, d), ("S", 0))
        out[p + "attention.wk.weight"] = ((kv, d), ("S", 0))
        out[p + "attention.wv.weight"] = ((kv, d), ("S", 0))
        out[p + "attention.wo.weight"] = ((d, d), ("S", 1))
        out[p + "feed_forward.w1.weight"] = ((ffn, d), ("S", 0))
        out[p + "feed_forward.w2.weight"] = ((d, ffn), ("S", 1))
        out[p + "feed_forward.w3.weight"] = ((ffn, d), ("S", 0))
        out[p + "attention_norm.weight"] = ((d,), ("R",))
        out[p + "ffn_norm.weight"] = ((d,), ("R",))
    if with_embeddings:
        out["norm.weight"] = ((d,), ("R",))
        out["output.weight"] = ((vocab, d), ("S", 0))
    return out


def shard_box(shape, n: int, rank: int, placement):
    """(offsets, local_shape) of `rank` on a 1-D mesh of size n; even or torch.chunk-style uneven."""
    offsets = [0] * len(shape)
    local = list(shape)
    if placement[0] == "S":
        dim = placement[1]
        size = shape[dim]
        chunk = -(-size // n)
        start = min(size, chunk * rank)
        stop = min(size, chunk * (rank + 1))
        offsets[dim] = start if stop > start else size
        local[dim] = max(0, stop - start)
    return tuple(offsets), tuple(local)


def state_dict_bytes(layout, itemsize: int = 2) -> int:
    return sum(math.prod(shape) for shape, _ in layout.values()) * itemsize


def fsdp_to_tp_rects(layout, n: int, dest_rank: int, itemsize: int = 2):
    """Rectangles dest_rank pulls for FSDP(n) Shard(0) -> TP(n): list of
    (name, src_rank, src_index, dst_index, exact) with index = tuple of (start, stop) per dim,
    in the reference's plan order (dest param major, source rank minor, replicated dedup)."""
    out = []
    for name, (shape, tp) in layout.items():
        d_off, d_shape = shard_box(shape, n, dest_rank, tp) if n > 1 else ((0,) * len(shape), tuple(shape))
        seen = set()
        for s in range(n):
            s_off, s_shape = shard_box(shape, n, s, ("S", 0))
            lo = [max(a, b) for a, b in zip(s_off, d_off)]
            hi = [min(a + x, b + y) for a, x, b, y in zip(s_off, s_shape, d_off, d_shape)]
            if any(h <= l for l, h in zip(lo, hi)):
                continue
            key = (tuple(lo), tuple(h - l for l, h in zip(lo, hi)))
            if key in seen:
                continue
            seen.add(key)
            exact = tuple(s_off) == tuple(d_off) and tuple(s_shape) == tuple(d_shape)
            src_idx = tuple((l - o, h - o) for l, h, o in zip(lo, hi, s_off))
            dst_idx = tuple((l - o, h - o) for l, h, o in zip(lo, hi, d_off))
            out.append((name, s, src_idx, dst_idx, exact))
    return out


_HF_LLAMA = {"attention.wq": "self_attn.q_proj", "attention.wk": "self_attn.k_proj", "attention.wv": "self_attn.v_proj",
             "attention.wo": "self_attn.o_proj", "feed_forward.w1": "mlp.gate_proj", "feed_forward.w2": "mlp.down_proj",
             "feed_forward.w3": "mlp.up_proj", "attention_norm": "input_layernorm", "ffn_norm": "post_attention_layernorm"}


def hf_name(name: str) -> str:
    """The Hugging Face name of a :func:`llama_layout` (torchtitan) name."""
    if name.startswith("layers."):
        _, i, rest = name.split(".", 2)
        return f"model.layers.{i}.{_HF_LLAMA[rest.removesuffix('.weight')]}.weight"
    return {"tok_embeddings.weight": "model.embed_tokens.weight", "norm.weight": "model.norm.weight",
            "output.weight": "lm_head.weight"}[name]


def hf_llama_layout(cfg=LLAMA3_8B, n_layers: int | None = None, scale: int = 1, with_embeddings: bool = True):
    """:func:`llama_layout` under the Hugging Face names a trainer of an HF-layout model publishes
    (``model.layers.{i}.self_attn.q_proj.weight``, ``mlp.gate_proj``, ``model.embed_tokens``, ``lm_head``, ...):
    the same shapes and placements, in the same order."""
    return {hf_name(name): entry for name, entry in llama_layout(cfg, n_layers, scale, with_embeddings).items()}


def qwen3_moe_layout(cfg=QWEN3_MOE, n_layers: int | None = None, scale: int = 1, with_embeddings: bool = True,
                     n_experts: int | None = None, grouped_experts: bool = False):
    """A Qwen3-MoE model under its Hugging Face names: name -> (global shape, placement), as :func:`llama_layout`
    (the placements are those of an FSDP-style trainer's view and do not matter for packed pulls).  Per layer: q/k/v/o
    projections with q_norm / k_norm, the router ``mlp.gate``, and one gate/up/down projection per expert.
    ``scale`` divides hidden size, head_dim, expert width and vocabulary; ``n_experts`` overrides the expert count.
    ``grouped_experts`` replaces each layer's per-expert tensors by the input-major stacks of a grouped-GEMM trainer
    (the layout ``torch._grouped_mm(x, w)`` takes without a transpose), placement Shard(0):
    ``mlp.experts.w1`` / ``mlp.experts.w3`` ``[E, dim, moe_ffn]`` and ``mlp.experts.w2`` ``[E, moe_ffn, dim]``."""
    d, hd = cfg["dim"] // scale, cfg["head_dim"] // scale
    q, kv, ffn = cfg["n_heads"] * hd, cfg["n_kv_heads"] * hd, cfg["moe_ffn"] // scale
    experts = cfg["n_experts"] if n_experts is None else n_experts
    layers = cfg["n_layers"] if n_layers is None else n_layers
    out = {}
    if with_embeddings:
        out["model.embed_tokens.weight"] = ((cfg["vocab"] // scale, d), ("S", 0))
    for i in range(layers):
        p = f"model.layers.{i}."
        out[p + "self_attn.q_proj.weight"] = ((q, d), ("S", 0))
        out[p + "self_attn.k_proj.weight"] = ((kv, d), ("S", 0))
        out[p + "self_attn.v_proj.weight"] = ((kv, d), ("S", 0))
        out[p + "self_attn.o_proj.weight"] = ((d, q), ("S", 1))
        out[p + "self_attn.q_norm.weight"] = ((hd,), ("R",))
        out[p + "self_attn.k_norm.weight"] = ((hd,), ("R",))
        out[p + "mlp.gate.weight"] = ((experts, d), ("R",))
        if grouped_experts:
            out[p + "mlp.experts.w1"] = ((experts, d, ffn), ("S", 0))
            out[p + "mlp.experts.w3"] = ((experts, d, ffn), ("S", 0))
            out[p + "mlp.experts.w2"] = ((experts, ffn, d), ("S", 0))
        for e in range(0 if grouped_experts else experts):
            out[p + f"mlp.experts.{e}.gate_proj.weight"] = ((ffn, d), ("S", 0))
            out[p + f"mlp.experts.{e}.up_proj.weight"] = ((ffn, d), ("S", 0))
            out[p + f"mlp.experts.{e}.down_proj.weight"] = ((d, ffn), ("S", 1))
        out[p + "input_layernorm.weight"] = ((d,), ("R",))
        out[p + "post_attention_layernorm.weight"] = ((d,), ("R",))
    if with_embeddings:
        out["model.norm.weight"] = ((d,), ("R",))
        out["lm_head.weight"] = ((cfg["vocab"] // scale, d), ("S", 0))
    return out


def vllm_tp_layout(hf_layout, cfg, tp: int, rank: int, ep: bool = False, source: str = "hf"):
    """What vLLM tensor-parallel rank ``rank`` of ``tp`` holds for ``hf_layout`` (:func:`hf_llama_layout` or
    :func:`qwen3_moe_layout` of ``cfg``): vLLM name -> (local shape, parts, box).

    ``source="torchtitan"`` reads a torchtitan trainer instead: ``hf_layout`` is then a :func:`llama_layout`
    (``layers.{i}.attention.wq.weight``, ...), and every vLLM parameter is a packed destination whose parts read the
    torchtitan names (wq / wk / wv into ``qkv_proj``, w1 / w3 into ``gate_up_proj``, and one part per renamed tensor:
    wo, w2, tok_embeddings, output and the norms).  The q and k parts carry ``rotary_head_dim = dim / n_heads``:
    torchtitan keeps Meta's interleaved rotary rows, vLLM (like Hugging Face) the half-split ones.

    * Fused parameters have ``parts``, a tuple of ``PackedPart`` reading the HF tensors, and ``box`` None:
      ``qkv_proj`` = ``[q_r; k_r; v_r]`` (rank r's query heads, then its kv head(s): when tp exceeds the kv heads,
      kv head ``r // (tp / n_kv)``, as vLLM replicates them), ``gate_up_proj`` = ``[gate_r; up_r]``, and for MoE
      ``mlp.experts.w13_weight [E, 2I/tp, H]`` / ``w2_weight [E, H, I/tp]`` with every expert stacked on dim 0.
      With ``ep`` the experts are split over the ranks instead (``E/tp`` whole experts each).  From a
      ``qwen3_moe_layout(grouped_experts=True)`` both are filled by transposed parts (``PackedPart(transpose=True)``)
      of the input-major stacks: ``w13_weight`` from ``w1`` and ``w3``, ``w2_weight`` from ``w2``, one part each.
    * Every other parameter keeps its HF name: ``parts`` None and ``box`` = (global offsets, global shape) of the
      rank's shard of that tensor: ``o_proj`` / ``down_proj`` column shards, vocab-parallel ``embed_tokens`` /
      ``lm_head`` row shards, replicated norms and router."""
    from torchstore_b200.direct_weight_sync import PackedPart

    if source == "torchtitan":
        return _from_torchtitan(hf_layout, cfg, tp, rank, ep)
    if source != "hf":
        raise ValueError(f"source must be 'hf' or 'torchtitan', not {source!r}")
    n_heads, n_kv = cfg["n_heads"], cfg["n_kv_heads"]
    if n_heads % tp or (n_kv % tp and tp % n_kv):
        raise ValueError(f"tp={tp} must divide {n_heads} query heads and divide or be a multiple of {n_kv} kv heads")
    out = {}
    for name, (shape, _) in hf_layout.items():
        mod = name.removesuffix(".weight")
        if mod.endswith("self_attn.q_proj"):
            base = mod.removesuffix("q_proj")
            qs, h = shape
            kvs = hf_layout[base + "k_proj.weight"][0][0]
            hd = qs // n_heads
            q_r = qs // tp
            if tp <= n_kv:
                kv_r, kv0 = kvs // tp, rank * (kvs // tp)
            else:
                kv_r, kv0 = hd, rank // (tp // n_kv) * hd
            parts = (PackedPart(name, (slice(0, q_r), slice(0, h)), (rank * q_r, 0)),
                     PackedPart(base + "k_proj.weight", (slice(q_r, q_r + kv_r), slice(0, h)), (kv0, 0)),
                     PackedPart(base + "v_proj.weight", (slice(q_r + kv_r, q_r + 2 * kv_r), slice(0, h)), (kv0, 0)))
            out[base + "qkv_proj.weight"] = ((q_r + 2 * kv_r, h), parts, None)
        elif mod.endswith(("self_attn.k_proj", "self_attn.v_proj", "mlp.up_proj")) or ".experts." in mod:
            continue  # read by the fused parameters
        elif mod.endswith("mlp.gate_proj"):
            base = mod.removesuffix("gate_proj")
            ffn, h = shape
            f_r = ffn // tp
            parts = (PackedPart(name, (slice(0, f_r), slice(0, h)), (rank * f_r, 0)),
                     PackedPart(base + "up_proj.weight", (slice(f_r, 2 * f_r), slice(0, h)), (rank * f_r, 0)))
            out[base + "gate_up_proj.weight"] = ((2 * f_r, h), parts, None)
        elif mod.endswith("mlp.gate") and "n_experts" in cfg:
            out[name] = (tuple(shape), None, ((0,) * len(shape), tuple(shape)))  # the router, replicated
            base = mod.removesuffix("gate")
            n_exp = shape[0]
            if base + "experts.w1" in hf_layout:
                out.update(_grouped_experts(base, hf_layout[base + "experts.w1"][0], tp, rank, ep))
                continue
            ffn, h = hf_layout[base + "experts.0.gate_proj.weight"][0]
            if ep:
                if n_exp % tp:
                    raise ValueError(f"ep over tp={tp} ranks needs the {n_exp} experts to split evenly")
                mine, f_r, f0 = range(rank * n_exp // tp, (rank + 1) * n_exp // tp), ffn, 0
            else:
                mine, f_r, f0 = range(n_exp), ffn // tp, rank * (ffn // tp)
            w13, w2 = [], []
            for j, e in enumerate(mine):
                ex = f"{base}experts.{e}."
                w13 += [PackedPart(ex + "gate_proj.weight", (j, slice(0, f_r), slice(0, h)), (f0, 0)),
                        PackedPart(ex + "up_proj.weight", (j, slice(f_r, 2 * f_r), slice(0, h)), (f0, 0))]
                w2.append(PackedPart(ex + "down_proj.weight", (j, slice(0, h), slice(0, f_r)), (0, f0)))
            out[base + "experts.w13_weight"] = ((len(mine), 2 * f_r, h), tuple(w13), None)
            out[base + "experts.w2_weight"] = ((len(mine), h, f_r), tuple(w2), None)
        else:
            if mod.endswith(("o_proj", "down_proj")):
                placement = ("S", 1)
            elif mod.endswith(("embed_tokens", "lm_head")):
                placement = ("S", 0)
            else:
                placement = ("R",)
            off, loc = shard_box(shape, tp, rank, placement) if tp > 1 else ((0,) * len(shape), tuple(shape))
            out[name] = (tuple(loc), None, (tuple(off), tuple(shape)))
    return out


def _grouped_experts(base: str, w1_shape, tp: int, rank: int, ep: bool):
    """:func:`vllm_tp_layout`'s ``w13_weight`` / ``w2_weight`` of rank ``rank`` from grouped-GEMM stacks ``w1`` / ``w3``
    ``[E, H, I]`` and ``w2`` ``[E, I, H]`` (``w1_shape``): transposed parts, TP slicing the ffn dim or EP the experts."""
    from torchstore_b200.direct_weight_sync import PackedPart

    n_exp, h, ffn = w1_shape
    if ep:
        if n_exp % tp:
            raise ValueError(f"ep over tp={tp} ranks needs the {n_exp} experts to split evenly")
        e_r, e0, f_r, f0 = n_exp // tp, rank * (n_exp // tp), ffn, 0
    else:
        e_r, e0, f_r, f0 = n_exp, 0, ffn // tp, rank * (ffn // tp)
    ex = base + "experts."
    w13 = (PackedPart(ex + "w1", (slice(0, e_r), slice(0, f_r), slice(0, h)), (e0, 0, f0), transpose=True),
           PackedPart(ex + "w3", (slice(0, e_r), slice(f_r, 2 * f_r), slice(0, h)), (e0, 0, f0), transpose=True))
    w2 = (PackedPart(ex + "w2", (slice(0, e_r), slice(0, h), slice(0, f_r)), (e0, f0, 0), transpose=True),)
    return {ex + "w13_weight": ((e_r, 2 * f_r, h), w13, None), ex + "w2_weight": ((e_r, h, f_r), w2, None)}


def _from_torchtitan(titan_layout, cfg, tp: int, rank: int, ep: bool):
    """:func:`vllm_tp_layout` with ``source="torchtitan"``: the HF layout's parts renamed back to the torchtitan
    tensors, the q and k parts rotary, and every unpacked parameter one part of its renamed tensor."""
    import dataclasses

    from torchstore_b200.direct_weight_sync import PackedPart

    back = {hf_name(n): n for n in titan_layout}
    hf = {hf_name(n): e for n, e in titan_layout.items()}
    out = {}
    for name, (shape, parts, box) in vllm_tp_layout(hf, cfg, tp, rank, ep).items():
        if parts is None:
            parts = (PackedPart(back[name], tuple(slice(0, e) for e in shape), tuple(box[0])),)
        else:
            hd = hf[parts[0].source][0][0] // cfg["n_heads"] if name.endswith("qkv_proj.weight") else None
            parts = tuple(dataclasses.replace(p, source=back[p.source],
                                              rotary_head_dim=hd if p.source.endswith(("q_proj.weight", "k_proj.weight"))
                                              else None) for p in parts)
        out[name] = (tuple(shape), parts, None)
    return out
