"""TEST INFRASTRUCTURE ONLY -- records tests/golden/int8_source_vectors.npz.

The inputs are rebuilt bit for bit from an integer hash wherever the tests run, so the fixture does not carry them:
* quantising cases (int8_source_oracle.quant_inputs, the shard-local cases of source-side quantisation): per case
  the dtype, granularity and shard offset, the sha256 of the input bits, torch CPU's scale_inv in full and the
  sha256 of torch CPU's int8 bytes (int8_source_oracle.torch_quantize);
* dequantising cases (int8_source_oracle.dequant_inputs): per case the sha256 of the int8 bytes and of the scales,
  and per destination dtype the sha256 of torch CPU's ``(q.float() * s_expanded).to(dst)`` bits.

    python oracle/gen_golden_int8_source.py
"""

from __future__ import annotations

import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle.int8_source_oracle import (DSTS, bits_of, dequant_inputs, digest, quant_inputs,  # noqa: E402
                                       torch_dequantize, torch_quantize)

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden",
                   "int8_source_vectors.npz")


def main():
    arrays = {}
    names = []
    for i, (name, x, g, r0, c0) in enumerate(quant_inputs()):
        names.append(name)
        arrays[f"dtype{i}"] = np.array(str(x.dtype).replace("torch.", ""))
        arrays[f"granularity{i}"] = np.array(g)
        arrays[f"offset{i}"] = np.array([r0, c0])
        arrays[f"x_sha{i}"] = np.array(digest(bits_of(x)))
        q, s = torch_quantize(x, g, r0, c0)
        arrays[f"s{i}"] = s.numpy()
        arrays[f"q_sha{i}"] = np.array(digest(q.view(torch.uint8).numpy()))
    dq_names = []
    for i, (name, g, r0, c0, q, s) in enumerate(dequant_inputs()):
        dq_names.append(name)
        arrays[f"dq_q_sha{i}"] = np.array(digest(q.view(torch.uint8).numpy()))
        arrays[f"dq_s_sha{i}"] = np.array(digest(s.numpy().view(np.uint32)))
        for dst in DSTS:
            y = torch_dequantize(q, s, g, r0, c0, getattr(torch, dst))
            arrays[f"dq_{dst}_sha{i}"] = np.array(digest(bits_of(y)))
    arrays["names"] = np.array(names)
    arrays["dq_names"] = np.array(dq_names)
    np.savez_compressed(OUT, **arrays)
    print(f"wrote {len(names)} quantising and {len(dq_names)} dequantising cases to {OUT}")


if __name__ == "__main__":
    main()
