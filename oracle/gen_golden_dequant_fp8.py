"""TEST INFRASTRUCTURE ONLY -- records tests/golden/dequant_fp8_vectors.npz.

The inputs are dequant_fp8_oracle.fixture_inputs(), rebuilt bit for bit from an integer hash wherever the
tests run, so the fixture does not carry them: per case it keeps the granularity, the shard offset, the
sha256 of the fp8 bytes and of the scale bits (to catch a drifted generator), and per destination dtype
the sha256 of torch CPU's output bits (dequant_fp8_oracle.torch_dequantize).  The all-bytes table, whose
scale set holds Inf and NaN, keeps its outputs in full: NaN bits are platform-specific, so the tests
compare them NaN-agnostically.

    python oracle/gen_golden_dequant_fp8.py
"""

from __future__ import annotations

import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle.dequant_fp8_oracle import DST, digest, fixture_inputs, torch_dequantize  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "dequant_fp8_vectors.npz")


def bits(y: torch.Tensor) -> np.ndarray:
    return y.view(torch.int16 if y.element_size() == 2 else torch.int32).numpy().view(
        np.uint16 if y.element_size() == 2 else np.uint32)


def main():
    arrays = {}
    names = []
    for i, (name, g, r0, c0, q, s) in enumerate(fixture_inputs()):
        names.append(name)
        arrays[f"g{i}"] = np.array(g)
        arrays[f"off{i}"] = np.array([r0, c0])
        arrays[f"q_sha{i}"] = np.array(digest(q.view(torch.uint8).numpy()))
        arrays[f"s_sha{i}"] = np.array(digest(s.numpy().view(np.uint32)))
        for dst, dtype in DST.items():
            y = bits(torch_dequantize(q, s, g, r0, c0, dtype))
            if name == "all_bytes":
                arrays[f"y_{dst}{i}"] = y
            else:
                arrays[f"y_sha_{dst}{i}"] = np.array(digest(y))
    arrays["names"] = np.array(names)
    np.savez_compressed(OUT, **arrays)
    print(f"wrote {len(names)} cases to {OUT}")


if __name__ == "__main__":
    main()
