"""TEST INFRASTRUCTURE ONLY -- records tests/golden/requant_fp8_vectors.npz.

The inputs are requant_fp8_oracle.fixture_inputs(), rebuilt bit for bit from an integer hash wherever the
tests run, so the fixture does not carry them: per case it keeps both granularities, the window offset, the
sha256 of the fp8 bytes and of the scale bits (to catch a drifted generator), and torch CPU's output
(requant_fp8_oracle.torch_requantize): the sha256 of the fp8 bytes with every NaN byte written as 0x7F (a NaN's
sign is platform-specific) and scale_inv in full, which the tests compare NaN-agnostically.

    python oracle/gen_golden_requant_fp8.py
"""

from __future__ import annotations

import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle.requant_fp8_oracle import canonical_nan, digest, fixture_inputs, torch_requantize  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "requant_fp8_vectors.npz")


def main():
    arrays = {}
    names = []
    for i, (name, sg, dg, r0, c0, q, s) in enumerate(fixture_inputs()):
        names.append(name)
        arrays[f"g{i}"] = np.array([sg, dg])
        arrays[f"off{i}"] = np.array([r0, c0])
        arrays[f"q_sha{i}"] = np.array(digest(q.view(torch.uint8).numpy()))
        arrays[f"s_sha{i}"] = np.array(digest(s.numpy().view(np.uint32)))
        y, y_scale = torch_requantize(q, s, sg, r0, c0, dg)
        arrays[f"y_sha{i}"] = np.array(digest(canonical_nan(y.view(torch.uint8).numpy())))
        arrays[f"y_scale{i}"] = y_scale.numpy()
    arrays["names"] = np.array(names)
    np.savez_compressed(OUT, **arrays)
    print(f"wrote {len(names)} cases to {OUT}")


if __name__ == "__main__":
    main()
