"""TEST INFRASTRUCTURE ONLY -- records tests/golden/ue8m0_vectors.npz.

The inputs are ue8m0_oracle.fixture_inputs(), rebuilt bit for bit from an integer hash wherever the tests run,
so the fixture does not carry them: per case it keeps the dtype, granularity and shard offset, the sha256 of the
input bits (to catch a drifted generator), torch CPU's UE8M0 scale_inv in full and the sha256 of torch CPU's fp8
bytes (ue8m0_oracle.torch_quantize with scale_fmt="ue8m0", tensor/tensor ops and integer views, no log2).  A
case with a non-finite scale keeps its fp8 bytes in full instead: NaN bytes are platform-specific there, so the
tests compare them NaN-agnostically.

    python oracle/gen_golden_ue8m0.py
"""

from __future__ import annotations

import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle.ue8m0_oracle import bits_of, digest, fixture_inputs, torch_quantize  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "ue8m0_vectors.npz")


def main():
    arrays = {}
    names = []
    for i, (name, x, g, r0, c0) in enumerate(fixture_inputs()):
        names.append(name)
        arrays[f"dtype{i}"] = np.array(str(x.dtype).replace("torch.", ""))
        arrays[f"where{i}"] = np.array([g, str(r0), str(c0)])
        arrays[f"x_sha{i}"] = np.array(digest(bits_of(x)))
        q, s = torch_quantize(x, g, r0, c0, scale_fmt="ue8m0")
        q, s = q.view(torch.uint8).numpy(), s.numpy()
        arrays[f"s{i}"] = s
        if np.isfinite(s).all():
            arrays[f"q_sha{i}"] = np.array(digest(q))
        else:
            arrays[f"q{i}"] = q
    arrays["names"] = np.array(names)
    np.savez_compressed(OUT, **arrays)
    print(f"wrote {len(names)} cases to {OUT}")


if __name__ == "__main__":
    main()
