"""TEST INFRASTRUCTURE ONLY -- records tests/golden/int8_vectors.npz.

The inputs are int8_oracle.fixture_inputs(), rebuilt bit for bit from an integer hash wherever the tests run, so
the fixture does not carry them: per case it keeps the dtype and granularity, the sha256 of the input bits (to
catch a drifted generator), torch CPU's scale_inv in full and the sha256 of torch CPU's int8 bytes
(int8_oracle.torch_quantize: ``torch.round(xf * scale).nan_to_num(nan=0.0).clamp(-128, 127).to(torch.int8)``).

    python oracle/gen_golden_int8.py
"""

from __future__ import annotations

import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle.int8_oracle import bits_of, digest, fixture_inputs, torch_quantize  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "int8_vectors.npz")


def main():
    arrays = {}
    names = []
    for i, (name, x, g) in enumerate(fixture_inputs()):
        names.append(name)
        arrays[f"dtype{i}"] = np.array(str(x.dtype).replace("torch.", ""))
        arrays[f"granularity{i}"] = np.array(g)
        arrays[f"x_sha{i}"] = np.array(digest(bits_of(x)))
        q, s = torch_quantize(x, g)
        arrays[f"s{i}"] = s.numpy()
        arrays[f"q_sha{i}"] = np.array(digest(q.view(torch.uint8).numpy()))
    arrays["names"] = np.array(names)
    np.savez_compressed(OUT, **arrays)
    print(f"wrote {len(names)} cases to {OUT}")


if __name__ == "__main__":
    main()
