"""The MMA warpgroup of the tensor-core build kernel places its fragments by a compile-time column mapping (csrc/mma_role.cuh) but
forms every element from the same 8-pixel products, added in the same order: lm_build's outputs are bitwise equal to the frozen
digests in tests/golden/build_mma.json (written by tests/golden/gen_build_mma.py with the previous, runtime-indexed MMA role), in
every precision mode, both conv2 layouts and K = 128 / 64 / 32."""
import json
import os
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))


def test_generation_6_outputs_bitwise_equal_to_golden():
    import gen_build_mma
    with open(os.path.join(HERE, "golden", "build_mma.json")) as f:
        want = json.load(f)
    p = torch.cuda.get_device_properties(0)
    if p.multi_processor_count != want["sm_count"]:
        pytest.skip(f"digests were taken with {want['sm_count']} SMs ({want['device']}); this device has {p.multi_processor_count}: "
                    "another tile partition sums the span partials in another order")
    got = gen_build_mma.outputs()
    assert set(got["cases"]) == set(want["cases"])
    bad = {c: [k for k in want["cases"][c] if got["cases"][c][k] != want["cases"][c][k]] for c in want["cases"]}
    bad = {c: ks for c, ks in bad.items() if ks}
    assert not bad, f"outputs differ from the golden digests: {bad}"
