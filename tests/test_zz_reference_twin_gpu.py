"""The CUDA path against vectors produced by the reference's own code (tests/golden/reference_twin.json: the reference's
Python twin executed, see tests/golden/make_reference_twin_golden.py): the call rows it produced go through the C ABI
(encode -> wgmma Gram -> centering) and every similarity count and every centred double must come out identical.
(File name: sorted last on purpose, so that this late addition can never mask another GPU test under `-x`.)"""
import json
from pathlib import Path

import numpy as np
import pytest

from spark_examples_b200 import native

pytestmark = pytest.mark.gpu

GOLD = json.loads((Path(__file__).resolve().parent / "golden" / "reference_twin.json").read_text())


@pytest.mark.parametrize("case", GOLD["cases"], ids=[c["name"] for c in GOLD["cases"]])
def test_gram_and_centering_equal_the_reference_twin(case):
    n, rows = case["n"], case["call_rows"]
    S_want = np.zeros((n, n), np.int32)
    for y, x, v in case["similarity_records"]:
        S_want[y, x] = v
    C_want = np.zeros((n, n))
    for row, cols in enumerate(case["centered_rows"]):
        for col, hexval in cols:
            C_want[row, col] = float.fromhex(hexval)
    off = np.zeros(len(rows) + 1, np.int64)
    off[1:] = np.cumsum([len(r) for r in rows])
    idx = np.asarray([i for r in rows for i in r], np.int32)
    half = len(rows) // 2                                      # two partitions, like two tasks of mapPartitions (:184-189)
    with native.NativePca(n, max_multiplicity=2) as nat:
        nat.accumulateCalls(0, off[: half + 1], idx[: off[half]])
        nat.accumulateCalls(1, off[half:] - off[half], idx[off[half]:])
        nat.commit(0)
        nat.commit(1)
        nat.finalizeGram()
        S = nat.getGram()
        C = nat.getCentered()
    assert np.array_equal(S, S_want)                           # calculate_similarity_matrix (variants_pca.py:54-82)
    assert np.array_equal(C, C_want)                           # center_matrix (:84-121), bit for bit
