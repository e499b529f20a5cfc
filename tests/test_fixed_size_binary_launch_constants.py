"""The launch constants tests/test_gpu_fixed_size_binary.py sizes its grid-round cases from are the ones
csrc/fixed_size_binary.cu launches with."""
import os
import re

import test_gpu_fixed_size_binary as t

SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "arrow-rs_b200", "csrc", "fixed_size_binary.cu")


def test_launch_constants_match_the_source():
    src = open(SRC).read()
    assert re.search(r"#define FSB_THREADS (\d+)", src).group(1) == str(t.FSB_THREADS)
    assert re.search(r"#define FSB_PER_SM (\d+)", src).group(1) == str(t.FSB_PER_SM)
    # rows per chunk and chunks per thread by width, as the test restates them
    assert "int max_rows(int64_t w) { return w >= 16 ? 2 : w >= 8 ? 3 : w >= 4 ? 5 : w >= 2 ? 9 : 17; }" in src
    assert "static constexpr int CHUNKS = MAXR <= 3 ? 4 : MAXR <= 5 ? 2 : 1;" in src
    # grid-stride over blocks of FSB_THREADS x CHUNKS chunks on acu_grid(ctx, blocks, FSB_PER_SM)
    assert "const int64_t per_block = (int64_t)FSB_THREADS * FsbCfg<MAXR>::CHUNKS;" in src
    assert "const int grid = acu_grid(ctx, (n_chunks + per_block - 1) / per_block, FSB_PER_SM);" in src
    assert "r0 += (int64_t)gridDim.x * FSB_THREADS * K" in src
