"""The launch constants tests/test_gpu_union.py sizes its partition boundary cases from are the ones csrc/union.cu launches
with."""
import os
import re

import test_gpu_union as t

SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "arrow-rs_b200", "csrc", "union.cu")


def test_launch_constants_match_the_source():
    src = open(SRC).read()
    assert re.search(r"#define UN_THREADS (\d+)", src).group(1) == str(t.UN_THREADS)
    assert re.search(r"#define UN_TILE_ROWS (\d+)", src).group(1) == str(t.UN_TILE_ROWS)
    assert re.search(r"#define UN_PER_SM (\d+)", src).group(1) == str(t.UN_PER_SM)
    # both tile kernels walk tiles of UN_TILE_ROWS rows grid-stride on acu_grid(ctx, tiles, UN_PER_SM) blocks of UN_THREADS
    assert "const int64_t n_tiles = (m + UN_TILE_ROWS - 1) / UN_TILE_ROWS;" in src
    assert "const int grid = acu_grid(ctx, n_tiles, UN_PER_SM);" in src
    for k in ("k_union_count", "k_union_scatter"):
        assert re.search(k + r", grid, UN_THREADS, 0,", src), k
    assert src.count("for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x)") == 2
    assert src.count("r0 += UN_THREADS") == 2
