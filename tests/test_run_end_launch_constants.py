"""The launch constants tests/test_gpu_run_end.py sizes its grid-round cases from are the ones csrc/run_end.cu launches with."""
import os
import re

import test_gpu_run_end as t

SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "arrow-rs_b200", "csrc", "run_end.cu")


def test_launch_constants_match_the_source():
    src = open(SRC).read()
    assert re.search(r"#define RE_THREADS (\d+)", src).group(1) == str(t.RE_THREADS)
    assert re.search(r"#define RE_PER_SM (\d+)", src).group(1) == str(t.RE_PER_SM)
    assert "acu_grid(ctx, (threads + RE_THREADS - 1) / RE_THREADS, RE_PER_SM)" in src
    # every grid-stride kernel launches through re_grid with RE_THREADS-thread blocks
    for k in ("k_ree_filter_runs<R>", "k_ree_take_map<R, uint64_t>", "k_ree_take_map<R, uint32_t>", "k_ree_run_ends<decltype(src), uint64_t>",
              "k_ree_run_ends<decltype(src), uint32_t>"):
        assert re.search(re.escape(k) + r"\)?, (re_grid\(ctx, [^;]*\)|bgrid|grid), RE_THREADS", src), k
    assert "const int grid = re_grid(ctx, m);" in src and "const int bgrid = re_grid(ctx, (m + 1 + 31) / 32 * 32);" in src
