"""The launch constants tests/test_gpu_zip.py sizes its grid-round cases from are the ones csrc/zip.cu and
csrc/bytes_engine.cuh launch with."""
import os
import re

import test_gpu_zip as t

CSRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "arrow-rs_b200", "csrc")


def test_launch_constants_match_the_source():
    src = open(os.path.join(CSRC, "zip.cu")).read()
    assert re.search(r"#define ZIP_THREADS (\d+)", src).group(1) == str(t.ZIP_THREADS)
    assert re.search(r"#define ZIP_PER_SM (\d+)", src).group(1) == str(t.ZIP_PER_SM)
    assert re.search(r"#define ZIP_FSB_CHUNKS (\d+)", src).group(1) == str(t.ZIP_FSB_CHUNKS)
    # k_zip_bits: one thread per 64-row word; k_zip_views: one per row; k_zip_fsb: ZIP_FSB_CHUNKS 16-byte chunks per thread
    assert "acu_grid(ctx, (words + ZIP_THREADS - 1) / ZIP_THREADS, ZIP_PER_SM)" in src
    assert "acu_grid(ctx, (z.len + ZIP_THREADS - 1) / ZIP_THREADS, ZIP_PER_SM)" in src
    assert "const int64_t per_block = (int64_t)ZIP_THREADS * ZIP_FSB_CHUNKS;" in src
    assert "acu_grid(ctx, (n_chunks + per_block - 1) / per_block, ZIP_PER_SM)" in src
    eng = open(os.path.join(CSRC, "bytes_engine.cuh")).read()
    threads = int(re.search(r"#define BY_THREADS (\d+)", eng).group(1))
    assert "#define BY_ROWS (BY_THREADS * 4)" in eng and t.BY_ROWS == threads * 4
