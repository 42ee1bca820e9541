"""The numpy replicas of tests/_encode_ref.py against the engine's own headers, on the host.

tests/test_encode_gpu.py builds its adversarial keys (probe chains, full shared-memory buckets,
the reserved fold hash) from these replicas.  A wrong replica would not fail anything there: the
cases would silently stop reaching their branches.  So a host-only program that includes
csrc/common.cuh and csrc/lookup.cuh evaluates every function on 2^17 inputs (edges + random), and
the replicas must agree bit for bit.  It is compiled with nvcc and runs without a GPU; the test is
skipped where nvcc is absent.  The value hash of the reference (oracle/hashing.py) is pinned to
pandas.util.hash_array on every dtype the encode tests hash."""
import os
import re
import shutil
import subprocess

import numpy as np
import pandas as pd
import pytest

import _encode_ref as R
from oracle.hashing import hash_values

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "nvtabular_b200", "csrc")

PROGRAM = r"""
#include <cstdio>
#include <vector>
#include "common.cuh"
#include "lookup.cuh"
using namespace nvtb;
int main(int argc, char** argv) {
  FILE* f = fopen(argv[1], "rb");
  std::vector<uint64_t> x;
  uint64_t v;
  while (fread(&v, 8, 1, f) == 1) x.push_back(v);
  fclose(f);
  FILE* o = fopen(argv[2], "wb");
  for (uint64_t k : x) {
    const uint32_t lo = (uint32_t)k;
    const uint64_t r[6] = {table_mix32(lo), fold_hash(lo), fold_unhash(lo), table_mix64(k), pandas_mix64(k),
                           ((uint64_t)fold_hash(lo) * 7168u) >> 32};
    fwrite(r, 8, 6, o);
  }
  for (int e = 0; e <= 40; ++e) {
    const int64_t nb = (int64_t)1 << e;
    const int64_t r[4] = {narrow_slice_buckets(nb), narrow_next(0, nb), narrow_next(nb - 1, nb),
                          narrow_next((int64_t)(x[e] & (uint64_t)(nb - 1)), nb)};
    fwrite(r, 8, 4, o);
  }
  fclose(o);
  return 0;
}
"""


def _nvcc():
    exe = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    return exe if os.path.exists(exe) else None


def _inputs():
    rng = np.random.default_rng(5)
    edges = np.array([0, 1, 2, 0x7FFFFFFF, 0x80000000, 0xFFFFFFFF, 0x100000000, 0xFFFFFFFFFFFFFFFF,
                      0x8000000000000000, 0x7FFFFFFFFFFFFFFF, 0x7FF8000000000000, R.FOLD_EMPTY - 1,
                      int(R.fold_unhash(np.uint32(R.FOLD_EMPTY)))], dtype=np.uint64)
    return np.concatenate([edges, rng.integers(0, 1 << 63, (1 << 17) - len(edges), dtype=np.uint64) * np.uint64(2)
                           + rng.integers(0, 2, (1 << 17) - len(edges), dtype=np.uint64)])


def test_replicas_match_header(tmp_path):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    src, exe = tmp_path / "replicas.cu", tmp_path / "replicas"
    src.write_text(PROGRAM)
    subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "--expt-relaxed-constexpr",
                    "-I", CSRC, str(src), "-o", str(exe)], check=True, capture_output=True, timeout=300)
    x = _inputs()
    (tmp_path / "in.bin").write_bytes(x.tobytes())
    subprocess.run([str(exe), str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], check=True, timeout=60)
    raw = np.frombuffer((tmp_path / "out.bin").read_bytes(), dtype=np.uint64)
    per_key = raw[: 6 * len(x)].reshape(-1, 6)
    lo = (x & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    np.testing.assert_array_equal(per_key[:, 0], R.table_mix32(lo))
    np.testing.assert_array_equal(per_key[:, 1], R.fold_hash(lo))
    np.testing.assert_array_equal(per_key[:, 2], R.fold_unhash(lo))
    np.testing.assert_array_equal(per_key[:, 3], R.table_mix64(x))
    np.testing.assert_array_equal(per_key[:, 4], R._mix(x))
    np.testing.assert_array_equal(per_key[:, 5].astype(np.int64), R.smem_bucket(lo.view(np.int32)))
    geo = raw[6 * len(x):].view(np.int64).reshape(-1, 4)
    for e in range(41):
        nb = 1 << e
        assert geo[e, 0] == R.narrow_slice_buckets(nb), e
        assert geo[e, 1] == R.narrow_next(0, nb), e
        assert geo[e, 2] == R.narrow_next(nb - 1, nb), e
        assert geo[e, 3] == R.narrow_next(int(x[e]) & (nb - 1), nb), e


def test_replica_inverses_and_bucket_rules():
    x = _inputs()
    lo = (x & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    np.testing.assert_array_equal(R.table_unmix32(R.table_mix32(lo)), lo)
    np.testing.assert_array_equal(R.table_mix32(R.table_unmix32(lo)), lo)
    np.testing.assert_array_equal(R.fold_unhash(R.fold_hash(lo)), lo)
    np.testing.assert_array_equal(R.table_unmix64(R.table_mix64(x)), x)
    np.testing.assert_array_equal(R.table_mix64(R.table_unmix64(x)), x)
    assert R.fold_hash(R.fold_unhash(np.uint32(R.FOLD_EMPTY))) == R.FOLD_EMPTY
    rng = np.random.default_rng(1)
    # a chain shares its home bucket in every table of at most 2^L buckets, and all-ones low bits
    # put it in the last bucket (the end of the last slice)
    ch = R.narrow_chain(rng, 20, (1 << 20) - 1, 12)
    for lg in (4, 13, 14, 20):
        assert (R.narrow_home(ch, 1 << lg) == (1 << lg) - 1).all()
    ch = R.narrow_chain(rng, 14, (1 << 13) - 1, 12)            # bucket 8191: the end of slice 0
    assert (R.narrow_home(ch, 1 << 14) == 8191).all() and R.narrow_next(8191, 1 << 14) == 0
    wc = R.wide_chain(rng, 24, (1 << 24) - 1, 9)
    for lg in (5, 17, 24):
        assert (R.wide_home(wc, 1 << lg) == (1 << lg) - 1).all()
    assert (R.smem_bucket(R.smem_bucket_keys(4321, 8)) == 4321).all()


def test_vocab_constants_are_the_replicas():
    """the shared-memory encode's table size lives in vocab.cu, not in a header"""
    src = open(os.path.join(CSRC, "vocab.cu")).read()
    assert re.search(r"kEncSmemBuckets\s*=\s*%d;" % R.SMEM_BUCKETS, src)
    assert re.search(r"kEncSmemMaxKeys\s*=\s*\(int64_t\)kEncSmemBuckets\s*\*\s*2;", src)
    hdr = open(os.path.join(CSRC, "lookup.cuh")).read()
    assert re.search(r"kSliceBuckets\s*=\s*%d;" % R.SLICE_BUCKETS, hdr)
    assert re.search(r"kSliceParts\s*=\s*%d;" % R.SLICE_PARTS, hdr)


@pytest.mark.parametrize("dtype", ["int32", "int64", "float32", "float64", "uint8", "bool"])
def test_oracle_hash_is_pandas(dtype):
    rng = np.random.default_rng(3)
    if dtype == "bool":
        a = rng.random(4096) < 0.5
    elif dtype in ("float32", "float64"):
        a = (rng.normal(0, 1e6, 4096)).astype(dtype)
        a[:6] = [0.0, -0.0, np.inf, -np.inf, 1.5, -1.5]
    else:
        info = np.iinfo(dtype)
        a = rng.integers(info.min, info.max, 4096, endpoint=True).astype(dtype)
        a[:3] = [info.min, info.max, 0]
    np.testing.assert_array_equal(hash_values(a), pd.util.hash_array(a))
    if dtype == "float64":                       # a null is what pandas sees: the float64 NaN
        np.testing.assert_array_equal(hash_values(np.array([np.nan])), pd.util.hash_array(np.array([np.nan])))
