"""CPU: the numpy hash restatements in tests/keys.py agree bit for bit with csrc/dj_device.cuh.

The adversarial join cases (test_kernel_edges.py) are only skewed or colliding while these
restatements match the hashes the kernels use; this pins them to the header itself, compiled for
the host by nvcc, so a change to either hash fails here rather than quietly turning those cases
into random ones."""
import os
import shutil
import subprocess

import numpy as np
import pytest

import keys as K

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "distributed-join_b200", "csrc")

_PROG = r"""
#include <cstdio>
#include <vector>
#include "dj_device.cuh"
// stdin: int64 keys; stdout: (local_hash_i64, slot_hash_i64) per key as uint32 pairs
int main()
{
  std::vector<int64_t> k;
  int64_t v;
  while (fread(&v, 8, 1, stdin) == 1) k.push_back(v);
  for (int64_t x : k) {
    uint32_t h[2] = {dj::local_hash_i64(x), dj::slot_hash_i64(x)};
    fwrite(h, 4, 2, stdout);
  }
  return 0;
}
"""


def _nvcc():
    for p in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if p and os.path.exists(p):
            return p
    return None


@pytest.fixture(scope="module")
def device_hashes(tmp_path_factory):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    d = tmp_path_factory.mktemp("hashpin")
    src, exe = d / "hashes.cu", d / "hashes"
    src.write_text(_PROG)
    subprocess.run([nvcc, "-std=c++17", "-O1", "-I", CSRC, "-o", str(exe), str(src)], check=True,
                   capture_output=True, text=True)

    def run(keys):
        keys = np.ascontiguousarray(keys, dtype=np.int64)
        out = subprocess.run([str(exe)], input=keys.tobytes(), capture_output=True, check=True).stdout
        h = np.frombuffer(out, dtype=np.uint32).reshape(-1, 2)
        assert h.shape[0] == keys.size
        return h[:, 0], h[:, 1]

    return run


def test_hash_restatements_match_header(device_hashes):
    rng = np.random.default_rng(2024)
    i64 = np.iinfo(np.int64)
    keys = np.concatenate([
        rng.integers(i64.min, i64.max, 60_000, dtype=np.int64, endpoint=True),
        rng.integers(-1000, 1000, 20_000, dtype=np.int64),
        np.array([0, 1, -1, i64.min, i64.max, 1 << 32, -(1 << 32), 0xFFFFFFFF], dtype=np.int64),
        np.int64(1) << rng.integers(0, 63, 20_000).astype(np.int64),
    ])
    lh, sh = device_hashes(keys)
    assert (K.local_hash(keys) == lh).all()
    assert (K.slot_hash(keys) == sh).all()


def test_mix64_is_a_full_width_bijection():
    """unmix64 inverts mix64 on edge and random words, matches the splitmix64 finalizer written with
    Python integers, and mix64 of consecutive ids sets bit 31 and bit 63 both ways (the payloads of
    the GPU cases carry full-width 32-bit halves)."""
    rng = np.random.default_rng(64)
    i64 = np.iinfo(np.int64)
    edges = np.array([0, 1, -1, 2, -2, i64.min, i64.max, i64.min + 1, i64.max - 1, 0x7FFFFFFF, 0x80000000,
                      0xFFFFFFFF, 1 << 32, 0x7FFFFFFF80000000, -0x7FFFFFFF80000000, -(1 << 32)], dtype=np.int64)
    words = np.concatenate([edges, rng.integers(i64.min, i64.max, 100_000, dtype=np.int64, endpoint=True)])
    assert (K.unmix64(K.mix64(words)) == words).all()
    assert (K.mix64(K.unmix64(words)) == words).all()
    assert np.unique(K.mix64(words)).size == np.unique(words).size

    def mix_int(x):
        m = (1 << 64) - 1
        x &= m
        x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & m
        x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & m
        return x ^ (x >> 31)

    got = K.mix64(words[:2000]).view(np.uint64)
    assert [int(g) for g in got] == [mix_int(int(w)) for w in words[:2000]]
    for base in (0, 1 << 20, 1 << 40, 1 << 48, (1 << 48) + (3 << 36)):
        m = K.mix64(np.arange(base, base + 4096, dtype=np.int64)).view(np.uint64)
        for bit in (31, 63):
            b = (m >> np.uint64(bit)) & np.uint64(1)
            assert 0 < int(b.sum()) < m.size, (base, bit)


@pytest.mark.parametrize("bits", [1, 4, 10, 13])
def test_constructed_keys_hit_their_bucket_and_slot(device_hashes, bits):
    """keys_in_bucket and slot_twins, checked with the header's hashes rather than the restatements."""
    rng = np.random.default_rng(bits)
    bucket = int(rng.integers(0, 1 << bits))
    ks = K.keys_in_bucket(bits, bucket, 3000, rng)
    tw = K.slot_twins(ks[:300], bits, rng)
    assert np.unique(ks).size == ks.size
    lh, _ = device_hashes(ks)
    assert ((lh >> np.uint32(32 - bits)) == bucket).all()
    lt, st = device_hashes(tw)
    _, sk = device_hashes(ks[:300])
    assert ((lt >> np.uint32(32 - bits)) == bucket).all()
    assert (st == sk).all() and (tw != ks[:300]).all()
