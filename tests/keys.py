"""Adversarial int64 join keys, built by inverting the join's own hashes (csrc/dj_device.cuh).

numpy restatements (uint64, wrapping) of the two hashes the join kernels branch on:
  local_hash_i64  its top bits pick the radix bucket (partition.cu, mode 1);
  slot_hash_i64   slot and 20-bit fingerprint inside a bucket's shared-memory table (join.cu).
test_keys.py pins both, bit for bit, to the CUDA header compiled on the host.

keys_in_bucket  distinct keys whose local hash has the given top bits (one radix bucket);
slot_twins      for each key, a different key with the same 32-bit slot hash in the same bucket,
                so a probe reaches the build row's slot with a matching fingerprint and only the
                full key comparison tells them apart.
mix64, unmix64  the splitmix64 finalizer and its inverse: test payloads are mix64(base + row), so
                every 32-bit half of a payload word takes full-width values (bit 31 and bit 63
                set about half the time) while the row stays recoverable with unmix64.
"""
import numpy as np

_C1 = 0x9E3779B97F4A7C15
_C2 = 0xD6E8FEB86659FD93
_C1_INV = pow(_C1, -1, 1 << 64)
_C2_INV = pow(_C2, -1, 1 << 64)
_M1 = 0xBF58476D1CE4E5B9  # splitmix64 finalizer multipliers
_M2 = 0x94D049BB133111EB
_M1_INV = pow(_M1, -1, 1 << 64)
_M2_INV = pow(_M2, -1, 1 << 64)


def _u64(keys):
    return np.ascontiguousarray(keys, dtype=np.int64).view(np.uint64)


def mix64(x) -> np.ndarray:
    """splitmix64 finalizer on int64 words (uint64 wrap): a bijection of the 64-bit words."""
    z = _u64(x).copy()
    with np.errstate(over="ignore"):
        z ^= z >> np.uint64(30)
        z *= np.uint64(_M1)
        z ^= z >> np.uint64(27)
        z *= np.uint64(_M2)
        z ^= z >> np.uint64(31)
    return z.view(np.int64)


def unmix64(y) -> np.ndarray:
    """Inverse of mix64: each xor-shift by s >= 22 is undone by xoring in the shifts by s and 2s,
    each multiply by the modular inverse."""
    z = _u64(y).copy()
    with np.errstate(over="ignore"):
        z ^= (z >> np.uint64(31)) ^ (z >> np.uint64(62))
        z *= np.uint64(_M2_INV)
        z ^= (z >> np.uint64(27)) ^ (z >> np.uint64(54))
        z *= np.uint64(_M1_INV)
        z ^= (z >> np.uint64(30)) ^ (z >> np.uint64(60))
    return z.view(np.int64)


def local_hash(keys) -> np.ndarray:
    """local_hash_i64: top 32 bits of ((k * C1) ^ >>29) * C2."""
    with np.errstate(over="ignore"):
        x = _u64(keys) * np.uint64(_C1)
        x ^= x >> np.uint64(29)
        x *= np.uint64(_C2)
    return (x >> np.uint64(32)).astype(np.uint32)


def _g(hi):
    with np.errstate(over="ignore"):
        return hi * np.uint32(0x85EBCA6B) + np.uint32(0x632BE5AB)


def slot_hash(keys) -> np.ndarray:
    """slot_hash_i64: lo ^ g(hi), then a 32-bit bijection."""
    k = _u64(keys)
    lo = (k & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    hi = (k >> np.uint64(32)).astype(np.uint32)
    with np.errstate(over="ignore"):
        x = lo ^ _g(hi)
        x *= np.uint32(0x9E3779B1)
        x ^= x >> np.uint32(15)
        x *= np.uint32(0x2C1B3C6D)
    return x


def bucket_of(keys, bits: int) -> np.ndarray:
    """Radix bucket of a `bits`-bit plan: the top bits of the local hash (level 1 then level 2)."""
    return (local_hash(keys) >> np.uint32(32 - bits)).astype(np.int64) if bits else np.zeros(len(keys), np.int64)


def keys_in_bucket(bits: int, bucket: int, n: int, rng) -> np.ndarray:
    """`n` distinct keys in radix bucket `bucket` of a `bits`-bit plan, by inverting local_hash: the
    final 64-bit product is chosen with the bucket in its top bits, then the multiply by C2, the
    xor-shift by 29 and the multiply by C1 are undone (all three are bijections on 64-bit words)."""
    assert 0 <= bucket < (1 << bits) and bits <= 32
    low = 64 - bits
    ys = np.empty(0, np.uint64)
    while ys.size < n:
        r = rng.integers(0, 1 << 64, n - ys.size, dtype=np.uint64)
        if low < 64:
            r &= np.uint64((1 << low) - 1)
            r |= np.uint64(bucket << low)
        ys = np.unique(np.concatenate([ys, r]))
    ys = rng.permutation(ys)[:n]
    with np.errstate(over="ignore"):
        x = ys * np.uint64(_C2_INV)
        x = x ^ (x >> np.uint64(29)) ^ (x >> np.uint64(58))
        x *= np.uint64(_C1_INV)
    keys = x.view(np.int64)
    assert (bucket_of(keys, bits) == bucket).all()
    return keys


def slot_twins(keys, bits: int, rng) -> np.ndarray:
    """For every key a different key with the same slot_hash and the same `bits`-bit radix bucket.
    slot_hash only sees lo ^ g(hi): with a new hi' and lo' = lo ^ g(hi) ^ g(hi') the mixed word is
    unchanged.  hi' is redrawn until the twin's local hash keeps the top `bits` (2^bits tries per
    twin on average, drawn for all pending keys at once)."""
    k = _u64(keys)
    lo = (k & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    hi = (k >> np.uint64(32)).astype(np.uint32)
    want = bucket_of(keys, bits)
    out = np.zeros(k.size, np.uint64)
    pending = np.arange(k.size)
    per = max(1, min(1 << bits, (1 << 22) // max(k.size, 1)))  # candidates per pending key and round
    while pending.size:
        idx = np.repeat(pending, per)
        hi2 = rng.integers(0, 1 << 32, idx.size, dtype=np.uint64).astype(np.uint32)
        lo2 = lo[idx] ^ _g(hi[idx]) ^ _g(hi2)
        cand = (hi2.astype(np.uint64) << np.uint64(32)) | lo2.astype(np.uint64)
        ok = (hi2 != hi[idx]) & (bucket_of(cand.view(np.int64), bits) == want[idx])
        hit_idx, first = np.unique(idx[ok], return_index=True)
        out[hit_idx] = cand[ok][first]
        pending = np.setdiff1d(pending, hit_idx, assume_unique=True)
    twins = out.view(np.int64)
    assert (slot_hash(twins) == slot_hash(keys)).all() and (twins != keys).all()
    return twins
