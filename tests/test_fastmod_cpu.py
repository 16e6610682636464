"""fastmod (ngp_common.cuh), which forms the dense hash-grid levels' base index in the fused backward's scatter, equals n % d: the
header's own functions compiled for the host, against `%` over every n below 2^20, the n on both sides of multiples of d and of 2^32,
and random n, for the divisors at the ends of the 32-bit range and random ones."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SRC = r"""
#include "ngp_common.cuh"
#include <cstdio>
void ngp_set_error(const std::string&) {}
static uint64_t rng = 0x9e3779b97f4a7c15ull;
static uint32_t next() { rng ^= rng << 13; rng ^= rng >> 7; rng ^= rng << 17; return (uint32_t)rng; }
static long bad = 0;
static void check(uint32_t n, uint64_t m, uint32_t d) {
    if (fastmod(n, m, d) != n % d && bad++ < 8) printf("d=%u n=%u: %u != %u\n", d, n, fastmod(n, m, d), n % d);
}
int main() {
    uint32_t ds[96] = {1u, 2u, 3u, 5u, 7u, 641u, 4913u, 35937u, 65537u, 274625u, 2146689u, 0x7fffffffu, 0x80000000u, 0x80000001u,
                       0xfffffffeu, 0xffffffffu};
    for (int i = 16; i < 96; ++i) ds[i] = next() >> (next() & 31);
    for (uint32_t d : ds) {
        if (!d) d = 1;
        const uint64_t m = fastmod_m(d);
        if (m != (d == 1 ? 0ull : ~0ull / d + 1) && bad++ < 8) printf("d=%u: m wrong\n", d);
        for (uint32_t n = 0; n < (1u << 20); ++n) check(n, m, d);
        for (uint32_t n = 0; n < (1u << 16); ++n) check(0xffffffffu - n, m, d);
        for (int k = 0; k < 1 << 16; ++k) {
            const uint64_t q = (uint64_t)next() % (0xffffffffull / d + 1), base = q * d;
            for (int e = -2; e <= 2; ++e) if ((int64_t)base + e >= 0 && base + e <= 0xffffffffull) check((uint32_t)(base + e), m, d);
            check(next(), m, d);
        }
    }
    printf("%ld mismatches\n", bad);
    return bad != 0;
}
"""


@pytest.mark.skipif(shutil.which("nvcc") is None, reason="nvcc not available")
def test_fastmod_equals_remainder(tmp_path):
    src, exe = tmp_path / "fastmod.cu", tmp_path / "fastmod"
    src.write_text(SRC)
    r = subprocess.run(["nvcc", "-O2", "-std=c++17", "-I", os.path.join(ROOT, "jnerf_b200", "csrc"), str(src), "-o", str(exe)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    r = subprocess.run([str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-3000:]
