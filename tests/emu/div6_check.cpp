// tests/emu/div6_check.cpp — TEST-ONLY: bsb_div6 (bsb_common.h) against the IEEE division v / 6 for every float32
// bit pattern, under FTZ + DAZ (what nvcc -ftz=true does to the device code).  Prints the number of mismatches and
// the first few of them; exit status 0 when there are none.  Built and run by tests/test_chain_overhead.py.
#include <xmmintrin.h>

#include <cstdio>
#include <cstring>
#include <thread>
#include <vector>

#include "bsb_common.h"

static unsigned bits(float f) { unsigned u; std::memcpy(&u, &f, 4); return u; }

static void run(unsigned long long lo, unsigned long long hi, unsigned long long* bad, unsigned* first) {
  _mm_setcsr(_mm_getcsr() | 0x8040u);             // FTZ | DAZ
  unsigned long long n = 0;
  for (unsigned long long i = lo; i < hi; ++i) {
    const unsigned u = (unsigned)i;
    float v;
    std::memcpy(&v, &u, 4);
    volatile float six = 6.f;                      // a real division, never a multiply by a reciprocal
    const float ref = v / six, got = bsb::bsb_div6(v);
    if (bits(ref) != bits(got) && !(ref != ref && got != got)) {
      if (n < 4) first[n] = u;
      ++n;
    }
  }
  *bad = n;
}

int main() {
  const int T = std::max(1u, std::min(32u, std::thread::hardware_concurrency()));
  std::vector<unsigned long long> bad(T);
  std::vector<unsigned> first(4 * T);
  std::vector<std::thread> th;
  const unsigned long long N = 1ull << 32;
  for (int t = 0; t < T; ++t) th.emplace_back(run, N * t / T, N * (t + 1) / T, &bad[t], &first[4 * t]);
  unsigned long long total = 0;
  for (int t = 0; t < T; ++t) {
    th[t].join();
    for (unsigned long long k = 0; k < bad[t] && k < 4; ++k) std::printf("mismatch 0x%08x\n", first[4 * t + k]);
    total += bad[t];
  }
  std::printf("patterns %llu mismatches %llu\n", N, total);
  return total != 0;
}
