// Generator of tests/golden/bloom_kat.json: the reference's bloom_filter.hpp, compiled in place (-I <reference src/mash>),
// constructed as MinHashHeap does for -b (projected 1e9 elements, false_positive_probability 0, maximum_size 8 b bits); prints
// the number of salts, the table size, the salt and compute_indices(hash_ap(key)) for 8-byte and 4-byte keys.
//   g++ -O2 -I <reference>/src/mash tests/golden/bloom_kat.cpp -o kat && ./kat > tests/golden/bloom_kat.json
#include <limits>
#include <cstdio>
#include <cstdint>
#include <cmath>
#include <cstdlib>
#include "bloom_filter.hpp"
struct Peek : bloom_filter {
  Peek(const bloom_parameters &p) : bloom_filter(p) {}
  unsigned long long index(const unsigned char *d, size_t n) const { size_t bi, b; compute_indices(hash_ap(d, n, salt_[0]), bi, b); return bi; }
  size_t salts() const { return salt_.size(); } unsigned salt0() const { return salt_[0]; } unsigned long long bits() const { return table_size_; }
};
int main(int argc, char **argv) {
  const uint64_t max_bytes = argc > 1 ? strtoull(argv[1], 0, 10) : ~0ull;     // skip the tables above this size (memory)
  uint64_t sizes[] = {1000ull, 65536ull, 16ull<<20, 100000000ull, (1ull<<29) + 12345ull, 3ull<<30};
  uint64_t x = 0x9E3779B97F4A7C15ull;
  printf("{\"cases\": [");
  bool first = true;
  for (int si = 0; si < 6; si++) {
    if (sizes[si] > max_bytes) continue;
    bloom_parameters bp; bp.projected_element_count = 1000000000; bp.false_positive_probability = 0; bp.maximum_size = sizes[si] * 8l;
    bp.compute_optimal_parameters();
    Peek f(bp);
    printf("%s{\"bytes\": %llu, \"hashes\": %zu, \"bits\": %llu, \"salt\": %u, \"idx64\": [", first ? "" : ", ", (unsigned long long)sizes[si], f.salts(), f.bits(), f.salt0());
    uint64_t y = x;
    for (int i = 0; i < 64; i++) { y = y * 6364136223846793005ull + 1442695040888963407ull; printf("%s[%llu, %llu]", i ? ", " : "", (unsigned long long)y, f.index((const unsigned char *)&y, 8)); }
    printf("], \"idx32\": [");
    for (int i = 0; i < 64; i++) { y = y * 6364136223846793005ull + 1442695040888963407ull; uint32_t h = (uint32_t)(y >> 17); printf("%s[%u, %llu]", i ? ", " : "", h, f.index((const unsigned char *)&h, 4)); }
    printf("]}");
    first = false;
  }
  printf("]}\n");
}
