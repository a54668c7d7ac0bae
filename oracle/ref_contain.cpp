// ref_contain.cpp -- grid entry point over the reference's OWN containSketches (CommandContain.cpp:231-265), compiled in place by
// oracle/contain.mk into _ref/libmash_ref_contain.so.  Test infrastructure, never the product.
//
// ref_contain_grid: pairs p in [pair_begin, pair_begin + pair_count) of the query-major grid, p = q * n_ref + r, each
// containSketches(reference r, query q) with the reference's HashList built from the row's n hashes (32-bit lists when
// use64 == 0, as HashList stores hash_u); score[p - pair_begin] = its return value, error[...] = the error it sets.
#include <algorithm>
#include <thread>
#include <vector>

#include "CommandContain.h"

namespace {

std::vector<HashList> lists(const uint64_t *h, const uint32_t *n, uint64_t stride, uint64_t count, int use64)
{
    std::vector<HashList> out;
    out.reserve(count);
    for (uint64_t s = 0; s < count; s++) {
        out.emplace_back(use64 != 0);
        for (uint32_t i = 0; i < n[s]; i++) {
            if (use64) out.back().push_back64(h[s * stride + i]);
            else out.back().push_back32((hash32_t)h[s * stride + i]);
        }
    }
    return out;
}

}  // namespace

extern "C" __attribute__((visibility("default")))
void ref_contain_grid(const uint64_t *ref, const uint32_t *ref_n, uint64_t ref_stride, uint64_t n_ref,
                      const uint64_t *qry, const uint32_t *qry_n, uint64_t qry_stride, uint64_t n_qry,
                      uint64_t pair_begin, uint64_t pair_count, int use64, int threads, double *score, double *error)
{
    if (n_ref == 0 || n_qry == 0 || pair_count == 0) return;
    const std::vector<HashList> R = lists(ref, ref_n, ref_stride, n_ref, use64), Q = lists(qry, qry_n, qry_stride, n_qry, use64);
    const uint64_t T = std::max<uint64_t>(1, std::min<uint64_t>((uint64_t)std::max(1, threads), pair_count));
    auto work = [&](uint64_t t) {
        for (uint64_t k = pair_count * t / T; k < pair_count * (t + 1) / T; k++) {
            const uint64_t p = pair_begin + k;
            score[k] = mash::containSketches(R[p % n_ref], Q[p / n_ref], error[k]);
        }
    };
    std::vector<std::thread> pool;
    for (uint64_t t = 1; t < T; t++) pool.emplace_back(work, t);
    work(0);
    for (auto &th : pool) th.join();
}
