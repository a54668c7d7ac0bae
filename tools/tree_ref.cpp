// A plain CPU reference of the three trees of `mash triangle` as include/mashgpu.h defines them: neighbor joining
// (mashgpu_neighbor_joining_matrix) and average / complete linkage (mashgpu_linkage_matrix).  Every step finds its pair by a full
// scan of the live lower triangle; there are no nearest-neighbour caches and no column compaction, so it shares none of the device's
// shortcuts.  Every arithmetic step is one IEEE double operation in the header's order, so the outputs are the device's bit for bit.
// Only the scan is parallel (OpenMP over rows); its partial minima are reduced by the same strict total order, so the result does
// not depend on the thread count.  Used by tests/test_tree_ref.py and tests/test_gpu_trees_at_scale.py.
//
//   tree_ref nj|average|complete n ld matrix out
// matrix: n rows of ld float64 (raw, native byte order); only the entries j < i of row i are read.
// out, raw arrays in this order:  nj: parent uint32[2n - 2], length float64[2n - 2]
//                                 linkage: id_lo uint32[n - 1], id_hi uint32[n - 1], size uint32[n - 1], height float64[n - 1]
// Build: g++ -O2 -std=c++17 -fopenmp -ffp-contract=off tools/tree_ref.cpp -o tree_ref
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>

namespace {

constexpr uint32_t NONE = 0xFFFFFFFFu;

// the least (value, key) seen; a NaN value is never before anything
struct Best {
    double v = __builtin_inf();
    uint64_t key = ~0ull;
    void offer(double v2, uint64_t k2)
    {
        if (v2 < v || (v2 == v && k2 < key)) { v = v2; key = k2; }
    }
};

// The least (f(row, col), row, col) over live slots col < row, live[] ascending.  f(i, j) gets the positions of the two slots.
template <class F>
Best scan(const std::vector<uint32_t> &live, F f)
{
    Best best;
    const int64_t m = (int64_t)live.size();
#pragma omp parallel
    {
        Best mine;
#pragma omp for schedule(dynamic, 16) nowait
        for (int64_t q = 1; q < m; q++)
            for (int64_t p = 0; p < q; p++) mine.offer(f(q, p), (uint64_t)q << 32 | (uint64_t)p);
#pragma omp critical
        best.offer(mine.v, mine.key);
    }
    return best;
}

// the lower triangle of the input, mirrored, diagonal 0: A[i * n + j] = D(max(i, j), min(i, j))
std::vector<double> symmetric(const std::vector<double> &in, uint64_t n, uint64_t ld)
{
    std::vector<double> A(n * n);
    for (uint64_t i = 0; i < n; i++) {
        A[i * n + i] = 0.0;
        for (uint64_t j = 0; j < i; j++) A[i * n + j] = A[j * n + i] = in[i * ld + j];
    }
    return A;
}

void nj(std::vector<double> A, uint64_t n, std::vector<uint32_t> &parent, std::vector<double> &length)
{
    parent.assign(2 * n - 2, 0);
    length.assign(2 * n - 2, 0.0);
    std::vector<double> r(n);
    for (uint64_t i = 0; i < n; i++) {          // over ascending k, the diagonal's 0 included
        double s = A[i * n];
        for (uint64_t k = 1; k < n; k++) s = s + A[i * n + k];
        r[i] = s;
    }
    // the position of a live slot is its rank among the live slots: u takes a's slot and position, b's are removed
    std::vector<uint32_t> live(n), id(n);
    for (uint64_t i = 0; i < n; i++) live[i] = id[i] = (uint32_t)i;
    for (uint64_t s = 0; s + 3 < n; s++) {
        const uint64_t m = n - s;
        const double mm2 = (double)(m - 2);
        const Best best = scan(live, [&](int64_t q, int64_t p) {
            const uint32_t a = live[p], b = live[q];
            return ((mm2 * A[(uint64_t)b * n + a]) - r[a]) - r[b];
        });
        if (best.key == ~0ull) { std::fprintf(stderr, "tree_ref: no comparable Q at join %llu\n", (unsigned long long)s); std::exit(1); }
        const uint64_t p = best.key & 0xFFFFFFFFu, q = best.key >> 32;
        const uint32_t a = live[p], b = live[q];
        const double dab = A[(uint64_t)b * n + a], ra = r[a], rb = r[b];
        const double la = dab * 0.5 + (ra - rb) / (2.0 * (double)(m - 2));
        parent[id[a]] = parent[id[b]] = (uint32_t)(n + s);
        length[id[a]] = la;
        length[id[b]] = dab - la;
        for (const uint32_t k : live) {
            if (k == a || k == b) continue;
            const double dak = A[(uint64_t)a * n + k], dbk = A[(uint64_t)b * n + k];
            const double duk = ((dak + dbk) - dab) * 0.5;
            r[k] = ((r[k] - dak) - dbk) + duk;
            A[(uint64_t)a * n + k] = A[(uint64_t)k * n + a] = duk;
        }
        r[a] = ((ra + rb) - (double)m * dab) * 0.5;
        id[a] = (uint32_t)(n + s);
        live.erase(live.begin() + q);
    }
    const uint32_t x = live[0], y = live[1], z = live[2];
    const double dxy = A[(uint64_t)y * n + x], dxz = A[(uint64_t)z * n + x], dyz = A[(uint64_t)z * n + y];
    const uint64_t c = 2 * n - 3;
    parent[id[x]] = parent[id[y]] = parent[id[z]] = (uint32_t)c;
    length[id[x]] = ((dxy + dxz) - dyz) * 0.5;
    length[id[y]] = ((dxy + dyz) - dxz) * 0.5;
    length[id[z]] = ((dxz + dyz) - dxy) * 0.5;
    parent[c] = NONE;
    length[c] = 0.0;
}

void linkage(std::vector<double> A, uint64_t n, bool average, std::vector<uint32_t> &lo, std::vector<uint32_t> &hi,
             std::vector<uint32_t> &size_out, std::vector<double> &height)
{
    lo.assign(n - 1, 0);
    hi.assign(n - 1, 0);
    size_out.assign(n - 1, 0);
    height.assign(n - 1, 0.0);
    std::vector<uint32_t> live(n), id(n), size(n, 1);
    for (uint64_t i = 0; i < n; i++) live[i] = id[i] = (uint32_t)i;
    for (uint64_t s = 0; s + 1 < n; s++) {
        // live is ascending, so (value, position of b, position of a) orders as (value, b, a)
        const Best best = scan(live, [&](int64_t q, int64_t p) { return A[(uint64_t)live[q] * n + live[p]]; });
        if (best.key == ~0ull) { std::fprintf(stderr, "tree_ref: no comparable distance at merge %llu\n", (unsigned long long)s); std::exit(1); }
        const uint64_t p = best.key & 0xFFFFFFFFu, q = best.key >> 32;
        const uint32_t a = live[p], b = live[q], na = size[a], nb = size[b];
        lo[s] = id[a] < id[b] ? id[a] : id[b];
        hi[s] = id[a] < id[b] ? id[b] : id[a];
        height[s] = best.v;
        size_out[s] = na + nb;
        for (const uint32_t k : live) {
            if (k == a || k == b) continue;
            const double dak = A[(uint64_t)a * n + k], dbk = A[(uint64_t)b * n + k];
            const double v = average ? ((double)na * dak + (double)nb * dbk) / (double)(na + nb) : (dbk > dak ? dbk : dak);
            A[(uint64_t)a * n + k] = A[(uint64_t)k * n + a] = v;
        }
        size[a] = na + nb;
        id[a] = (uint32_t)(n + s);
        live.erase(live.begin() + q);
    }
}

template <class T>
void put(FILE *f, const std::vector<T> &v)
{
    if (std::fwrite(v.data(), sizeof(T), v.size(), f) != v.size()) { std::perror("tree_ref: write"); std::exit(1); }
}

}  // namespace

int main(int argc, char **argv)
{
    if (argc != 6) {
        std::fprintf(stderr, "usage: tree_ref nj|average|complete n ld matrix out\n");
        return 2;
    }
    const std::string method = argv[1];
    const uint64_t n = std::strtoull(argv[2], nullptr, 10), ld = std::strtoull(argv[3], nullptr, 10);
    const bool is_nj = method == "nj";
    if ((!is_nj && method != "average" && method != "complete") || ld < n || n < (is_nj ? 3u : 2u) || n >= NONE / 2) {
        std::fprintf(stderr, "tree_ref: bad arguments\n");
        return 2;
    }
    std::vector<double> in(n * ld);
    FILE *f = std::fopen(argv[4], "rb");
    if (!f || std::fread(in.data(), sizeof(double), in.size(), f) != in.size()) { std::perror("tree_ref: read"); return 1; }
    std::fclose(f);
    std::vector<double> A = symmetric(in, n, ld);
    in = std::vector<double>();
    FILE *o = std::fopen(argv[5], "wb");
    if (!o) { std::perror("tree_ref: open output"); return 1; }
    if (is_nj) {
        std::vector<uint32_t> parent;
        std::vector<double> length;
        nj(std::move(A), n, parent, length);
        put(o, parent);
        put(o, length);
    } else {
        std::vector<uint32_t> lo, hi, size;
        std::vector<double> height;
        linkage(std::move(A), n, method == "average", lo, hi, size, height);
        put(o, lo);
        put(o, hi);
        put(o, size);
        put(o, height);
    }
    return std::fclose(o) == 0 ? 0 : 1;
}
