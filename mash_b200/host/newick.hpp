// newick.hpp -- the Newick line of `mash triangle -N` (DESIGN.md 3.10): a tree in the parent / length form of
// mashgpu_neighbor_joining_matrix (leaves 0..n-1, the center 2n - 3 with parent UINT32_MAX).
#pragma once
#include <cstdint>
#include <string>
#include <utility>
#include <vector>

#include "fastout.hpp"

namespace mashhost {

// a name as a Newick label: single-quoted, with ' doubled, when it is empty or holds a blank or one of ()[]':;,
inline void newickName(OutBuf &o, const std::string &name)
{
    if (!name.empty() && name.find_first_of(" \t()[]':;,") == std::string::npos) { o.str(name); return; }
    o.ch('\'');
    for (char c : name) { if (c == '\'') o.ch('\''); o.ch(c); }
    o.ch('\'');
}

// The unrooted tree written from its center: children in ascending node id, internal nodes unlabelled, lengths as `cout << v`.
// Iterative, so that a caterpillar of any size fits the stack.
inline void writeNewick(OutBuf &o, const std::vector<uint32_t> &parent, const std::vector<double> &length, const std::vector<std::string> &names)
{
    const uint32_t nodes = (uint32_t)parent.size(), n = (uint32_t)names.size(), center = nodes - 1;
    std::vector<uint32_t> start(nodes + 1, 0), child(nodes);          // children lists, ascending (ids are visited in order)
    for (uint32_t v = 0; v < nodes; v++) if (v != center) start[parent[v] + 1]++;
    for (uint32_t v = 0; v < nodes; v++) start[v + 1] += start[v];
    std::vector<uint32_t> fill(start.begin(), start.end() - 1);
    for (uint32_t v = 0; v < nodes; v++) if (v != center) child[fill[parent[v]]++] = v;
    std::vector<std::pair<uint32_t, uint32_t>> stack{{center, 0}};  // (node, children written)
    while (!stack.empty()) {
        auto &[v, done] = stack.back();
        if (v < n) {                                                   // a leaf
            newickName(o, names[v]); o.ch(':'); o.dbl(length[v]);
            stack.pop_back();
            continue;
        }
        const uint32_t k = start[v + 1] - start[v];
        if (done == k) {
            o.ch(')');
            if (v != center) { o.ch(':'); o.dbl(length[v]); }
            stack.pop_back();
            continue;
        }
        o.ch(done ? ',' : '(');
        const uint32_t c = child[start[v] + done++];
        stack.push_back({c, 0});
    }
    o.ch(';'); o.ch('\n');
}

}  // namespace mashhost
