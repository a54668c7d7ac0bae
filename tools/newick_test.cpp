// Prints the Newick line of mash_b200/host/newick.hpp for a tree read from stdin, for tests/test_nj_model.py:
//   n, then n names (one per line, may be empty), then 2n - 2 lines "parent length" (length as a hexadecimal float).
// Build: g++ -O2 -std=c++17 -I mash_b200/host tools/newick_test.cpp -o newick_test
#include <cstdio>
#include <cstdlib>
#include <iostream>
#include <string>
#include <vector>

#include "newick.hpp"

int main()
{
    std::string line;
    std::getline(std::cin, line);
    const size_t n = std::strtoull(line.c_str(), nullptr, 10);
    std::vector<std::string> names(n);
    for (auto &nm : names) std::getline(std::cin, nm);
    std::vector<uint32_t> parent(2 * n - 2);
    std::vector<double> length(2 * n - 2);
    for (size_t v = 0; v < parent.size(); v++) {
        std::getline(std::cin, line);
        char *end = nullptr;
        parent[v] = (uint32_t)std::strtoul(line.c_str(), &end, 10);
        length[v] = std::strtod(end, nullptr);
    }
    mashhost::OutBuf o;
    mashhost::writeNewick(o, parent, length, names);
    fwrite(o.b.data(), 1, o.b.size(), stdout);
    return 0;
}
