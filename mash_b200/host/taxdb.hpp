// taxdb.hpp -- NCBI taxonomy dump reader and Kraken-style report writer of `mash taxscreen` (reference taxdb.hpp:85-236).
//
// The reference reads nodes.dmp / names.dmp with iostream extractions (taxdb.hpp:117-125, 138-155); IStream below replays
// exactly those extractions over the file held in memory, so odd files (missing fields, long lines, several scientific names
// per taxID) parse as they do there, at the speed of a byte scan: the 2.7 M-node NCBI dump loads in about a second.
// Nodes are dense: taxid[i], parent[i] (parent[i] == i for a root), rank[i], name[i].  Where the reference is undefined -- a
// parent missing from nodes.dmp leaves TaxEntry::parent uninitialised (taxdb.hpp:37, 92-95) -- the node is a root here.
#pragma once
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <fstream>
#include <iostream>
#include <sstream>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/mashgpu.h"

namespace mashhost {

// the subset of std::istream used by the reference's parsers, with its state rules: an operation on a stream that is not
// good() fails without touching its target; extractions skip leading whitespace; running out of input sets eof
struct IStream {
    const char *p, *end;
    bool eof = false, fail = false;
    IStream(const char *b, const char *e) : p(b), end(e) {}
    explicit operator bool() const { return !fail; }
    bool good() const { return !eof && !fail; }
    static bool space(char c) { return c == ' ' || (c >= '\t' && c <= '\r'); }
    bool skipws()
    {
        if (!good()) { fail = true; return false; }
        while (p < end && space(*p)) p++;
        if (p == end) { eof = fail = true; return false; }
        return true;
    }
    // operator>>(unsigned long): sign, decimal digits; no digits -> 0 and fail, overflow -> max and fail, '-' negates
    IStream &num(uint64_t &v)
    {
        if (!skipws()) return *this;
        bool neg = false;
        if (*p == '+' || *p == '-') { neg = *p == '-'; p++; }
        uint64_t x = 0;
        bool digits = false, over = false;
        while (p < end && *p >= '0' && *p <= '9') {
            const uint64_t d = (uint64_t)(*p - '0');
            if (x > (UINT64_MAX - d) / 10) over = true;
            else x = x * 10 + d;
            digits = true;
            p++;
        }
        if (p == end) eof = true;
        if (!digits) { v = 0; fail = true; }
        else if (over) { v = UINT64_MAX; fail = true; }
        else v = neg ? (uint64_t)0 - x : x;
        return *this;
    }
    IStream &chr(char &c)
    {
        if (!skipws()) return *this;
        c = *p++;
        return *this;
    }
    IStream &word(std::string &w)
    {
        if (!skipws()) return *this;
        const char *b = p;
        while (p < end && !space(*p)) p++;
        w.assign(b, p);
        if (p == end) eof = true;
        return *this;
    }
    void ignore(uint64_t n, int delim = -1)
    {
        if (!good()) { fail = true; return; }
        for (uint64_t i = 0; i < n; i++) {
            if (p == end) { eof = true; return; }
            if (*p++ == delim) return;
        }
    }
    void getline(std::string &s, char delim)
    {
        if (!good()) { fail = true; return; }
        const char *b = p;
        while (p < end && *p != delim) p++;
        s.assign(b, p);
        if (p == end) { eof = true; if (b == p) fail = true; }
        else p++;
    }
};

inline bool readFile(const std::string &path, std::string &out)
{
    std::ifstream f(path, std::ios::binary);
    if (!f.is_open()) return false;
    std::ostringstream ss;
    ss << f.rdbuf();
    out = ss.str();
    return true;
}

struct TaxTree {
    std::vector<uint64_t> taxid;
    std::vector<uint32_t> parent;
    std::vector<std::string> rank, name;
    std::unordered_map<uint64_t, uint32_t> index;

    int64_t find(uint64_t t) const
    {
        auto it = index.find(t);
        return it == index.end() ? -1 : (int64_t)it->second;
    }

    // TaxDB::TaxDB(names, nodes) (taxdb.hpp:85-156) with the same messages on `err`.  Throws std::runtime_error where the
    // reference does (a file that cannot be opened).
    void load(const std::string &namesFile, const std::string &nodesFile, std::ostream &err)
    {
        std::string text;
        if (!readFile(nodesFile, text)) throw std::runtime_error("unable to open nodes file");
        std::vector<uint64_t> parentTaxid;
        {
            IStream in(text.data(), text.data() + text.size());
            uint64_t t = 0, pt = 0;
            char delim = 0;
            std::string r;
            index.reserve(text.size() / 40);
            while (in.num(t).chr(delim).num(pt).chr(delim)) {
                in.ignore(1);
                in.getline(r, '\t');
                if (index.emplace(t, (uint32_t)taxid.size()).second) {       // emplace: the first line of a taxID wins
                    taxid.push_back(t);
                    parentTaxid.push_back(pt);
                    rank.push_back(r);
                }
                in.ignore(2560, '\n');
            }
        }
        const uint32_t n = (uint32_t)taxid.size();
        parent.resize(n);
        name.assign(n, std::string());
        for (uint32_t i = 0; i < n; i++) {
            parent[i] = i;
            if (parentTaxid[i] == taxid[i]) continue;
            const int64_t p = find(parentTaxid[i]);
            if (p < 0) err << "Could not find parent with tax ID " << parentTaxid[i] << " for tax ID " << taxid[i] << std::endl;
            else parent[i] = (uint32_t)p;
        }
        if (!readFile(namesFile, text)) throw std::runtime_error("unable to open names file");
        IStream in(text.data(), text.data() + text.size());
        uint64_t t = 0;
        std::string nm, type;
        while (in.num(t)) {
            in.ignore(3);
            in.getline(nm, '\t');
            in.ignore(3);
            in.ignore(256, '|');
            in.ignore(1);
            in.getline(type, '\t');
            if (type == "scientific name") {
                const int64_t i = find(t);
                if (i < 0) err << "Entry for " << t << " does not exist - it should!" << '\n';
                else name[i] = nm;                                          // the last scientific name wins
            }
            in.ignore(2560, '\n');
        }
        err << "   " << n << " distinct taxa\n";
    }
};

// TaxDB::writeReport (taxdb.hpp:192-236) over the rows of mashgpu_screen_taxonomy (the keys of the reference's counts map).
// Counts are printed as the reference prints them: truncated to unsigned int, %i, and 100 * count in 32-bit arithmetic.
// A node's children are the row nodes whose parent it is, in ascending taxID order, ordered by std::sort on cladeCount
// (descending) as the reference sorts them, so that ties come out in the same order.
inline void writeTaxReport(FILE *fp, const TaxTree &tax, const std::vector<mashgpu_tax_row> &rows, unsigned long totalCounts)
{
    std::unordered_map<uint64_t, const mashgpu_tax_row *> byTaxid;
    byTaxid.reserve(rows.size() * 2);
    std::vector<uint64_t> order;
    for (const auto &r : rows) { byTaxid[r.taxid] = &r; order.push_back(r.taxid); }
    std::sort(order.begin(), order.end());
    std::unordered_map<uint64_t, std::vector<uint64_t>> children;
    for (uint64_t t : order) {
        const int64_t i = tax.find(t);
        if (i < 0 || tax.parent[i] == (uint32_t)i) continue;
        children[tax.taxid[tax.parent[i]]].push_back(t);
    }
    auto row = [&](uint64_t t) -> const mashgpu_tax_row * {
        auto it = byTaxid.find(t);
        return it == byTaxid.end() ? nullptr : it->second;
    };
    std::vector<uint64_t> none;
    struct Writer {
        FILE *fp; const TaxTree &tax; unsigned long totalCounts;
        decltype(row) &get; std::unordered_map<uint64_t, std::vector<uint64_t>> &children; std::vector<uint64_t> &none;
        void operator()(uint64_t t, int depth)
        {
            const mashgpu_tax_row *r = get(t);
            const unsigned int cladeCount = r ? r->clade_count : 0, cladeHashCount = r ? r->clade_hash_count : 0;
            const unsigned int taxCount = r ? r->tax_count : 0, taxHashCount = r ? r->tax_hash_count : 0;
            if (cladeCount == 0) return;
            const int64_t i = tax.find(t);
            fprintf(fp, "%.4f\t%i\t%i\t%i\t%i\t%s\t%llu\t%s%s\n", 100 * cladeCount / double(totalCounts), cladeCount, taxCount, cladeHashCount,
                    taxHashCount, tax.rank[i].c_str(), (unsigned long long)t, std::string(2 * depth, ' ').c_str(), tax.name[i].c_str());
            auto it = children.find(t);
            std::vector<uint64_t> kids = it == children.end() ? none : it->second;
            std::sort(kids.begin(), kids.end(), [&](uint64_t a, uint64_t b) { return get(a)->clade_count > get(b)->clade_count; });
            for (uint64_t c : kids) (*this)(c, depth + 1);
        }
    } write{fp, tax, totalCounts, row, children, none};
    fprintf(fp, "%%\thashes\ttaxHashes\thashesDB\ttaxHashesDB\ttaxID\trank\tname\n");
    const mashgpu_tax_row *r0 = row(0);
    const unsigned int cladeCount0 = r0 ? r0->clade_count : 0, taxCount0 = r0 ? r0->tax_count : 0;
    if (cladeCount0 > 0)
        fprintf(fp, "%.4f\t%i\t%i\tno rank\t0\tunclassified\n", 100 * cladeCount0 / double(totalCounts), cladeCount0, taxCount0);
    write(1, 0);
}

}  // namespace mashhost
