// ref_taxdb.cpp -- a command-line front end to the REFERENCE'S OWN taxonomy code (test infrastructure).
//
// taxdb.hpp is header-only: it is compiled in place from /root/reference by oracle/taxdb.mk into oracle/_ref/taxdb_ref
// (git-ignored; nothing is copied).  It expects cerr, endl, unordered_map and unordered_set in scope, which the lines below
// provide.  The product path never runs this.
//
//   taxdb_ref <dir> dump              TaxDB(names, nodes) (taxdb.hpp:85-156); every entry as
//                                     "taxid \t parent taxid (itself for a root) \t rank \t name", ascending taxid
//   taxdb_ref <dir> fold              per stdin line of taxIDs: the fold of getLowestCommonAncestor over them in that order,
//                                     as CommandTaxScreen.cpp:420-424 folds a hash's sketches
//   taxdb_ref <dir> report <rows>     stdin lines "taxid taxCount taxHashCount" = counts as the fold loop leaves them
//                                     (:433-439); the roll-up of :442-471 (every taxon present before the loop rolled up
//                                     once, as the loop intends) is restated below; writeReport (taxdb.hpp:192-236) goes to
//                                     stdout, the keys of counts to <rows>: "totalCount totalHashCount", then
//                                     "taxid taxCount taxHashCount cladeCount cladeHashCount" ascending
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <iostream>
#include <map>
#include <sstream>
#include <unordered_map>
#include <unordered_set>

using std::cerr;
using std::endl;
using std::unordered_map;
using std::unordered_set;

#include "taxdb.hpp"

using mash::TaxCounts;
using mash::TaxDB;
using mash::TaxEntry;

int main(int argc, char **argv)
{
    if (argc < 3) { cerr << "usage: taxdb_ref <taxonomy dir> dump | fold | report <rows out>" << endl; return 1; }
    const std::string dir = argv[1], cmd = argv[2];
    TaxDB db(dir + "/names.dmp", dir + "/nodes.dmp");
    if (cmd == "dump") {
        std::map<TaxID, const TaxEntry *> sorted;
        for (auto &e : db.entries) sorted[e.first] = &e.second;
        for (auto &e : sorted)
            printf("%llu\t%llu\t%s\t%s\n", (unsigned long long)e.first, (unsigned long long)(e.second->parent ? e.second->parent->taxID : e.first),
                   e.second->rank.c_str(), e.second->name.c_str());
        return 0;
    }
    if (cmd == "fold") {
        std::string line;
        while (std::getline(std::cin, line)) {
            std::istringstream in(line);
            TaxID t, taxID = 0;
            while (in >> t) taxID = db.getLowestCommonAncestor(t, taxID);
            printf("%llu\n", (unsigned long long)taxID);
        }
        return 0;
    }
    if (cmd == "report" && argc > 3) {
        unordered_map<TaxID, TaxCounts> counts;
        TaxID t;
        uint64_t tc, thc;
        while (std::cin >> t >> tc >> thc) {
            counts[t].taxCount += tc;
            counts[t].taxHashCount += thc;
        }
        std::map<TaxID, TaxCounts> before(counts.begin(), counts.end());
        uint64_t totalCount = 0, totalHashCount = 0;
        for (auto &it : before) {
            const uint64_t hashCount = it.second.taxHashCount, count = it.second.taxCount;
            totalHashCount += hashCount;
            totalCount += count;
            TaxEntry const *taxon = db.getEntry(it.first);
            while (taxon != NULL) {
                counts[taxon->taxID].cladeCount += count;
                counts[taxon->taxID].cladeHashCount += hashCount;
                if (taxon->parent == NULL) break;
                std::vector<TaxID> &children = counts[taxon->parent->taxID].children;
                auto at = std::lower_bound(children.begin(), children.end(), taxon->taxID);
                if (at == children.end() || *at != taxon->taxID) children.insert(at, taxon->taxID);
                taxon = taxon->parent;
            }
        }
        FILE *rows = fopen(argv[3], "w");
        if (!rows) { cerr << "cannot write " << argv[3] << endl; return 1; }
        fprintf(rows, "%llu %llu\n", (unsigned long long)totalCount, (unsigned long long)totalHashCount);
        std::map<TaxID, const TaxCounts *> sorted;
        for (auto &c : counts) sorted[c.first] = &c.second;
        for (auto &c : sorted)
            fprintf(rows, "%llu %llu %llu %llu %llu\n", (unsigned long long)c.first, (unsigned long long)c.second->taxCount,
                    (unsigned long long)c.second->taxHashCount, (unsigned long long)c.second->cladeCount, (unsigned long long)c.second->cladeHashCount);
        fclose(rows);
        db.writeReport(stdout, counts, totalCount, totalHashCount);
        return 0;
    }
    cerr << "unknown command " << cmd << endl;
    return 1;
}
