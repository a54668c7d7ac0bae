// mash.cpp -- thin command-line front end over the host shim: `mash sketch | dist | triangle | within | screen | taxscreen | info |
// paste`.  Mirrors the reference's command drivers (CommandSketch.cpp:36-169, CommandDistance.cpp:44-304,
// CommandTriangle.cpp:45-214, CommandContain.cpp:33-203, CommandScreen.cpp:54-461, CommandTaxScreen.cpp:57-480,
// CommandInfo.cpp:222-299): same option identifiers and defaults (Command.cpp:165-200), same stdout formats (iostream default
// precision), same ordering contracts.  It exists so that the reference's `make test` flow can be replayed against the GPU engine;
// help text, `bounds` and `find` are out of scope.  `triangle -G` (clusters) and `triangle -T` (the single-linkage tree as a minimum
// spanning forest) have no counterpart in the reference: its users compute both from the `-E` output.  Nor has `triangle -N` (the
// neighbor-joining tree as a Newick line), which its users compute from the matrix with an NJ program, nor `triangle -L` (average
// or complete linkage as a Newick line, or its flat clusters at `-d`), which its users compute from the matrix with scipy, nor
// `triangle -R` (greedy representatives, the dereplication of CD-HIT and skDER), which its users run over the `-E` output, nor
// `screen -I` (each mixture argument screened as its own sample against one table kept on the GPU), which its users get from
// one `mash screen` process per sample.
#include <chrono>
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <iterator>
#include <iostream>
#include <map>
#include <string>
#include <vector>

#include "Sketch.h"
#include <unistd.h>

#include "fastout.hpp"
#include "newick.hpp"
#include "fastx.hpp"
#include "taxdb.hpp"

using namespace std;
using namespace mash;

namespace {

// reference Command::Option (Command.h:28-69, Command.cpp:48-156): numbers are parsed with stof into a float
struct Option {
    enum Type { Boolean, Number, Integer, Size, File, String } type;
    string identifier, argument;
    float number = 0;
    float argMin = 0, argMax = 0;
    bool active = false;
    Option() : type(Boolean) {}
    Option(Type t, const string &id, const string &def, float lo = 0, float hi = 0) : type(t), identifier(id), argMin(lo), argMax(hi) { set(def); }
    void set(string a)
    {
        argument = a;
        if (type == Number || type == Integer) {
            if (a.empty()) { number = 0; return; }
            bool failed = false;
            try {
                number = stof(a);
                if (argMin != argMax && (number < argMin || number > argMax)) failed = true;
                else if (type == Integer && uint64_t(number) != number) failed = true;
            } catch (const exception &) { failed = true; }
            if (failed) {
                cerr << "ERROR: Argument to -" << identifier << " must be a" << (type == Integer ? "n integer" : " number");
                if (argMin != argMax) cerr << " between " << argMin << " and " << argMax;
                cerr << " (" << a << " given)" << endl;
                exit(1);
            }
        } else if (type == Size) {
            if (a.empty()) { number = 0; return; }
            char suffix = a[a.size() - 1];
            uint64_t factor = 1;
            if (suffix < '0' || suffix > '9') {
                switch (suffix) {
                    case 'k': case 'K': factor = 1000; break;
                    case 'm': case 'M': factor = 1000000; break;
                    case 'g': case 'G': factor = 1000000000; break;
                    case 't': case 'T': factor = 1000000000000; break;
                    default:
                        cerr << "ERROR: Unrecognized unit (\"" << suffix << "\") in argument to -" << identifier << ". If specified, unit must be one of [kKmMgGtT]." << endl;
                        exit(1);
                }
                a.resize(a.size() - 1);
            }
            bool fail = false;
            try { number = stof(a); } catch (const exception &) { fail = true; }
            if (number <= 0 || (uint64_t)number != number) fail = true;
            if (fail) {
                cerr << "ERROR: Argument to -" << identifier << " must be a whole number, optionally followed by one of [kKmMgGtT]." << endl;
                exit(1);
            }
            number *= factor;
        }
    }
};

struct Command {
    string name;
    map<string, Option> options;          // by name
    map<string, string> byIdentifier;
    vector<string> arguments;

    void add(const string &n, const Option &o) { options[n] = o; byIdentifier[o.identifier] = n; }
    const Option &opt(const string &n) const { return options.at(n); }
    bool has(const string &n) const { return options.count(n) != 0; }

    void useSketchOptions()   // reference Command.cpp:354-379 with the defaults of :165-200
    {
        add("threads", Option(Option::Integer, "p", "1"));
        add("kmer", Option(Option::Integer, "k", "21", 1, 32));
        add("noncanonical", Option(Option::Boolean, "n", ""));
        add("protein", Option(Option::Boolean, "a", ""));
        add("alphabet", Option(Option::String, "z", ""));
        add("case", Option(Option::Boolean, "Z", ""));
        add("sketchSize", Option(Option::Integer, "s", "1000"));
        add("individual", Option(Option::Boolean, "i", ""));
        add("seed", Option(Option::Integer, "S", "42", 0, 0xFFFFFFFF));
        add("warning", Option(Option::Number, "w", "0.01", 0, 1));
        add("reads", Option(Option::Boolean, "r", ""));
        add("memory", Option(Option::Size, "b", ""));
        add("minCov", Option(Option::Integer, "m", "1"));
        add("targetCov", Option(Option::Number, "c", ""));
        add("genome", Option(Option::Size, "g", ""));
    }

    int parse(int argc, const char **argv)   // reference Command::run(argc, argv), Command.cpp:311-347
    {
        for (int i = 0; i < argc; i++) {
            if (argv[i][0] == '-' && argv[i][1] != 0) {
                if (byIdentifier.count(argv[i] + 1) == 0) {
                    cerr << "ERROR: Unrecognized option: " << argv[i] << endl;
                    return 1;
                }
                Option &option = options.at(byIdentifier.at(argv[i] + 1));
                option.active = true;
                if (option.type != Option::Boolean) {
                    i++;
                    if (i == argc) {
                        cerr << "ERROR: -" << option.identifier << " requires an argument" << endl;
                        return 1;
                    }
                    option.set(argv[i]);
                }
            } else {
                arguments.push_back(argv[i]);
            }
        }
        return 0;
    }
};

// reference sketchParameterSetup.cpp:15-105
int sketchParameterSetup(Sketch::Parameters &parameters, const Command &command)
{
    parameters.kmerSize = command.opt("kmer").number;
    parameters.minHashesPerWindow = command.opt("sketchSize").number;
    parameters.concatenated = !command.opt("individual").active;
    parameters.noncanonical = command.opt("noncanonical").active;
    parameters.seed = command.opt("seed").number;
    parameters.reads = command.opt("reads").active;
    parameters.minCov = command.opt("minCov").number;
    parameters.targetCov = command.opt("targetCov").number;
    parameters.parallelism = command.opt("threads").number;
    parameters.preserveCase = command.opt("case").active;
    if (command.has("warning")) parameters.warning = command.opt("warning").number;
    if (command.opt("memory").active) {
        parameters.reads = true;
        parameters.memoryBound = command.opt("memory").number;
        if (command.opt("minCov").active) {
            cerr << "ERROR: The option " << command.opt("minCov").identifier << " cannot be used with " << command.opt("memory").identifier << "." << endl;
            return 1;
        }
    }
    if (command.opt("minCov").active || command.opt("targetCov").active) parameters.reads = true;
    if (command.opt("genome").active) {
        parameters.reads = true;
        parameters.genomeSize = command.opt("genome").number;
    }
    if (parameters.reads) parameters.counts = true;
    if (parameters.reads && command.opt("threads").active)
        cerr << "WARNING: The option " << command.opt("threads").identifier << " will be ignored with " << command.opt("reads").identifier << "." << endl;
    if (parameters.reads && !parameters.concatenated) {
        cerr << "ERROR: The option " << command.opt("individual").identifier << " cannot be used with " << command.opt("reads").identifier << "." << endl;
        return 1;
    }
    if (command.opt("protein").active) {
        parameters.noncanonical = true;
        setAlphabetFromString(parameters, alphabetProtein);
        if (!command.opt("kmer").active) parameters.kmerSize = 9;
        setAlphabetFromString(parameters, alphabetProtein);   // use64 depends on the final k
    } else if (command.opt("alphabet").active) {
        parameters.noncanonical = true;
        setAlphabetFromString(parameters, command.opt("alphabet").argument.c_str());
    } else {
        setAlphabetFromString(parameters, alphabetNucleotide);
    }
    return 0;
}

void warnKmerSize(const Sketch::Parameters &parameters, uint64_t lengthMax, const string &lengthMaxName, double randomChance, int kMin, int warningCount)
{
    cerr << "\nWARNING: For the k-mer size used (" << parameters.kmerSize << "), the random match probability (" << randomChance
         << ") is above the specified warning threshold (" << parameters.warning << ") for the sequence \"" << lengthMaxName << "\" of size " << lengthMax;
    if (warningCount > 1) cerr << " (and " << (warningCount - 1) << " others)";
    cerr << ". Distances to " << (warningCount == 1 ? "this sequence" : "these sequences")
         << " may be underestimated as a result. To meet the threshold of " << parameters.warning << ", a k-mer size of at least " << kMin
         << " is required. See: -k, -w." << endl << endl;
}

void splitFile(const string &file, vector<string> &lines)   // reference Command.cpp splitFile
{
    ifstream in(file);
    if (!in) { cerr << "ERROR: could not open " << file << " for reading." << endl; exit(1); }
    string line;
    while (getline(in, line)) lines.push_back(line);
}

struct KmerWarning {
    uint64_t lengthMax = 0; double randomChance = 0; int kMin = 0; string lengthMaxName; int warningCount = 0;
    void scan(const Sketch &sketch, const Sketch::Parameters &parameters)
    {
        double lengthThreshold = (parameters.warning * sketch.getKmerSpace()) / (1. - parameters.warning);
        for (uint64_t i = 0; i < sketch.getReferenceCount(); i++) {
            uint64_t length = sketch.getReference(i).length;
            if (length > lengthThreshold) {
                if (warningCount == 0 || length > lengthMax) {
                    lengthMax = length; lengthMaxName = sketch.getReference(i).name;
                    randomChance = sketch.getRandomKmerChance(i); kMin = sketch.getMinKmerSize(i);
                }
                warningCount++;
            }
        }
    }
};

void gpuFail()
{
    cerr << "ERROR: " << mashgpu_last_error(gpuContext()) << endl;
    exit(1);
}

// ---------------------------------------------------------------------------------------------------- sketch
int runSketch(int argc, const char **argv)
{
    Command c;
    c.add("help", Option(Option::Boolean, "h", ""));
    c.add("list", Option(Option::Boolean, "l", ""));
    c.add("prefix", Option(Option::File, "o", ""));
    c.add("id", Option(Option::File, "I", ""));
    c.add("comment", Option(Option::File, "C", ""));
    c.add("counts", Option(Option::Boolean, "M", ""));
    c.useSketchOptions();
    if (c.parse(argc, argv)) return 1;
    if (c.arguments.size() == 0 || c.opt("help").active) { cerr << "usage: mash sketch [options] <input> [<input>] ..." << endl; return 0; }
    Sketch::Parameters parameters;
    parameters.counts = c.opt("counts").active;
    if (sketchParameterSetup(parameters, c)) return 1;
    vector<string> files;
    for (auto &a : c.arguments) { if (c.opt("list").active) splitFile(a, files); else files.push_back(a); }
    if (c.opt("id").active || c.opt("comment").active)
        if (files.size() > 1 && !parameters.reads) cerr << "WARNING: -I and -C will only apply to first sketch" << endl;
    Sketch sketch;
    const bool trace = getenv("MASHGPU_TRACE") != 0;
    const auto tStart = std::chrono::steady_clock::now();
    auto elapsed = [&]() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - tStart).count(); };
    if (parameters.reads) sketch.initFromReads(files, parameters);
    else sketch.initFromFiles(files, parameters, trace ? 0 : 1);
    if (trace) cerr << "[mash] parse + sketch of " << files.size() << " files: " << elapsed() << " ms" << endl;
    if (c.opt("id").active) sketch.setReferenceName(0, c.opt("id").argument);
    if (c.opt("comment").active) sketch.setReferenceComment(0, c.opt("comment").argument);
    KmerWarning w;
    w.scan(sketch, parameters);
    string prefix = c.opt("prefix").argument.length() > 0 ? c.opt("prefix").argument : (c.arguments[0] == "-" ? string("stdin") : c.arguments[0]);
    if (!hasSuffix(prefix, suffixSketch)) prefix += suffixSketch;
    cerr << "Writing to " << prefix << "..." << endl;
    sketch.writeToCapnp(prefix.c_str());
    if (trace) cerr << "[mash] .msh written at " << elapsed() << " ms" << endl;
    if (w.warningCount > 0 && !parameters.reads) warnKmerSize(parameters, w.lengthMax, w.lengthMaxName, w.randomChance, w.kMin, w.warningCount);
    return 0;
}

// ---------------------------------------------------------------------------------------------------- dist
// one line of dist's output (reference CommandDistance.cpp:247-304): reference, query (name:comment with -C) and the pair's values
static void writePair(mashhost::OutBuf &o, const Sketch &sketchRef, uint64_t r, const Sketch &sketchQuery, uint64_t q, bool comment,
                      double distance, double pValue, uint64_t numer, uint64_t denom)
{
    o.str(sketchRef.getReference(r).name);
    if (comment) { o.ch(':'); o.str(sketchRef.getReference(r).comment); }
    o.ch('\t'); o.str(sketchQuery.getReference(q).name);
    if (comment) { o.ch(':'); o.str(sketchQuery.getReference(q).comment); }
    o.ch('\t'); o.dbl(distance); o.ch('\t'); o.dbl(pValue); o.ch('\t'); o.u64(numer); o.ch('/'); o.u64(denom); o.ch('\n');
}

struct PairBlock {
    vector<uint32_t> numer, denom; vector<double> distance, pValue; vector<uint8_t> pass;
    void resize(size_t n) { numer.resize(n); denom.resize(n); distance.resize(n); pValue.resize(n); pass.resize(n); }
};

// `mash dist -B`: per query its nBest nearest references that share a hash with it, nearest first, in the five columns of writeOutput.
// The engine selects on the device and returns rows x nBest entries, so the blocks are sized by that and not by rows x nRef.
static void writeBestHits(mashgpu_dist_job *job, uint32_t nBest, const Sketch &sketchRef, const Sketch &sketchQuery, bool comment, int threads)
{
    const uint64_t nQry = sketchQuery.getReferenceCount();
    const uint64_t rows = std::min<uint64_t>(nQry, std::max<uint64_t>(1, (1ull << 22) / nBest));
    vector<uint32_t> hits(rows), ref(rows * nBest), numer(rows * nBest), denom(rows * nBest);
    vector<double> distance(rows * nBest), pValue(rows * nBest);
    for (uint64_t q = 0; q < nQry; q += rows) {
        const uint64_t r = std::min(rows, nQry - q);
        if (mashgpu_dist_run_best(job, q, r, nBest, hits.data(), 0, ref.data(), numer.data(), denom.data(), distance.data(), pValue.data()) != MASHGPU_OK) gpuFail();
        mashhost::writeRows(r, threads, nBest, [&](uint64_t i, mashhost::OutBuf &o) {
            for (uint64_t e = i * nBest; e < i * nBest + hits[i]; e++)
                writePair(o, sketchRef, ref[e], sketchQuery, q + i, comment, distance[e], pValue[e], numer[e], denom[e]);
        });
    }
}

int runDist(int argc, const char **argv)
{
    Command c;
    c.add("help", Option(Option::Boolean, "h", ""));
    c.add("list", Option(Option::Boolean, "l", ""));
    c.add("table", Option(Option::Boolean, "t", ""));
    c.add("pvalue", Option(Option::Number, "v", "1.0", 0., 1.));
    c.add("distance", Option(Option::Number, "d", "1.0", 0., 1.));
    c.add("comment", Option(Option::Boolean, "C", ""));
    c.add("best", Option(Option::Integer, "B", "", 1, 1024));      // not an option of the reference: its users pipe into sort
    c.useSketchOptions();
    if (c.parse(argc, argv)) return 1;
    if (c.arguments.size() < 2 || c.opt("help").active) {
        cerr << "usage: mash dist [options] <reference> <query> [<query>] ..." << endl
             << "  -B <int>  Best hits: per query only its <int> nearest references that share a hash with it, nearest first (1-1024; not with -t)." << endl;
        return 0;
    }
    bool table = c.opt("table").active, comment = c.opt("comment").active;
    const uint32_t nBest = c.opt("best").active ? (uint32_t)c.opt("best").number : 0;
    if (nBest && table) { cerr << "ERROR: The option -B cannot be used with -t (a table has one column per reference)." << endl; return 1; }
    double pValueMax = c.opt("pvalue").number, distanceMax = c.opt("distance").number;
    Sketch::Parameters parameters;
    if (sketchParameterSetup(parameters, c)) return 1;
    Sketch sketchRef;
    const string &fileReference = c.arguments[0];
    bool isSketch = hasSuffix(fileReference, suffixSketch);
    if (isSketch) {
        for (const char *o : {"kmer", "noncanonical", "protein", "alphabet"})
            if (c.opt(o).active) {
                cerr << "ERROR: The option -" << c.opt(o).identifier << " cannot be used when a sketch is provided; it is inherited from the sketch." << endl;
                return 1;
            }
    } else {
        cerr << "Sketching " << fileReference << " (provide sketch file made with \"mash sketch\" to skip)...";
    }
    vector<string> refArgVector(1, fileReference);
    sketchRef.initFromFiles(refArgVector, parameters);
    KmerWarning w;
    if (isSketch) {
        if (c.opt("sketchSize").active && parameters.reads && parameters.minHashesPerWindow != sketchRef.getMinHashesPerWindow()) {
            cerr << "ERROR: The sketch size must match the reference when using a bloom filter (leave this option out to inherit from the reference sketch)." << endl;
            return 1;
        }
        parameters.minHashesPerWindow = sketchRef.getMinHashesPerWindow();
        parameters.kmerSize = sketchRef.getKmerSize();
        parameters.noncanonical = sketchRef.getNoncanonical();
        parameters.preserveCase = sketchRef.getPreserveCase();
        parameters.seed = sketchRef.getHashSeed();
        string alphabet;
        sketchRef.getAlphabetAsString(alphabet);
        setAlphabetFromString(parameters, alphabet.c_str());
    } else {
        w.scan(sketchRef, parameters);
        cerr << "done.\n";
    }
    if (table) {
        cout << "#query";
        for (uint64_t i = 0; i < sketchRef.getReferenceCount(); i++) cout << '\t' << sketchRef.getReference(i).name;
        cout << endl;
    }
    vector<string> queryFiles;
    for (size_t i = 1; i < c.arguments.size(); i++) { if (c.opt("list").active) splitFile(c.arguments[i], queryFiles); else queryFiles.push_back(c.arguments[i]); }
    Sketch sketchQuery;
    sketchQuery.initFromFiles(queryFiles, parameters, 0, true);

    const uint64_t nRef = sketchRef.getReferenceCount(), nQry = sketchQuery.getReferenceCount();
    if (nRef && nQry) {
        uint64_t sketchSize = sketchQuery.getMinHashesPerWindow() < sketchRef.getMinHashesPerWindow() ? sketchQuery.getMinHashesPerWindow() : sketchRef.getMinHashesPerWindow();
        mashgpu_dist_params dp = {sketchSize, sketchRef.getKmerSize(), sketchRef.getKmerSpace(), distanceMax, pValueMax};
        mashgpu_sketch_set setRef, setQry;
        vector<uint64_t> hR, lR, hQ, lQ; vector<uint32_t> nR, nQ;
        sketchRef.toSketchSet(setRef, hR, nR, lR);
        sketchQuery.toSketchSet(setQry, hQ, nQ, lQ);
        mashgpu_dist_job *job = 0;
        if (mashgpu_dist_open(gpuContext(), &setRef, &setQry, &dp, &job) != MASHGPU_OK) gpuFail();
        if (nBest) writeBestHits(job, nBest, sketchRef, sketchQuery, comment, parameters.parallelism);
        const uint64_t nDense = nBest ? 0 : nQry;       // queries still to be printed pair by pair
        uint64_t rows = std::max<uint64_t>(1, (1ull << 24) / nRef);
        PairBlock out;
        out.resize(std::min(rows, nDense) * nRef);
        // with -d / -v filters only the passing pairs are needed (writeOutput prints nothing else): ask the engine for the
        // compacted pass-list, already in query-major order, instead of the dense grid
        const bool filtered = !table && (distanceMax < 1.0 || pValueMax < 1.0);
        const uint64_t listCapacity = 1ull << 22;
        vector<uint64_t> lIdx; vector<uint32_t> lNumer, lDenom; vector<double> lDist, lP;
        if (filtered) { lIdx.resize(listCapacity); lNumer.resize(listCapacity); lDenom.resize(listCapacity); lDist.resize(listCapacity); lP.resize(listCapacity); }
        for (uint64_t q = 0; q < nDense; q += rows) {
            uint64_t r = std::min(rows, nQry - q);
            if (filtered) {
                uint64_t nPass = 0;
                if (mashgpu_dist_run_list(job, q, r, listCapacity, lIdx.data(), lNumer.data(), lDenom.data(), lDist.data(), lP.data(), &nPass) != MASHGPU_OK) gpuFail();
                if (nPass <= listCapacity) {
                    mashhost::writeRows(nPass, parameters.parallelism, 1, [&](uint64_t e, mashhost::OutBuf &o) {
                        writePair(o, sketchRef, lIdx[e] % nRef, sketchQuery, q + lIdx[e] / nRef, comment, lDist[e], lP[e], lNumer[e], lDenom[e]);
                    });
                    continue;
                }
                // more passing pairs than the list holds: dense path for this block
            }
            if (mashgpu_dist_run(job, q, r, out.numer.data(), out.denom.data(), out.distance.data(), out.pValue.data(), out.pass.data()) != MASHGPU_OK) gpuFail();
            mashhost::writeRows(r, parameters.parallelism, nRef, [&](uint64_t i, mashhost::OutBuf &o) {   // == writeOutput, reference CommandDistance.cpp:247-304
                for (uint64_t j = 0; j < nRef; j++) {
                    size_t k = i * nRef + j;
                    if (table && j == 0) o.str(sketchQuery.getReference(q + i).name);
                    if (table) {
                        o.ch('\t');
                        if (out.pass[k]) o.dbl(out.distance[k]);
                    } else if (out.pass[k]) {
                        writePair(o, sketchRef, j, sketchQuery, q + i, comment, out.distance[k], out.pValue[k], out.numer[k], out.denom[k]);
                    }
                }
                if (table) o.ch('\n');
            });
        }
        mashgpu_dist_close(job);
    }
    if (w.warningCount > 0 && !parameters.reads) warnKmerSize(parameters, w.lengthMax, w.lengthMaxName, w.randomChance, w.kMin, w.warningCount);
    return 0;
}

// ---------------------------------------------------------------------------------------------------- within
int runWithin(int argc, const char **argv)   // reference CommandContain.cpp:33-203
{
    Command c;
    c.add("help", Option(Option::Boolean, "h", ""));
    c.add("list", Option(Option::Boolean, "l", ""));
    c.add("errorThreshold", Option(Option::Number, "e", "0.05"));
    c.useSketchOptions();
    if (c.parse(argc, argv)) return 1;
    if (c.arguments.size() < 2 || c.opt("help").active) { cerr << "usage: mash within [options] <reference> <query> [<query>] ..." << endl; return 0; }
    const float errorMax = c.opt("errorThreshold").number;      // writeOutput takes it as a float (:179)
    Sketch::Parameters parameters;
    if (sketchParameterSetup(parameters, c)) return 1;
    Sketch sketchRef;
    const string &fileReference = c.arguments[0];
    bool isSketch = hasSuffix(fileReference, suffixSketch);
    if (isSketch) {
        // no dash before the identifier here (unlike dist); -a and -z are reported and ignored (:60-82)
        for (const char *o : {"kmer", "noncanonical", "protein", "alphabet"})
            if (c.opt(o).active) {
                cerr << "ERROR: The option " << c.opt(o).identifier << " cannot be used when a sketch is provided; it is inherited from the sketch." << endl;
                if (!strcmp(o, "kmer") || !strcmp(o, "noncanonical")) return 1;
            }
    } else {
        cerr << "Sketching " << fileReference << " (provide sketch file made with \"mash sketch\" to skip)...";
    }
    vector<string> refArgVector(1, fileReference);
    sketchRef.initFromFiles(refArgVector, parameters);
    if (isSketch) {
        parameters.minHashesPerWindow = sketchRef.getMinHashesPerWindow();
        parameters.kmerSize = sketchRef.getKmerSize();
        parameters.noncanonical = sketchRef.getNoncanonical();
        parameters.preserveCase = sketchRef.getPreserveCase();
        parameters.seed = sketchRef.getHashSeed();
        string alphabet;
        sketchRef.getAlphabetAsString(alphabet);
        setAlphabetFromString(parameters, alphabet.c_str());
    } else {
        cerr << "done.\n";
    }
    vector<string> queryFiles;
    for (size_t i = 1; i < c.arguments.size(); i++) { if (c.opt("list").active) splitFile(c.arguments[i], queryFiles); else queryFiles.push_back(c.arguments[i]); }
    Sketch sketchQuery;
    sketchQuery.initFromFiles(queryFiles, parameters, 0, true, true);      // contain: a query .msh with a smaller s is used, not skipped

    // With no reference sketch the reference divides by zero (iFloor, :137); here nothing is printed.
    const uint64_t nRef = sketchRef.getReferenceCount(), nQry = sketchQuery.getReferenceCount();
    if (nRef && nQry) {
        mashgpu_sketch_set setRef, setQry;
        vector<uint64_t> hR, lR, hQ, lQ; vector<uint32_t> nR, nQ;
        sketchRef.toSketchSet(setRef, hR, nR, lR);
        sketchQuery.toSketchSet(setQry, hQ, nQ, lQ);
        mashgpu_within_job *job = 0;
        if (mashgpu_within_open(gpuContext(), &setRef, &setQry, (double)errorMax, &job) != MASHGPU_OK) gpuFail();
        const uint64_t rows = std::max<uint64_t>(1, (1ull << 24) / nRef);
        vector<double> score, error; vector<uint8_t> pass;
        const uint64_t cap = std::min(rows, nQry) * nRef;
        score.resize(cap); error.resize(cap); pass.resize(cap);
        for (uint64_t q = 0; q < nQry; q += rows) {
            const uint64_t r = std::min(rows, nQry - q);
            if (mashgpu_within_run(job, q, r, nullptr, nullptr, score.data(), error.data(), pass.data()) != MASHGPU_OK) gpuFail();
            mashhost::writeRows(r, parameters.parallelism, nRef, [&](uint64_t i, mashhost::OutBuf &o) {   // == writeOutput, :179-203
                for (uint64_t j = 0; j < nRef; j++) {
                    const size_t k = i * nRef + j;
                    if (!pass[k]) continue;
                    o.dbl(score[k]); o.ch('\t'); o.dbl(error[k]); o.ch('\t');
                    o.str(sketchRef.getReference(j).name); o.ch('\t'); o.str(sketchQuery.getReference(q + i).name); o.ch('\n');
                }
            });
        }
        mashgpu_within_close(job);
    }
    return 0;
}

// ---------------------------------------------------------------------------------------------------- triangle
// a sketch as triangle prints it: its comment with -C, else its name
static const string &sketchLabel(const Sketch &s, uint64_t i, bool comment) { return comment ? s.getReference(i).comment : s.getReference(i).name; }

// the -E line of the pair (row, col): both sketches, distance, p-value and shared hashes
static void writeEdge(mashhost::OutBuf &o, const Sketch &sketch, uint64_t row, uint64_t col, bool comment, double distance, double pValue,
                      uint64_t numer, uint64_t denom)
{
    o.str(sketchLabel(sketch, row, comment)); o.ch('\t'); o.str(sketchLabel(sketch, col, comment)); o.ch('\t');
    o.dbl(distance); o.ch('\t'); o.dbl(pValue); o.ch('\t'); o.u64(numer); o.ch('/'); o.u64(denom); o.ch('\n');
}

// `-G`, and `-L` with -d: one line per sketch in input order, its name (comment with -C) and its cluster.  Sketches of one cluster
// share a key (key[i] < keys); the clusters are numbered from 0 in the order of their first member.  Returns the cluster count.
static uint32_t writeClusterLines(const Sketch &sketch, bool comment, int threads, const vector<uint32_t> &key, uint64_t keys)
{
    const uint64_t n = sketch.getReferenceCount();
    vector<uint32_t> number(keys, UINT32_MAX), cluster(n);
    uint32_t clusters = 0;
    for (uint64_t i = 0; i < n; i++) cluster[i] = number[key[i]] == UINT32_MAX ? (number[key[i]] = clusters++) : number[key[i]];
    mashhost::writeRows(n, threads, 1, [&](uint64_t i, mashhost::OutBuf &o) {
        o.str(sketchLabel(sketch, i, comment)); o.ch('\t'); o.u64(cluster[i]); o.ch('\n');
    });
    return clusters;
}

// `-N`, and `-L` without -d: the tree (writeNewick's parent / length form) as one Newick line; one sketch is its name alone
static void writeNewickLine(const Sketch &sketch, bool comment, const vector<uint32_t> &parent, const vector<double> &length)
{
    const uint64_t n = sketch.getReferenceCount();
    vector<string> names(n);
    for (uint64_t i = 0; i < n; i++) names[i] = sketchLabel(sketch, i, comment);
    mashhost::OutBuf o;
    if (n == 1) { mashhost::newickName(o, names[0]); o.ch(';'); o.ch('\n'); }
    else if (n > 1) mashhost::writeNewick(o, parent, length, names);
    cout.flush();
    fwrite(o.b.data(), 1, o.b.size(), stdout);
    fflush(stdout);
}

// the self job over every sketch, with the -d / -v thresholds; with `order`, job row t is sketch order[t]
static mashgpu_dist_job *openSelfJob(const Sketch &sketch, double distanceMax, double pValueMax, const vector<uint32_t> *order = nullptr)
{
    mashgpu_dist_params dp = {(uint64_t)sketch.getMinHashesPerWindow(), sketch.getKmerSize(), sketch.getKmerSpace(), distanceMax, pValueMax};
    mashgpu_sketch_set set;
    vector<uint64_t> h, l; vector<uint32_t> nn;
    sketch.toSketchSet(set, h, nn, l);
    if (order) {
        vector<uint64_t> ph(h.size()), pl(l.size()); vector<uint32_t> pn(nn.size());
        for (uint64_t t = 0; t < order->size(); t++) {
            const uint64_t i = (*order)[t];
            std::copy(h.begin() + i * set.stride, h.begin() + (i + 1) * set.stride, ph.begin() + t * set.stride);
            pn[t] = nn[i]; pl[t] = l[i];
        }
        h.swap(ph); nn.swap(pn); l.swap(pl);
        set.hashes = h.data(); set.n_hashes = nn.data(); set.length = l.data();
    }
    mashgpu_dist_job *job = 0;
    if (mashgpu_dist_open(gpuContext(), &set, 0, &dp, &job) != MASHGPU_OK) gpuFail();
    return job;
}

// `mash triangle -G`: per sketch its cluster, the connected component of the pairs that pass -d / -v and share a hash, built on the
// device.  The label the engine returns is the smallest index of the component, its first member.
static void writeClusters(mashgpu_dist_job *job, const Sketch &sketch, bool comment, int threads)
{
    const uint64_t n = sketch.getReferenceCount();
    vector<uint32_t> label(n);
    uint64_t edges = 0;
    if (n && mashgpu_dist_components(job, label.data(), &edges) != MASHGPU_OK) gpuFail();
    const uint32_t clusters = writeClusterLines(sketch, comment, threads, label, n);
    cerr << "Clusters: " << clusters << " from " << edges << " edges" << endl;
}

// `mash triangle -T`: the minimum spanning forest of the same graph, weighted by distance (ties broken by the smaller, then the
// larger sketch index), built on the device.  One `-E` line per forest edge, in forest order: the lines up to distance t are a
// forest of the clusters `-G -d t` gives, so a cut at any t <= -d is a prefix of the output (single linkage).
static void writeForest(mashgpu_dist_job *job, const Sketch &sketch, bool comment, int threads)
{
    const uint64_t n = sketch.getReferenceCount(), cap = n ? n - 1 : 0;
    vector<uint32_t> row(cap), col(cap), numer(cap), denom(cap);
    vector<double> distance(cap), pValue(cap);
    uint64_t edges = 0, rounds = 0;
    if (n > 1 && mashgpu_dist_spanning_forest(job, row.data(), col.data(), numer.data(), denom.data(), distance.data(), pValue.data(), &edges,
                                              &rounds) != MASHGPU_OK) gpuFail();
    mashhost::writeRows(edges, threads, 1, [&](uint64_t e, mashhost::OutBuf &o) {      // the -E line of the pair (q = row, r = col)
        writeEdge(o, sketch, row[e], col[e], comment, distance[e], pValue[e], numer[e], denom[e]);
    });
    cerr << "Forest: " << edges << " edges, " << n - edges << " trees in " << rounds << " rounds" << endl;
}

// `mash triangle -N`: the neighbor-joining tree of every pair's distance (DESIGN.md 3.10) as one Newick line.  Two sketches are a
// cherry with half the distance on each branch; from three on the tree is built on the device.
static void writeNeighborJoining(mashgpu_dist_job *job, const Sketch &sketch, bool comment)
{
    const uint64_t n = sketch.getReferenceCount();
    vector<uint32_t> parent(n > 2 ? 2 * n - 2 : 0);
    vector<double> length(parent.size());
    if (n > 2 && mashgpu_dist_neighbor_joining(job, parent.data(), length.data()) != MASHGPU_OK) gpuFail();
    if (n == 2) {
        double d[2] = {0, 0};                                                          // row q = 1: (1, 0) and (1, 1)
        if (mashgpu_dist_run(job, 1, 1, 0, 0, d, 0, 0) != MASHGPU_OK) gpuFail();
        parent = {2, 2, UINT32_MAX};                                                   // the cherry's center is node 2
        length = {d[0] * 0.5, d[0] * 0.5, 0.0};
    }
    writeNewickLine(sketch, comment, parent, length);
    cerr << "Tree: " << n << " leaves, " << (n > 3 ? n - 3 : 0) << " joins" << endl;
}

// `mash triangle -L average|complete`: average (UPGMA) or complete linkage of every pair's distance (DESIGN.md 3.11), merged on the
// device.  Without -d, the rooted tree as one Newick line: a merge's node sits at half its height, leaves at 0, and a branch is the
// parent's height minus the child's.  With -d t, per sketch its flat cluster at t in -G's format: scipy's fcluster(Z, t, "distance"),
// a maximal subtree whose every merge has height <= t (the largest height in it, since rounding in the average can make a later
// merge lower by an ulp).  The cut is linked per component of the pairs within about t (DESIGN.md 3.13), so it needs memory for the
// largest component's matrix, not for all n sketches.  One sketch has no merge: its name, or cluster 0.
static void writeLinkage(mashgpu_dist_job *job, const Sketch &sketch, bool comment, int method, bool cutting, double t, int threads)
{
    const uint64_t n = sketch.getReferenceCount(), m = n ? n - 1 : 0, nodes = n + m;
    if (cutting) {
        vector<uint32_t> label(n);
        uint64_t flat = 0, components = 0, largest = 0;
        if (n && mashgpu_dist_linkage_cut(job, method, t, label.data(), 0, 0, 0, 0, &flat, &components, &largest) != MASHGPU_OK) gpuFail();
        const uint32_t clusters = writeClusterLines(sketch, comment, threads, label, n);
        cerr << "Clusters: " << clusters << " at height <= " << t << endl;
        cerr << "Components: " << components << " linked, the largest of " << largest << " sketches" << endl;
        return;
    }
    vector<uint32_t> lo(m), hi(m), size(m);
    vector<double> height(m);
    uint64_t rows = 0;
    if (n > 1 && mashgpu_dist_linkage(job, method, lo.data(), hi.data(), height.data(), size.data(), &rows) != MASHGPU_OK) gpuFail();
    vector<uint32_t> parent(nodes, UINT32_MAX);
    vector<double> length(nodes, 0.0);
    auto nodeHeight = [&](uint64_t v) { return v < n ? 0.0 : height[v - n] * 0.5; };
    for (uint64_t s = 0; s < m; s++) parent[lo[s]] = parent[hi[s]] = (uint32_t)(n + s);
    for (uint64_t v = 0; v + 1 < nodes; v++) length[v] = nodeHeight(parent[v]) - nodeHeight(v);
    writeNewickLine(sketch, comment, parent, length);      // its center, the last node, is the root 2n - 2
    cerr << "Tree: " << n << " leaves, " << m << " merges, " << rows << " rows rescanned" << endl;
}

// `mash triangle -R length|input`: greedy dereplication (DESIGN.md 3.12) in priority order -- longest sketch first (ties by input
// position), or input order.  A sketch is a representative unless a representative before it has a pair with it that passes -d / -v
// and shares a hash; every other sketch goes to its nearest adjacent representative.  The job runs over the sketches in priority order;
// the lines are in input order: name, its representative's name (itself for a representative) and the distance to it.
static void writeRepresentatives(const Sketch &sketch, bool comment, bool byLength, double distanceMax, double pValueMax, int threads)
{
    const uint64_t n = sketch.getReferenceCount();
    vector<uint32_t> order(n);
    for (uint64_t i = 0; i < n; i++) order[i] = (uint32_t)i;
    if (byLength)
        std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return sketch.getReference(a).length > sketch.getReference(b).length; });
    mashgpu_dist_job *job = openSelfJob(sketch, distanceMax, pValueMax, &order);
    vector<uint32_t> rep(n), numer(n), denom(n);
    vector<double> distance(n), pValue(n);
    uint64_t reps = 0, rounds = 0;
    if (n && mashgpu_dist_representatives(job, rep.data(), numer.data(), denom.data(), distance.data(), pValue.data(), &reps, &rounds) != MASHGPU_OK)
        gpuFail();
    mashgpu_dist_close(job);
    vector<uint32_t> repOf(n);              // in input order
    vector<double> distOf(n);
    for (uint64_t t = 0; t < n; t++) { repOf[order[t]] = order[rep[t]]; distOf[order[t]] = distance[t]; }
    mashhost::writeRows(n, threads, 1, [&](uint64_t i, mashhost::OutBuf &o) {
        o.str(sketchLabel(sketch, i, comment)); o.ch('\t'); o.str(sketchLabel(sketch, repOf[i], comment)); o.ch('\t'); o.dbl(distOf[i]); o.ch('\n');
    });
    cerr << "Representatives: " << reps << " of " << n << " sketches in " << rounds << " rounds" << endl;
}

int runTriangle(int argc, const char **argv)
{
    Command c;
    c.add("help", Option(Option::Boolean, "h", ""));
    c.add("list", Option(Option::Boolean, "l", ""));
    c.add("comment", Option(Option::Boolean, "C", ""));
    c.add("edge", Option(Option::Boolean, "E", ""));
    c.add("cluster", Option(Option::Boolean, "G", ""));       // not an option of the reference: its users cluster the -E output
    c.add("tree", Option(Option::Boolean, "T", ""));          // not an option of the reference either
    c.add("nj", Option(Option::Boolean, "N", ""));            // nor is this one
    c.add("linkage", Option(Option::String, "L", ""));        // nor this one
    c.add("representatives", Option(Option::String, "R", ""));        // nor this one
    c.add("pvalue", Option(Option::Number, "v", "1.0", 0., 1.));
    c.add("distance", Option(Option::Number, "d", "1.0", 0., 1.));
    c.useSketchOptions();
    if (c.parse(argc, argv)) return 1;
    if (c.arguments.size() < 1 || c.opt("help").active) {
        cerr << "usage: mash triangle [options] <seq1> [<seq2>] ..." << endl
             << "  -G        Clusters: per sketch its cluster, the connected component of the pairs that pass -d / -v and share a hash (not with -E)." << endl
             << "  -T        Single-linkage tree: the minimum spanning forest of the -G graph by distance, as -E lines in order of distance (not with" << endl
             << "            -E or -G).  The lines up to distance t are the -G clusters at -d t." << endl
             << "  -N        Neighbor-joining tree of every pair's distance, as one Newick line (not with -E, -G, -T, -d or -v)." << endl
             << "  -L <m>    Average or complete linkage (m = average or complete) of every pair's distance as one Newick line; with -d t, per sketch its cluster at height <= t (not with -E, -G, -T, -N or -v)." << endl
             << "            The tree needs an n x n matrix on the device; with -d the limit is the largest component of the pairs within t, not n." << endl
             << "  -R <o>    Greedy representatives in order o (length: longest first, input: input order): a sketch is one unless an earlier one is within -d / -v; per sketch its representative, the nearest, and the distance (not with -E, -G, -T, -N or -L)." << endl;
        return 0;
    }
    bool comment = c.opt("comment").active, edge = c.opt("edge").active, cluster = c.opt("cluster").active, tree = c.opt("tree").active;
    const bool nj = c.opt("nj").active, link = c.opt("linkage").active;
    int linkMethod = -1;
    if (link) {
        const string &m = c.opt("linkage").argument;
        linkMethod = m == "average" ? MASHGPU_LINKAGE_AVERAGE : m == "complete" ? MASHGPU_LINKAGE_COMPLETE : -1;
        if (linkMethod < 0) { cerr << "ERROR: The argument to -L must be average or complete (" << m << " given)." << endl; return 1; }
    }
    const bool reps = c.opt("representatives").active;
    const string &repOrder = c.opt("representatives").argument;
    if (reps && repOrder != "length" && repOrder != "input") {
        cerr << "ERROR: The argument to -R must be length or input (" << repOrder << " given)." << endl;
        return 1;
    }
    // the output modes that replace the matrix, and the options each refuses, in the order they are checked
    const struct { const char *mode, *refused[5], *why; } conflicts[] = {
        {"cluster", {"edge"}, "clusters replace the edge list"},
        {"tree", {"edge"}, "the forest replaces the edge list"},
        {"tree", {"cluster"}, "cut the forest at the distance instead"},
        {"linkage", {"edge", "cluster", "tree", "nj", "pvalue"}, "the tree is built from every pair's distance; -d cuts it"},
        {"nj", {"edge", "cluster", "tree", "distance", "pvalue"}, "the tree is built from every pair's distance"},
        {"representatives", {"edge", "cluster", "tree", "nj", "linkage"}, "the representatives replace the edge list, clusters and trees"},
    };
    for (const auto &t : conflicts)
        for (const char *o : t.refused)
            if (o && c.opt(t.mode).active && c.opt(o).active) {
                cerr << "ERROR: The option -" << c.opt(t.mode).identifier << " cannot be used with -" << c.opt(o).identifier << " (" << t.why << ")." << endl;
                return 1;
            }
    double pValueMax = c.opt("pvalue").number, distanceMax = c.opt("distance").number, pValuePeak = 0;
    if ((c.opt("pvalue").active || c.opt("distance").active) && !cluster && !tree && !link && !reps) edge = true;
    Sketch::Parameters parameters;
    if (sketchParameterSetup(parameters, c)) return 1;
    if (c.arguments.size() == 1 && !c.opt("list").active) parameters.concatenated = false;
    vector<string> queryFiles;
    for (auto &a : c.arguments) { if (c.opt("list").active) splitFile(a, queryFiles); else queryFiles.push_back(a); }
    Sketch sketch;
    sketch.initFromFiles(queryFiles, parameters);
    KmerWarning w;
    w.scan(sketch, parameters);
    const uint64_t n = sketch.getReferenceCount();
    if (reps) {
        writeRepresentatives(sketch, comment, repOrder == "length", distanceMax, pValueMax, parameters.parallelism);
        if (w.warningCount > 0 && !parameters.reads) warnKmerSize(parameters, w.lengthMax, w.lengthMaxName, w.randomChance, w.kMin, w.warningCount);
        return 0;
    }
    if (cluster || tree || nj || link) {
        mashgpu_dist_job *job = openSelfJob(sketch, distanceMax, pValueMax);
        // the cut is the -d argument read as a double, so that -d 0.1 cuts where fcluster(Z, 0.1, "distance") does (-d itself is a float)
        if (link) writeLinkage(job, sketch, comment, linkMethod, c.opt("distance").active, strtod(c.opt("distance").argument.c_str(), nullptr),
                               parameters.parallelism);
        else if (nj) writeNeighborJoining(job, sketch, comment);
        else if (tree) writeForest(job, sketch, comment, parameters.parallelism);
        else writeClusters(job, sketch, comment, parameters.parallelism);
        mashgpu_dist_close(job);
        if (w.warningCount > 0 && !parameters.reads) warnKmerSize(parameters, w.lengthMax, w.lengthMaxName, w.randomChance, w.kMin, w.warningCount);
        return 0;
    }
    if (!edge) {
        cout << '\t' << n << endl;
        cout << sketchLabel(sketch, 0, comment) << endl;
    }
    if (n > 1) {
        // row i vs 0..i-1 (reference CommandTriangle.cpp:200-214): reference = sketch i, "query" = sketch j < i.
        // compareSketches(ref = row sketch, qry = column sketch); shared counts and distance are symmetric, the
        // p-value is symmetric in the two lengths, so the all-vs-all job's (q = i, r = j) entry is the same value.
        mashgpu_dist_job *job = openSelfJob(sketch, distanceMax, pValueMax);
        if (mashgpu_dist_set_triangle(job, 1) != MASHGPU_OK) gpuFail();     // only j < i is read below
        uint64_t rows = std::max<uint64_t>(1, (1ull << 24) / n);
        PairBlock out;
        out.resize(std::min(rows, n) * n);
        for (uint64_t q = 1; q < n; q += rows) {
            uint64_t r = std::min(rows, n - q);
            if (mashgpu_dist_run(job, q, r, out.numer.data(), out.denom.data(), out.distance.data(), out.pValue.data(), out.pass.data()) != MASHGPU_OK) gpuFail();
            mashhost::writeRows(r, parameters.parallelism, n, [&](uint64_t i, mashhost::OutBuf &o) {   // == writeOutput, reference CommandTriangle.cpp:159-198
                if (!edge) o.str(sketchLabel(sketch, q + i, comment));
                for (uint64_t j = 0; j < q + i; j++) {
                    size_t k = i * n + j;
                    if (!edge) { o.ch('\t'); o.dbl(out.distance[k]); }
                    else if (out.pass[k]) writeEdge(o, sketch, q + i, j, comment, out.distance[k], out.pValue[k], out.numer[k], out.denom[k]);
                }
                if (!edge) o.ch('\n');
            });
            for (uint64_t i = 0; i < r; i++)
                for (uint64_t j = 0; j < q + i; j++)
                    if (out.pValue[i * n + j] > pValuePeak) pValuePeak = out.pValue[i * n + j];
        }
        mashgpu_dist_close(job);
    }
    if (!edge) cerr << "Max p-value: " << pValuePeak << endl;
    if (w.warningCount > 0 && !parameters.reads) warnKmerSize(parameters, w.lengthMax, w.lengthMaxName, w.randomChance, w.kMin, w.warningCount);
    return 0;
}

// ---------------------------------------------------------------------------------------------------- screen
// The stream of `mash screen` and `mash taxscreen` (CommandScreen.cpp:156-270, CommandTaxScreen.cpp:212-384): round robin over
// the input files, '*'-joined chunks of 64 MiB instead of 1 MiB (any split gives the same counts) fed to the job.  Returns the
// number of sequence records; exits with the reference's messages on a file it cannot open or read.
uint64_t feedInputs(mashgpu_screen_job *job, const vector<string> &files, int kmerSize)
{
    vector<gzFile> fps;
    std::vector<mashhost::FastxReader *> readers;
    for (size_t f = 0; f < files.size(); f++) {
        const string &file = files[f];
        if (file == "-" && f > 0) { cerr << "ERROR: '-' for stdin must be first query" << endl; exit(1); }
        gzFile fp = mashhost::FastxReader::openPath(file);
        if (fp == 0) { cerr << "ERROR: could not open " << file << endl; exit(1); }
        fps.push_back(fp);
        readers.push_back(new mashhost::FastxReader(fp));
    }
    const size_t chunkSize = 64u << 20;
    string input;
    input.reserve(chunkSize + (1 << 20));
    uint64_t count = 0;
    int lstate = 0;
    size_t it = 0;
    auto flush = [&]() {
        if (input.empty()) return;
        if (mashgpu_screen_feed(job, input.data(), input.size()) != MASHGPU_OK) gpuFail();
        input.clear();
    };
    while (!readers.empty()) {
        int len = readers[it]->read();
        lstate = len;
        if (len < -1) break;
        if (len == -1) {
            delete readers[it];
            readers.erase(readers.begin() + it);
            if (it >= readers.size()) it = 0;
            continue;
        }
        if (input.length() + (len >= kmerSize ? len + 1 : 0) > chunkSize) flush();
        count++;
        if (len >= kmerSize) {
            input.append(1, '*');
            input.append(readers[it]->seq.data(), readers[it]->seq.size());
        }
        it++;
        if (it >= readers.size()) it = 0;
    }
    flush();
    if (lstate != -1) { cerr << "\nERROR: reading inputs" << endl; exit(1); }
    for (gzFile fp : fps) gzclose(fp);
    return count;
}

// all inputs arguments[1..] pooled into one mixture
void streamInputs(mashgpu_screen_job *job, const vector<string> &arguments, int kmerSize, bool trans)
{
    int queryCount = (int)arguments.size() - 1;
    cerr << (trans ? "Translating from " : "Streaming from ");
    if (queryCount == 1) cerr << arguments[1]; else cerr << queryCount << " inputs";
    cerr << "..." << endl;
    const uint64_t count = feedInputs(job, vector<string>(arguments.begin() + 1, arguments.end()), kmerSize);
    if (count == 0) { cerr << "\nERROR: Did not find sequence records in inputs" << endl; exit(1); }
}

// `mash screen -I`: every input arguments[1..] is a sample of its own, screened against the one table the job holds.  Per sample:
// stream the file, take the rows of the references it hit (mashgpu_screen_finish_hits) and print them after a column naming the
// sample, then reset the job for the next one.  A sample without records gets a warning and no rows.
void screenSamples(mashgpu_screen_job *job, const vector<string> &arguments, const Sketch &sketch, int kmerSize, bool trans,
                   double identityMin, double pValueMax)
{
    for (size_t f = 2; f < arguments.size(); f++)
        if (arguments[f] == "-") { cerr << "ERROR: '-' for stdin must be first query" << endl; exit(1); }
    const uint64_t n = sketch.getReferenceCount();
    vector<uint32_t> ref(n); vector<uint64_t> shared(n), median(n); vector<double> identity(n), pValue(n);
    for (size_t f = 1; f < arguments.size(); f++) {
        const string &sample = arguments[f];
        cerr << (trans ? "Translating from " : "Streaming from ") << sample << "..." << endl;
        if (feedInputs(job, vector<string>(1, sample), kmerSize) == 0) {
            cerr << "WARNING: Did not find sequence records in " << sample << endl;
            if (mashgpu_screen_reset(job) != MASHGPU_OK) gpuFail();
            continue;
        }
        uint64_t rows = 0, setSize = 0;
        if (mashgpu_screen_finish_hits(job, ref.data(), shared.data(), median.data(), identity.data(), pValue.data(), &rows, &setSize) != MASHGPU_OK)
            gpuFail();
        cerr << "   Estimated distinct" << (trans ? " (translated)" : "") << " k-mers in " << sample << ": " << setSize << endl;
        if (setSize == 0) cerr << "WARNING: no valid k-mers in " << sample << "." << endl;
        // rows of every reference under -i < 0; the ones the sample did not hit take the values of a reference with shared 0
        uint64_t row = 0;
        for (uint64_t i = 0; i < n; i++) {                   // reference CommandScreen.cpp:418-455
            const bool hit = row < rows && ref[row] == i;
            if (!hit && identityMin >= 0.0) continue;
            const size_t size = sketch.getReference(i).hashesSorted.size();
            const uint64_t sh = hit ? shared[row] : 0, med = hit ? median[row] : 0;
            const double id = hit ? identity[row] : (size == 0 ? 1. : 0.), pv = hit ? pValue[row] : 1.0;
            if (hit) row++;
            if (id < identityMin) continue;
            if (pv > pValueMax) continue;
            cout << sample << '\t' << id << '\t' << sh << '/' << size << '\t' << med << '\t' << pv
                 << '\t' << sketch.getReference(i).name << '\t' << sketch.getReference(i).comment << endl;
        }
        if (mashgpu_screen_reset(job) != MASHGPU_OK) gpuFail();
    }
}

int runScreen(int argc, const char **argv)
{
    Command c;
    c.add("help", Option(Option::Boolean, "h", ""));
    c.add("threads", Option(Option::Integer, "p", "1"));
    c.add("winning!", Option(Option::Boolean, "w", ""));
    c.add("identity", Option(Option::Number, "i", "0", -1., 1.));
    c.add("pvalue", Option(Option::Number, "v", "1.0", 0., 1.));
    c.add("samples", Option(Option::Boolean, "I", ""));     // not an option of the reference: its users run one screen per sample
    if (c.parse(argc, argv)) return 1;
    if (c.arguments.size() < 2 || c.opt("help").active) {
        cerr << "usage: mash screen [options] <queries>.msh <mixture> [<mixture>] ...\n"
                "       mash screen -I [options] <queries>.msh <sample> [<sample>] ...   (each sample screened on its own; rows prefixed by the sample)" << endl;
        return 0;
    }
    if (!hasSuffix(c.arguments[0], suffixSketch)) {
        cerr << "ERROR: " << c.arguments[0] << " does not look like a sketch (.msh)" << endl;
        exit(1);
    }
    double pValueMax = c.opt("pvalue").number, identityMin = c.opt("identity").number;
    Sketch sketch;
    Sketch::Parameters parameters;
    vector<string> refArgVector(1, c.arguments[0]);
    sketch.initFromFiles(refArgVector, parameters);
    parameters = sketch.getParameters();
    string alphabet;
    sketch.getAlphabetAsString(alphabet);
    const bool trans = alphabet == alphabetProtein;          // CommandScreen.cpp:120: the library translates the mixture in six frames
    cerr << "Loading " << c.arguments[0] << "..." << endl;
    mashgpu_sketch_params p;
    fillGpuParams(p, parameters);
    mashgpu_sketch_set set;
    vector<uint64_t> h, l; vector<uint32_t> nn;
    sketch.toSketchSet(set, h, nn, l);
    mashgpu_screen_job *job = 0;
    if (mashgpu_screen_open(gpuContext(), &p, &set, &job) != MASHGPU_OK) gpuFail();
    if (c.opt("winning!").active && mashgpu_screen_set_winner(job, 1) != MASHGPU_OK) gpuFail();     // -w, CommandScreen.cpp:357-407
    if (c.opt("samples").active) {
        screenSamples(job, c.arguments, sketch, parameters.kmerSize, trans, identityMin, pValueMax);
        mashgpu_screen_close(job);
        return 0;
    }
    streamInputs(job, c.arguments, parameters.kmerSize, trans);
    const uint64_t n = sketch.getReferenceCount();
    vector<uint64_t> shared(n), median(n); vector<double> identity(n), pValue(n);
    uint64_t setSize = 0;
    if (mashgpu_screen_finish(job, shared.data(), median.data(), identity.data(), pValue.data(), &setSize, 0, 0) != MASHGPU_OK) gpuFail();
    mashgpu_screen_close(job);
    cerr << "   Estimated distinct" << (trans ? " (translated)" : "") << " k-mers in mixture: " << setSize << endl;
    if (setSize == 0) cerr << "WARNING: no valid k-mers in input." << endl;
    cerr << "Summing shared..." << endl << "Computing coverage medians..." << endl << "Writing output..." << endl;
    for (uint64_t i = 0; i < n; i++) {                       // reference CommandScreen.cpp:418-455
        if (shared[i] != 0 || identityMin < 0.0) {
            if (identity[i] < identityMin) continue;
            if (pValue[i] > pValueMax) continue;
            cout << identity[i] << '\t' << shared[i] << '/' << sketch.getReference(i).hashesSorted.size() << '\t' << median[i] << '\t' << pValue[i]
                 << '\t' << sketch.getReference(i).name << '\t' << sketch.getReference(i).comment << endl;
        }
    }
    return 0;
}

// ---------------------------------------------------------------------------------------------------- taxscreen
// reference CommandTaxScreen.cpp:57-480: the screen stream, then the LCA taxon of every distinct reference hash, per-taxon
// counts and their roll-up on the GPU (mashgpu_screen_taxonomy), and the Kraken-style report (taxdb.hpp)
int runTaxScreen(int argc, const char **argv)
{
    Command c;
    c.add("help", Option(Option::Boolean, "h", ""));
    c.add("threads", Option(Option::Integer, "p", "1"));
    c.add("identity", Option(Option::Number, "i", "0", -1., 1.));      // parsed and unused, as in the reference
    c.add("pvalue", Option(Option::Number, "v", "1.0", 0., 1.));
    c.add("mapping-file", Option(Option::String, "m", ""));
    c.add("taxonomy-dir", Option(Option::String, "t", "."));
    if (c.parse(argc, argv)) return 1;
    if (c.arguments.size() < 2 || c.opt("help").active) { cerr << "usage: mash taxscreen [options] <queries>.msh <pool> [<pool>] ..." << endl; return 0; }
    if (!hasSuffix(c.arguments[0], suffixSketch)) {
        cerr << "ERROR: " << c.arguments[0] << " does not look like a sketch (.msh)" << endl;
        exit(1);
    }
    const string taxonomyDir = c.opt("taxonomy-dir").argument, mappingFileName = c.opt("mapping-file").argument;
    Sketch sketch;
    Sketch::Parameters parameters;
    vector<string> refArgVector(1, c.arguments[0]);
    sketch.initFromFiles(refArgVector, parameters);
    parameters = sketch.getParameters();
    string alphabet;
    sketch.getAlphabetAsString(alphabet);
    const bool trans = alphabet == alphabetProtein;
    const string namesDumpFile = taxonomyDir + "/names.dmp", nodesDumpFile = taxonomyDir + "/nodes.dmp";
    if (!ifstream(namesDumpFile).good() || !ifstream(nodesDumpFile).good()) {
        cerr << "Could not find a file names.dmp or nodes.dmp in directory " << taxonomyDir << "\n"
             << " To download the required taxonomy files into the current directory, use the following commands:\n"
             << "   wget ftp://ftp.ncbi.nih.gov/pub/taxonomy/taxdump.tar.gz\n"
             << "   tar xvvf taxdump.tar.gz\n"
             << endl;
        exit(1);
    }
    cerr << "Loading taxonomy files ..." << endl;
    mashhost::TaxTree tax;
    tax.load(namesDumpFile, nodesDumpFile, cerr);
    cerr << "Reading mapping file ..." << endl;
    const uint64_t n = sketch.getReferenceCount();
    vector<uint64_t> referenceTaxIDs(n, 0);
    if (mappingFileName != "") {                 // lines "taxID<one byte>reference name"; the first line of a name wins
        string text;
        if (!mashhost::readFile(mappingFileName, text)) throw std::runtime_error("unable to open mapping file");
        mashhost::IStream in(text.data(), text.data() + text.size());
        unordered_map<string, uint64_t> refTaxMap;
        uint64_t taxID = 0;
        string referenceID;
        while (in.num(taxID)) {
            in.ignore(1);
            in.getline(referenceID, '\n');
            refTaxMap.emplace(referenceID, taxID);
        }
        for (uint64_t i = 0; i < n; i++) {
            auto it = refTaxMap.find(sketch.getReference(i).name);
            if (it != refTaxMap.end()) referenceTaxIDs[i] = it->second;
        }
    }
    for (uint64_t i = 0; i < n; i++) {          // otherwise the number after the word "taxid" in the comment (the last one)
        uint64_t taxID = referenceTaxIDs[i];
        if (taxID == 0) {
            const string &comment = sketch.getReference(i).comment;
            mashhost::IStream in(comment.data(), comment.data() + comment.size());
            string word;
            while (in.word(word))
                if (word == "taxid") in.num(taxID);
        }
        if (taxID == 0) cerr << "Could not find taxID for reference " << sketch.getReference(i).name << " in comment field or mapping file!" << endl;
        else referenceTaxIDs[i] = taxID;
    }
    cerr << "Loading " << c.arguments[0] << "..." << endl;
    mashgpu_sketch_params p;
    fillGpuParams(p, parameters);
    mashgpu_sketch_set set;
    vector<uint64_t> h, l; vector<uint32_t> nn;
    sketch.toSketchSet(set, h, nn, l);
    mashgpu_screen_job *job = 0;
    if (mashgpu_screen_open(gpuContext(), &p, &set, &job) != MASHGPU_OK) gpuFail();
    uint32_t *dCounters = 0;
    uint64_t nDistinct = 0;
    if (mashgpu_screen_counters(job, &dCounters, &nDistinct) != MASHGPU_OK) gpuFail();
    cerr << "   " << nDistinct << " distinct hashes." << endl;
    streamInputs(job, c.arguments, parameters.kmerSize, trans);
    uint64_t setSize = 0;
    if (mashgpu_screen_finish(job, 0, 0, 0, 0, &setSize, 0, 0) != MASHGPU_OK) gpuFail();
    cerr << "   Estimated distinct" << (trans ? " (translated)" : "") << " k-mers in pool: " << setSize << endl;
    if (setSize == 0) cerr << "WARNING: no valid k-mers in input." << endl;
    cerr << "Assigning LCA taxIDs to hashes ..." << endl;
    // sketch codes: taxonomy node, or a slot per distinct taxID outside the taxonomy (ascending), or none for taxID 0
    vector<uint64_t> unknown;
    for (uint64_t t : referenceTaxIDs)
        if (t != 0 && tax.find(t) < 0) unknown.push_back(t);
    sort(unknown.begin(), unknown.end());
    unknown.erase(unique(unknown.begin(), unknown.end()), unknown.end());
    vector<uint32_t> code(n);
    for (uint64_t i = 0; i < n; i++) {
        const uint64_t t = referenceTaxIDs[i];
        const int64_t node = tax.find(t);
        if (t == 0) code[i] = MASHGPU_TAX_NONE;
        else if (node >= 0) code[i] = (uint32_t)node;
        else code[i] = (uint32_t)(tax.taxid.size() + (lower_bound(unknown.begin(), unknown.end(), t) - unknown.begin()));
    }
    mashgpu_taxonomy *gtax = 0;
    if (mashgpu_taxonomy_open(gpuContext(), tax.taxid.size(), tax.parent.data(), tax.taxid.data(), &gtax) != MASHGPU_OK) gpuFail();
    vector<mashgpu_tax_row> rows(tax.taxid.size() + unknown.size() + 2);
    vector<uint8_t> unknownInLca(unknown.size());
    uint64_t nRows = 0, totalCount = 0, totalHashCount = 0;
    if (mashgpu_screen_taxonomy(job, gtax, code.data(), (uint32_t)unknown.size(), unknown.data(), rows.data(), rows.size(), &nRows,
                                &totalCount, &totalHashCount, 0, unknownInLca.data()) != MASHGPU_OK) gpuFail();
    rows.resize(nRows);
    mashgpu_taxonomy_close(gtax);
    mashgpu_screen_close(job);
    // the reference prints this once per LCA call that meets the taxID (taxdb.hpp:166, 172), a number that depends on hash-set
    // order; here once per taxID that met another sketch's taxID in a fold
    for (size_t u = 0; u < unknown.size(); u++)
        if (unknownInLca[u]) cerr << "TaxID " << unknown[u] << " not in database - ignoring it.\n";
    vector<uint64_t> outside;                    // the roll-up's getEntry of a taxon outside the taxonomy (taxdb.hpp:74-82), ascending
    for (const auto &r : rows)
        if (tax.find(r.taxid) < 0) outside.push_back(r.taxid);
    sort(outside.begin(), outside.end());
    for (uint64_t t : outside) cerr << "Couldn't find tax entry with taxID " << t << endl;
    cerr << "Writing output..." << endl;
    mashhost::writeTaxReport(stdout, tax, rows, totalCount);
    return 0;
}

// test helpers of the taxonomy reader and the report writer (no GPU):
//   mash tax-dump <dir>              every node: taxid, parent taxid (itself for a root), rank, name, tab-separated, ascending taxid
//   mash tax-report <dir> <rows>     the report of the rows "taxid taxCount taxHashCount cladeCount cladeHashCount" (one per
//                                    line, first line "totalCount totalHashCount")
int runTaxDump(int argc, const char **argv)
{
    if (argc < 1) { cerr << "usage: mash tax-dump <taxonomy dir>" << endl; return 1; }
    mashhost::TaxTree tax;
    tax.load(string(argv[0]) + "/names.dmp", string(argv[0]) + "/nodes.dmp", cerr);
    vector<uint32_t> order(tax.taxid.size());
    for (uint32_t i = 0; i < order.size(); i++) order[i] = i;
    sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return tax.taxid[a] < tax.taxid[b]; });
    for (uint32_t i : order)
        cout << tax.taxid[i] << '\t' << tax.taxid[tax.parent[i]] << '\t' << tax.rank[i] << '\t' << tax.name[i] << '\n';
    return 0;
}

int runTaxReport(int argc, const char **argv)
{
    if (argc < 2) { cerr << "usage: mash tax-report <taxonomy dir> <rows>" << endl; return 1; }
    mashhost::TaxTree tax;
    tax.load(string(argv[0]) + "/names.dmp", string(argv[0]) + "/nodes.dmp", cerr);
    ifstream in(argv[1]);
    uint64_t totalCount = 0, totalHashCount = 0;
    in >> totalCount >> totalHashCount;
    vector<mashgpu_tax_row> rows;
    mashgpu_tax_row r;
    while (in >> r.taxid >> r.tax_count >> r.tax_hash_count >> r.clade_count >> r.clade_hash_count) rows.push_back(r);
    mashhost::writeTaxReport(stdout, tax, rows, totalCount);
    return 0;
}

// ---------------------------------------------------------------------------------------------------- info
int runInfo(int argc, const char **argv)
{
    Command c;
    c.add("help", Option(Option::Boolean, "h", ""));
    c.add("header", Option(Option::Boolean, "H", ""));
    c.add("tabular", Option(Option::Boolean, "t", ""));
    c.add("counts", Option(Option::Boolean, "c", ""));
    c.add("dump", Option(Option::Boolean, "d", ""));
    if (c.parse(argc, argv)) return 1;
    if (c.arguments.size() == 0 || c.opt("help").active) { cerr << "usage: mash info [options] <sketch>" << endl; return 0; }
    const string &file = c.arguments[0];
    if (!hasSuffix(file, suffixSketch)) { cerr << "ERROR: The file \"" << file << "\" does not look like a sketch." << endl; return 1; }
    Sketch sketch;
    Sketch::Parameters params;
    uint64_t referenceCount = sketch.initParametersFromCapnp(file.c_str());
    params = sketch.getParameters();
    if (c.opt("header").active) {
        string alphabet;
        sketch.getAlphabetAsString(alphabet);
        cout << "Header:" << endl;
        cout << "  Hash function (seed):          " << "MurmurHash3_x64_128" << " (" << sketch.getHashSeed() << ")" << endl;
        cout << "  K-mer size:                    " << sketch.getKmerSize() << " (" << (sketch.getUse64() ? "64" : "32") << "-bit hashes)" << endl;
        cout << "  Alphabet:                      " << alphabet << (sketch.getNoncanonical() ? "" : " (canonical)") << (sketch.getPreserveCase() ? " (case-sensitive)" : "") << endl;
        cout << "  Target min-hashes per sketch:  " << sketch.getMinHashesPerWindow() << endl;
        cout << "  Sketches:                      " << referenceCount << endl;
        return 0;
    }
    vector<string> files(1, file);
    sketch.initFromFiles(files, params);
    if (c.opt("dump").active) {                              // writeJson, reference CommandInfo.cpp:222-299
        string alphabet;
        sketch.getAlphabetAsString(alphabet);
        bool use64 = sketch.getUse64();
        cout << "{" << endl;
        cout << "	\"kmer\" : " << sketch.getKmerSize() << ',' << endl;
        cout << "	\"alphabet\" : \"" << alphabet << "\"," << endl;
        cout << "	\"preserveCase\" : " << (sketch.getPreserveCase() ? "true" : "false") << ',' << endl;
        cout << "	\"canonical\" : " << (sketch.getNoncanonical() ? "false" : "true") << ',' << endl;
        cout << "	\"sketchSize\" : " << sketch.getMinHashesPerWindow() << ',' << endl;
        cout << "	\"hashType\" : \"" << "MurmurHash3_x64_128" << "\"," << endl;
        cout << "	\"hashBits\" : " << (use64 ? 64 : 32) << ',' << endl;
        cout << "	\"hashSeed\" : " << sketch.getHashSeed() << ',' << endl;
        cout << " 	\"sketches\" :" << endl;
        cout << "	[" << endl;
        for (uint64_t i = 0; i < sketch.getReferenceCount(); i++) {
            const Sketch::Reference &ref = sketch.getReference(i);
            cout << "		{" << endl;
            cout << "			\"name\" : \"" << ref.name << "\"," << endl;
            cout << "			\"length\" : " << ref.length << ',' << endl;
            cout << "			\"comment\" : \"" << ref.comment << "\"," << endl;
            cout << "			\"hashes\" :" << endl;
            cout << "			[" << endl;
            for (int j = 0; j < ref.hashesSorted.size(); j++) {
                cout << "				" << (use64 ? ref.hashesSorted.at(j).hash64 : ref.hashesSorted.at(j).hash32);
                if (j < ref.hashesSorted.size() - 1) cout << ',';
                cout << endl;
            }
            cout << "			]" << endl;
            if (ref.countsSorted) {
                cout << "			\"counts\" :" << endl;
                cout << "			[" << endl;
                for (int j = 0; j < (int)ref.counts.size(); j++) {
                    cout << "				" << ref.counts.at(j);
                    if (j < ref.hashesSorted.size() - 1) cout << ',';
                    cout << endl;
                }
                cout << "			]" << endl;
            }
            cout << (i < sketch.getReferenceCount() - 1 ? "		}," : "		}") << endl;
        }
        cout << "	]" << endl;
        cout << "}" << endl;
        return 0;
    }
    // default / -t: one line per sketch: hashes, length, name, comment (reference CommandInfo.cpp:139-183, tabular form)
    if (!c.opt("tabular").active) cout << "#Hashes\tLength\tID\tComment" << endl;
    for (uint64_t i = 0; i < sketch.getReferenceCount(); i++) {
        const Sketch::Reference &ref = sketch.getReference(i);
        cout << ref.hashesSorted.size() << '\t' << ref.length << '\t' << ref.name << '\t' << ref.comment << endl;
    }
    return 0;
}

// ---------------------------------------------------------------------------------------------------- paste
// reference CommandPaste.cpp:30-88: concatenate sketch files with matching parameters into <out_prefix>.msh
int runPaste(int argc, const char **argv)
{
    Command c;
    c.add("help", Option(Option::Boolean, "h", ""));
    c.add("list", Option(Option::Boolean, "l", ""));
    if (c.parse(argc, argv)) return 1;
    if (c.arguments.size() < 2 || c.opt("help").active) { cerr << "usage: mash paste <out_prefix> <sketch> [<sketch>] ..." << endl; return 0; }
    vector<string> files;
    for (size_t i = 1; i < c.arguments.size(); i++) { if (c.opt("list").active) splitFile(c.arguments[i], files); else files.push_back(c.arguments[i]); }
    for (auto &f : files)
        if (!hasSuffix(f, suffixSketch)) { cerr << "ERROR: The file \"" << f << "\" does not look like a sketch." << endl; return 1; }
    Sketch sketch;
    Sketch::Parameters parameters;
    sketch.initFromFiles(files, parameters);
    string out = c.arguments[0];
    if (!hasSuffix(out, suffixSketch)) out += suffixSketch;
    cerr << "Writing " << out << "..." << endl;
    sketch.writeToCapnp(out.c_str());
    return 0;
}

// test helper: rebuild a .msh from a `mash info -d` JSON dump (the reference's golden files are such dumps)
int runImportJson(int argc, const char **argv)
{
    if (argc < 2) { cerr << "usage: mash import-json <dump.json> <out.msh>" << endl; return 1; }
    ifstream in(argv[0]);
    if (!in) { cerr << "ERROR: could not open " << argv[0] << endl; return 1; }
    string text((istreambuf_iterator<char>(in)), istreambuf_iterator<char>());
    auto scalar = [&](const string &key, size_t from = 0) -> string {
        size_t p = text.find("\"" + key + "\" :", from);
        if (p == string::npos) return "";
        p = text.find(':', p) + 1;
        size_t e = text.find('\n', p);
        string v = text.substr(p, e - p);
        while (!v.empty() && (v.back() == ',' || isspace((unsigned char)v.back()))) v.pop_back();
        size_t b = 0;
        while (b < v.size() && isspace((unsigned char)v[b])) b++;
        v = v.substr(b);
        if (v.size() >= 2 && v.front() == '"' && v.back() == '"') v = v.substr(1, v.size() - 2);
        return v;
    };
    Sketch::Parameters parameters;
    parameters.kmerSize = atoi(scalar("kmer").c_str());
    parameters.preserveCase = scalar("preserveCase") == "true";
    parameters.noncanonical = scalar("canonical") == "false";
    parameters.minHashesPerWindow = strtoull(scalar("sketchSize").c_str(), 0, 10);
    parameters.seed = (uint32_t)strtoul(scalar("hashSeed").c_str(), 0, 10);
    parameters.concatenated = true;
    setAlphabetFromString(parameters, scalar("alphabet").c_str());
    Sketch sketch;
    sketch.setParameters(parameters);
    size_t pos = text.find("\"sketches\"");
    while ((pos = text.find("\"name\" :", pos)) != string::npos) {
        Sketch::Reference ref;
        ref.name = scalar("name", pos);
        ref.length = strtoull(scalar("length", pos).c_str(), 0, 10);
        ref.comment = scalar("comment", pos);
        ref.hashesSorted.setUse64(parameters.use64);
        size_t a = text.find('[', text.find("\"hashes\"", pos)), e = text.find(']', a);
        const char *q = text.c_str() + a + 1, *end = text.c_str() + e;
        while (q < end) {
            while (q < end && !isdigit((unsigned char)*q)) q++;
            if (q >= end) break;
            char *next;
            uint64_t h = strtoull(q, &next, 10);
            ref.hashesSorted.push_back64(h);
            q = next;
        }
        sketch.addReference(ref);
        pos = e;
    }
    sketch.writeToCapnp(argv[1]);
    return 0;
}

}  // namespace

static int runCommand(int argc, const char **argv)
{
    string cmd = argv[1];
    if (cmd == "sketch") return runSketch(argc - 2, argv + 2);
    if (cmd == "dist") return runDist(argc - 2, argv + 2);
    if (cmd == "triangle") return runTriangle(argc - 2, argv + 2);
    if (cmd == "within") return runWithin(argc - 2, argv + 2);
    if (cmd == "screen") return runScreen(argc - 2, argv + 2);
    if (cmd == "taxscreen") return runTaxScreen(argc - 2, argv + 2);
    if (cmd == "tax-dump") return runTaxDump(argc - 2, argv + 2);
    if (cmd == "tax-report") return runTaxReport(argc - 2, argv + 2);
    if (cmd == "info") return runInfo(argc - 2, argv + 2);
    if (cmd == "paste") return runPaste(argc - 2, argv + 2);
    if (cmd == "import-json") return runImportJson(argc - 2, argv + 2);
    cerr << "ERROR: Unrecognized command: " << cmd << endl;
    return 1;
}

int main(int argc, const char **argv)
{
    if (argc < 2) {
        cerr << "usage: mash <sketch|dist|triangle|within|screen|taxscreen|info|paste> ...   (H100 engine; see INTEGRATION.md)" << endl;
        return 0;
    }
    const int rc = runCommand(argc, argv);
    // Everything the command wrote is closed or flushed here; leave without the static destructors and the CUDA runtime's
    // teardown (unmapping gigabytes of device and pinned memory one allocation at a time): the driver reclaims it all at once.
    cout.flush(); cerr.flush();
    fflush(stdout); fflush(stderr);
    _exit(rc);
}
