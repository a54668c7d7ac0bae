// Sketch.cpp -- host shim: the reference's Sketch surface on top of libmashgpu (see Sketch.h).
// Follows reference src/mash/Sketch.cpp for orchestration, messages and the .msh layout; all hashing / bottom-s
// work is delegated to mashgpu_sketch_batch (one call per batch of units instead of one ThreadPool job per unit).
#include "Sketch.h"

#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

#include <cmath>
#include <cstdlib>
#include <fstream>
#include <iostream>
#include <chrono>
#include <condition_variable>
#include <functional>
#include <list>
#include <mutex>
#include <thread>

#include "capnp_lite.hpp"
#include "fastx.hpp"

using namespace std;

namespace mash {

static double nowMs() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); }
static bool traceOn() { static const bool on = getenv("MASHGPU_TRACE") != 0; return on; }

// One engine context per process.  Creating it (CUDA context, streams, pinned staging) takes ~0.4 s, as long as parsing 2 GB of
// FASTA: gpuContextBegin() starts that work on a helper thread so that the parser threads fill the first batch meanwhile;
// gpuContext() waits for it (or does the work itself when nobody began).
static mashgpu_ctx *gpuCtx = 0;
static std::once_flag gpuCtxOnce;
static std::mutex gpuCtxMutex;
static std::condition_variable gpuCtxReady;
static bool gpuCtxDone = false;

static std::string gpuCtxError;

static void gpuContextCreate()
{
    const double t0 = nowMs();
    const char *dev = getenv("MASH_GPU_DEVICE");
    if (mashgpu_create(dev ? atoi(dev) : 0, &gpuCtx) != MASHGPU_OK) {
        gpuCtx = 0;
        gpuCtxError = mashgpu_last_error(0);        // reported by gpuContext() on the main thread: no exit() from the helper thread
    } else if (traceOn()) cerr << "[mash] GPU context: " << nowMs() - t0 << " ms" << endl;
    { std::lock_guard<std::mutex> lock(gpuCtxMutex); gpuCtxDone = true; }
    gpuCtxReady.notify_all();
}

void gpuContextBegin()
{
    std::call_once(gpuCtxOnce, [] { std::thread(gpuContextCreate).detach(); });     // detached: an exit(1) elsewhere must not find a joinable thread
}

mashgpu_ctx *gpuContext()
{
    std::call_once(gpuCtxOnce, gpuContextCreate);
    std::unique_lock<std::mutex> lock(gpuCtxMutex);
    gpuCtxReady.wait(lock, [] { return gpuCtxDone; });
    if (!gpuCtx) {      // no CPU path: without the engine there is nothing to fall back to
        cerr << "ERROR: " << gpuCtxError << endl;
        exit(1);
    }
    return gpuCtx;
}

void fillGpuParams(mashgpu_sketch_params &p, const Sketch::Parameters &parameters)
{
    memset(&p, 0, sizeof(p));
    p.kmer_size = parameters.kmerSize;
    p.sketch_size = (uint32_t)parameters.minHashesPerWindow;
    p.seed = parameters.seed;
    p.use64 = parameters.use64;
    p.noncanonical = parameters.noncanonical;
    p.preserve_case = parameters.preserveCase;
    for (int i = 0; i < 256; i++) p.alphabet[i] = parameters.alphabet[i];
    p.min_copies = parameters.reads ? parameters.minCov : 1;      // reference Sketch.cpp:1186: MinHashHeap(use64, s, reads ? minCov : 1, ...)
    p.target_cov = parameters.reads ? parameters.targetCov : 0;   // reference Sketch.cpp:1258
    p.bloom_bytes = parameters.reads ? parameters.memoryBound : 0; // reference Sketch.cpp:1186 (-b)
}

bool hasSuffix(string const &whole, string const &suffix)   // reference Sketch.cpp:897-905
{
    if (whole.length() >= suffix.length()) return 0 == whole.compare(whole.length() - suffix.length(), suffix.length(), suffix);
    return false;
}

void setAlphabetFromString(Sketch::Parameters &parameters, const char *characters)   // reference Sketch.cpp:1108-1137
{
    parameters.alphabetSize = 0;
    memset(parameters.alphabet, 0, 256);
    for (const char *c = characters; *c != 0; c++) {
        char upper = *c;
        if (!parameters.preserveCase && upper > 96 && upper < 123) upper -= 32;
        parameters.alphabet[(unsigned char)upper] = true;
    }
    for (int i = 0; i < 256; i++)
        if (parameters.alphabet[i]) parameters.alphabetSize++;
    parameters.use64 = pow(parameters.alphabetSize, parameters.kmerSize) > pow(2, 32);
}

void Sketch::getAlphabetAsString(string &alphabet) const
{
    for (int i = 0; i < 256; i++)
        if (parameters.alphabet[i]) alphabet.append(1, i);
}

int Sketch::getMinKmerSize(uint64_t reference) const
{
    return ceil(log(references[reference].length * (1 - parameters.warning) / parameters.warning) / log(parameters.alphabetSize));
}

double Sketch::getRandomKmerChance(uint64_t reference) const
{
    return 1. / (kmerSpace / references[reference].length + 1.);
}

void Sketch::getReferenceHistogram(uint64_t index, map<uint32_t, uint64_t> &histogram) const
{
    const Reference &reference = references.at(index);
    histogram.clear();
    for (uint64_t i = 0; i < reference.counts.size(); i++) histogram[reference.counts.at(i)]++;
}

uint64_t Sketch::getReferenceIndex(string id) const
{
    auto it = referenceIndecesById.find(id);
    return it == referenceIndecesById.end() ? (uint64_t)-1 : (uint64_t)it->second;
}

void Sketch::createIndex()   // reference Sketch.cpp:492-510 (non-windowed part)
{
    for (size_t i = 0; i < references.size(); i++) referenceIndecesById[references[i].name] = (int)i;
    kmerSpace = pow(parameters.alphabetSize, parameters.kmerSize);
}

// --------------------------------------------------------------------------------------------------------------
// batched GPU sketching
// --------------------------------------------------------------------------------------------------------------
struct Sketch::Batch {
    vector<mashhost::SeqBuffer> seqs;   // records (pool storage: returned for reuse when the batch is dropped)
    vector<uint32_t> unitOfRecord;
    vector<Reference> refs;          // one per unit, name/comment filled at parse time
    uint64_t bytes = 0;
};

static const uint64_t batchBytesMax = 1ull << 28;

// A batch is handed to the GPU when it holds 256 MiB of sequence (one call then takes ~10 ms, and batch + parser look-ahead stay
// a few hundred MB of recycled buffers, seqbuf.hpp) or so many units that their sketches (units x s hashes on the
// host and on the device) reach 256 MiB -- `-i` on a multi-FASTA of millions of short records must not allocate by unit count
template <typename B>
static bool batchFull(const B &batch, const Sketch::Parameters &parameters)
{
    const uint64_t unitsMax = std::max<uint64_t>(1024, (1ull << 28) / (8 * std::max<uint64_t>(1, parameters.minHashesPerWindow)));
    return batch.bytes > batchBytesMax || batch.refs.size() >= unitsMax;
}

void Sketch::flushBatch(Batch &batch)
{
    const uint64_t units = batch.refs.size();
    if (units == 0) return;
    mashgpu_sketch_params p;
    fillGpuParams(p, parameters);
    const uint32_t s = p.sketch_size;
    vector<const char *> ptrs(batch.seqs.size());
    vector<uint64_t> lens(batch.seqs.size());
    for (size_t i = 0; i < batch.seqs.size(); i++) { ptrs[i] = batch.seqs[i].data(); lens[i] = batch.seqs[i].size(); }
    vector<uint64_t> hashes(units * s), lengths(units);
    vector<uint32_t> n(units), counts(parameters.counts ? units * s : 0);
    mashgpu_ctx *ctx = gpuContext();
    const double tFlush = nowMs();
    const int rc = mashgpu_sketch_batch(ctx, &p, ptrs.size(), ptrs.data(), lens.data(), batch.unitOfRecord.data(), units,
                                        hashes.data(), parameters.counts ? counts.data() : 0, n.data(), lengths.data());
    if (traceOn()) cerr << "[mash] sketch batch: " << units << " units, " << batch.bytes / 1e6 << " MB in " << nowMs() - tFlush << " ms" << endl;
    if (rc != MASHGPU_OK) {
        cerr << "ERROR: " << mashgpu_last_error(ctx) << endl;
        exit(1);
    }
    for (uint64_t u = 0; u < units; u++) {
        Reference &reference = batch.refs[u];
        reference.hashesSorted.setUse64(parameters.use64);     // == setMinHashesForReference, reference Sketch.cpp:1139-1145
        reference.hashesSorted.clear();
        for (uint32_t i = 0; i < n[u]; i++) reference.hashesSorted.push_back64(hashes[u * s + i]);
        if (parameters.counts) reference.counts.assign(counts.begin() + u * s, counts.begin() + u * s + n[u]);
        reference.countsSorted = true;
        reference.length = lengths[u];
    }
    references.insert(references.end(), batch.refs.begin(), batch.refs.end());   // == useThreadOutput, reference Sketch.cpp:372-377
    batch = Batch();
}

// A file-mode unit whose parsed sequence passes this many bytes is not held whole: the batch before it is flushed (input order) and
// the unit streams through a unit job (mashgpu_unit_*, DESIGN.md 2.7), 16 MiB of records at a time.  MASHGPU_CLI_STREAM_BYTES
// lowers it (tests).
static uint64_t unitStreamBytes()
{
    static const uint64_t v = getenv("MASHGPU_CLI_STREAM_BYTES") ? strtoull(getenv("MASHGPU_CLI_STREAM_BYTES"), 0, 10) : batchBytesMax;
    return v;
}

static void gpuCheck(mashgpu_ctx *ctx, int rc)
{
    if (rc != MASHGPU_OK) {
        cerr << "ERROR: " << mashgpu_last_error(ctx) << endl;
        exit(1);
    }
}

static mashgpu_unit_job *openUnitJob(const Sketch::Parameters &parameters)
{
    mashgpu_sketch_params p;
    fillGpuParams(p, parameters);
    mashgpu_ctx *ctx = gpuContext();
    mashgpu_unit_job *job = 0;
    gpuCheck(ctx, mashgpu_unit_open(ctx, &p, &job));
    return job;
}

static void feedUnitJob(mashgpu_unit_job *job, vector<mashhost::SeqBuffer> &seqs)
{
    vector<const char *> ptrs(seqs.size());
    vector<uint64_t> lens(seqs.size());
    for (size_t i = 0; i < seqs.size(); i++) { ptrs[i] = seqs[i].data(); lens[i] = seqs[i].size(); }
    gpuCheck(gpuContext(), mashgpu_unit_feed(job, seqs.size(), ptrs.data(), lens.data()));
    seqs.clear();
}

// Finish and close the job; the sketch goes into `reference` as flushBatch puts a unit's.  Returns the kept records' number.
static uint64_t finishUnitJob(mashgpu_unit_job *job, const Sketch::Parameters &parameters, Sketch::Reference &reference,
                              vector<uint64_t> &hashes, vector<uint32_t> &counts)
{
    const uint32_t s = (uint32_t)parameters.minHashesPerWindow;
    hashes.assign(s, 0);
    counts.assign(s, 0);
    uint32_t n = 0;
    uint64_t length = 0, records = 0;
    gpuCheck(gpuContext(), mashgpu_unit_finish(job, hashes.data(), counts.data(), &n, &length, &records));
    mashgpu_unit_close(job);
    hashes.resize(n);
    counts.resize(n);
    reference.hashesSorted.setUse64(parameters.use64);
    reference.hashesSorted.clear();
    for (uint32_t i = 0; i < n; i++) reference.hashesSorted.push_back64(hashes[i]);
    if (parameters.counts) reference.counts.assign(counts.begin(), counts.end());
    reference.countsSorted = true;
    reference.length = length;
    return records;
}

// One unit over all records of the listed files, round robin (sketchFile, reference Sketch.cpp:1147-1336).  With `drain` (reads
// mode) the records are handed over whenever `bytes` passes drainBytes and at the end; drain returns the number of records used
// once the sketch is complete (the -c stop), which ends the reading and is the count of the comment, as in the reference's loop.
typedef std::function<uint64_t(vector<mashhost::SeqBuffer> &, vector<uint32_t> &, uint64_t &)> DrainFn;
static const uint64_t drainBytes = 1ull << 24;

static void parseUnit(const vector<string> &fileNames, const Sketch::Parameters &parameters, Sketch::Reference &reference,
                      vector<mashhost::SeqBuffer> &seqs, vector<uint32_t> &unitOfRecord, uint32_t unit, uint64_t &bytes,
                      const DrainFn &drain = DrainFn())
{
    int count = 0;
    bool skipped = false;
    int l = 0;
    vector<gzFile> fps;
    list<mashhost::FastxReader *> readers;
    for (size_t f = 0; f < fileNames.size(); f++) {
        if (fileNames[f] == "-") {
            if (f > 1) { cerr << "ERROR: '-' for stdin must be first input" << endl; exit(1); }
        } else if (reference.name == "") {
            reference.name = fileNames[f];
        }
        gzFile fp = mashhost::FastxReader::openPath(fileNames[f]);
        if (fp == 0) { cerr << "ERROR: could not open " << fileNames[f] << endl; exit(1); }
        fps.push_back(fp);
        readers.push_back(new mashhost::FastxReader(fp));
        struct stat info;
        if (fileNames[f] != "-" && stat(fileNames[f].c_str(), &info) == 0) readers.back()->setSizeHint((size_t)info.st_size);
    }
    auto it = readers.begin();
    while (readers.begin() != readers.end()) {
        l = (*it)->read();
        if (l < -1) break;
        if (l == -1) {
            delete *it;
            it = readers.erase(it);
            if (it == readers.end()) it = readers.begin();
            continue;
        }
        if (l < parameters.kmerSize) { skipped = true; continue; }
        if (count == 0) {
            if (fileNames[0] == "-") {
                reference.name = (*it)->name;
                reference.comment = (*it)->comment;
            } else {
                reference.comment = (*it)->name;
                reference.comment.append(" ");
                reference.comment.append((*it)->comment);
            }
        }
        count++;
        bytes += (*it)->seq.size();
        seqs.push_back(std::move((*it)->seq));
        unitOfRecord.push_back(unit);
        it++;
        if (it == readers.end()) it = readers.begin();
        if (drain && bytes >= drainBytes) {
            if (const uint64_t used = drain(seqs, unitOfRecord, bytes)) { count = (int)used; l = -1; break; }
        }
    }
    if (drain && l == -1) {
        if (const uint64_t used = drain(seqs, unitOfRecord, bytes)) count = (int)used;
    }
    if (count > 1) {
        reference.comment.insert(0, " seqs] ");
        reference.comment.insert(0, to_string(count));
        reference.comment.insert(0, "[");
        reference.comment.append(" [...]");
    }
    if (l != -1) {
        cerr << "\nERROR: reading " << (fileNames.size() > 0 ? "input files" : fileNames[0]) << "." << endl;
        exit(1);
    }
    if (count == 0) {   // reference: reference.length == 0 (Sketch.cpp:1300-1312)
        if (skipped)
            cerr << "\nWARNING: All fasta records in " << (fileNames.size() > 0 ? "input files" : fileNames[0]) << " were shorter than the k-mer size (" << parameters.kmerSize << ")." << endl;
        else
            cerr << "\nERROR: Did not find fasta records in \"" << (fileNames.size() > 0 ? "input files" : fileNames[0]) << "\"." << endl;
        exit(1);
    }
    for (gzFile fp : fps) gzclose(fp);
}

void Sketch::initFromReads(const vector<string> &files, const Parameters &parametersNew)   // reference Sketch.cpp:96-103
{
    parameters = parametersNew;
    gpuContextBegin();
    // one sketch of all reads (sketchFile with parameters.reads, reference Sketch.cpp:1186-1282), streamed through a reads job: the
    // host holds one feed of records at a time and the device a fixed working set, whatever the size of the read set
    mashgpu_sketch_params p;
    fillGpuParams(p, parameters);
    mashgpu_ctx *ctx = gpuContext();
    mashgpu_reads_job *job = 0;
    auto check = [&](int rc) { gpuCheck(ctx, rc); };
    // without -m > 1, -c and -b the sketch does not depend on the order of the reads: the parallel unit job, not the heap's replay
    mashgpu_unit_job *unitJob = 0;
    if (p.min_copies <= 1 && !(p.target_cov > 0) && p.bloom_bytes == 0) unitJob = openUnitJob(parameters);
    else check(mashgpu_reads_open(ctx, &p, &job));
    bool stopped = false;
    DrainFn drain = [&](vector<mashhost::SeqBuffer> &seqs, vector<uint32_t> &unitOfRecord, uint64_t &bytes) -> uint64_t {
        if (unitJob) {
            feedUnitJob(unitJob, seqs);
            unitOfRecord.clear();
            bytes = 0;
            return 0;
        }
        if (!stopped && !seqs.empty()) {
            vector<const char *> ptrs(seqs.size());
            vector<uint64_t> lens(seqs.size());
            for (size_t i = 0; i < seqs.size(); i++) { ptrs[i] = seqs[i].data(); lens[i] = seqs[i].size(); }
            int st = 0;
            check(mashgpu_reads_feed(job, seqs.size(), ptrs.data(), lens.data(), &st));
            stopped = st != 0;
        }
        seqs.clear();
        unitOfRecord.clear();
        bytes = 0;
        if (!stopped) return 0;
        vector<uint64_t> hashes(p.sketch_size);                    // only the count of reads used is needed here
        vector<uint32_t> counts(p.sketch_size);
        uint32_t n = 0;
        uint64_t used = 0;
        check(mashgpu_reads_finish(job, hashes.data(), counts.data(), &n, &used));
        return used;
    };
    Reference reference;
    vector<mashhost::SeqBuffer> seqs;
    vector<uint32_t> unitOfRecord;
    uint64_t bytes = 0;
    parseUnit(files, parameters, reference, seqs, unitOfRecord, 0, bytes, drain);
    const uint32_t s = p.sketch_size;
    vector<uint64_t> hashes(s);
    vector<uint32_t> counts(s);
    uint32_t n = 0;
    uint64_t readsUsed = 0;
    if (unitJob) {
        readsUsed = finishUnitJob(unitJob, parameters, reference, hashes, counts);
        n = (uint32_t)hashes.size();
    } else {
        check(mashgpu_reads_finish(job, hashes.data(), counts.data(), &n, &readsUsed));
        mashgpu_reads_close(job);
        reference.hashesSorted.setUse64(parameters.use64);         // == setMinHashesForReference, reference Sketch.cpp:1139-1145
        reference.hashesSorted.clear();
        for (uint32_t i = 0; i < n; i++) reference.hashesSorted.push_back64(hashes[i]);
        if (parameters.counts) reference.counts.assign(counts.begin(), counts.begin() + n);
        reference.countsSorted = true;
    }
    // reference Sketch.cpp:1272-1282, 1319-1328; estimateSetSize = MinHashHeap.h:45
    const double setSize = n ? pow(2.0, parameters.use64 ? 64.0 : 32.0) * (double)n / (double)hashes[n - 1] : 0;
    reference.length = parameters.genomeSize != 0 ? parameters.genomeSize : (uint64_t)setSize;
    double multiplicity = 0;                                        // estimateMultiplicity, MinHashHeap.h:44
    if (n) {
        uint64_t sum = 0;
        for (uint32_t i = 0; i < n; i++) sum += counts[i];
        multiplicity = (double)sum / n;
    }
    cerr << "Estimated genome size: " << setSize << endl;
    cerr << "Estimated coverage:    " << multiplicity << endl;
    if (parameters.targetCov > 0) cerr << "Reads used:            " << readsUsed << endl;      // reference Sketch.cpp:1324-1327
    references.push_back(reference);
    createIndex();
}

int Sketch::initFromFiles(const vector<string> &files, const Parameters &parametersNew, int verbosity, bool enforceParameters, bool contain)
{
    parameters = parametersNew;
    Batch batch;
    for (const string &f : files)
        if (!hasSuffix(f, suffixSketch)) { gpuContextBegin(); break; }      // sequence input: the context comes up while the first files are parsed

    for (size_t i = 0; i < files.size(); i++) {
        bool isSketch = hasSuffix(files[i], suffixSketch);
        if (isSketch) {
            // header checks, reference Sketch.cpp:113-172
            Sketch sketchTest;
            sketchTest.initParametersFromCapnp(files[i].c_str());
            if (i == 0 && !enforceParameters) initParametersFromCapnp(files[i].c_str());
            string alphabet, alphabetTest;
            getAlphabetAsString(alphabet);
            sketchTest.getAlphabetAsString(alphabetTest);
            if (alphabet != alphabetTest) {
                cerr << "\nWARNING: The sketch file " << files[i] << " has different alphabet (" << alphabetTest << ") than the current alphabet (" << alphabet << "). This file will be skipped." << endl << endl;
                continue;
            }
            if (sketchTest.getHashSeed() != parameters.seed) {
                cerr << "\nWARNING: The sketch " << files[i] << " has a seed size (" << sketchTest.getHashSeed() << ") that does not match the current seed (" << parameters.seed << "). This file will be skipped." << endl << endl;
                continue;
            }
            if (sketchTest.getKmerSize() != parameters.kmerSize) {
                cerr << "\nWARNING: The sketch " << files[i] << " has a kmer size (" << sketchTest.getKmerSize() << ") that does not match the current kmer size (" << parameters.kmerSize << "). This file will be skipped." << endl << endl;
                continue;
            }
            if (!contain && sketchTest.getMinHashesPerWindow() < parameters.minHashesPerWindow) {
                cerr << "\nWARNING: The sketch file " << files[i] << " has a target sketch size (" << sketchTest.getMinHashesPerWindow() << ") that is smaller than the current sketch size (" << parameters.minHashesPerWindow << "). This file will be skipped." << endl << endl;
                continue;
            }
            if (sketchTest.getNoncanonical() != parameters.noncanonical) {
                cerr << "\nWARNING: The sketch file " << files[i] << " is " << (sketchTest.getNoncanonical() ? "noncanonical" : "canonical") << ", which is incompatible with the current setting. This file will be skipped." << endl << endl;
                continue;
            }
            if (sketchTest.getMinHashesPerWindow() > parameters.minHashesPerWindow)
                cerr << "\nWARNING: The sketch file " << files[i] << " has a target sketch size (" << sketchTest.getMinHashesPerWindow() << ") that is larger than the current sketch size (" << parameters.minHashesPerWindow << "). Its sketches will be reduced." << endl << endl;
            flushBatch(batch);           // keep input order (ThreadPool delivers outputs in submission order)
            loadCapnp(files[i].c_str());
        } else {
            if (verbosity > 0) {
                if (files[i] == "-") cerr << "Sketching from stdin..." << endl;
                else cerr << "Sketching " << files[i] << "..." << endl;
            }
            if (files[i] != "-") {
                FILE *test = fopen(files[i].c_str(), "r");
                if (test == NULL) { cerr << "ERROR: could not open " << files[i] << " for reading." << endl; exit(1); }
                fclose(test);
            }
            if (parameters.concatenated && parameters.parallelism > 1 && files[i] != "-") {
                // -p N: the reference parses N files at a time, one ThreadPool job each (Sketch.cpp:202-212), and takes the
                // outputs in submission order.  Here N parser threads work through the whole run of sequence files that starts
                // at files[i], a bounded number of files ahead of this thread, which appends the parsed files to the batch in
                // input order and hands full batches to the GPU -- the parse of the next files overlaps the sketching.
                size_t run = 1;
                while (i + run < files.size() && !hasSuffix(files[i + run], suffixSketch) && files[i + run] != "-") run++;
                for (size_t t = 1; t < run; t++) {
                    FILE *test = fopen(files[i + t].c_str(), "r");
                    if (test == NULL) { cerr << "ERROR: could not open " << files[i + t] << " for reading." << endl; exit(1); }
                    fclose(test);
                }
                // A file past unitStreamBytes() is not parsed whole: its worker hands each 16 MiB of records to this thread, which
                // feeds them to a unit job once the file's turn has come (the GPU context stays on this thread), and waits until
                // they are taken.
                struct Parsed {
                    Reference ref; vector<mashhost::SeqBuffer> seqs; vector<uint32_t> unitOfRecord; uint64_t bytes = 0; bool ready = false;
                    bool streaming = false, chunkReady = false; vector<mashhost::SeqBuffer> chunk;
                };
                vector<Parsed> parsed(run);
                std::mutex mu;
                std::condition_variable cvReady, cvRoom, cvTaken;
                size_t nextFile = 0, consumed = 0;
                const size_t window = 2 * (size_t)parameters.parallelism;      // files parsed ahead of the consumer
                const size_t nWorkers = std::min<size_t>((size_t)parameters.parallelism, run);
                vector<std::thread> workers;
                for (size_t w = 0; w < nWorkers; w++)
                    workers.emplace_back([&]() {
                        for (;;) {
                            size_t t;
                            {
                                std::unique_lock<std::mutex> lock(mu);
                                if (nextFile >= run) return;
                                t = nextFile++;
                                cvRoom.wait(lock, [&] { return t < consumed + window; });
                            }
                            vector<string> file(1, files[i + t]);
                            DrainFn drain = [&, t](vector<mashhost::SeqBuffer> &s, vector<uint32_t> &u, uint64_t &b) -> uint64_t {
                                if (!parsed[t].streaming && b < unitStreamBytes()) return 0;
                                std::unique_lock<std::mutex> lock(mu);
                                parsed[t].streaming = true;
                                parsed[t].chunk = std::move(s);
                                parsed[t].chunkReady = true;
                                cvReady.notify_all();
                                cvTaken.wait(lock, [&] { return !parsed[t].chunkReady; });
                                s.clear();
                                u.clear();
                                b = 0;
                                return 0;
                            };
                            parseUnit(file, parameters, parsed[t].ref, parsed[t].seqs, parsed[t].unitOfRecord, 0, parsed[t].bytes, drain);
                            { std::lock_guard<std::mutex> lock(mu); parsed[t].ready = true; }
                            cvReady.notify_all();
                        }
                    });
                for (size_t t = 0; t < run; t++) {
                    if (t > 0 && verbosity > 0) cerr << "Sketching " << files[i + t] << "..." << endl;
                    mashgpu_unit_job *job = 0;
                    for (;;) {
                        vector<mashhost::SeqBuffer> chunk;
                        {
                            std::unique_lock<std::mutex> lock(mu);
                            cvReady.wait(lock, [&] { return parsed[t].ready || parsed[t].chunkReady; });
                            if (!parsed[t].chunkReady) break;
                            chunk = std::move(parsed[t].chunk);
                            parsed[t].chunk.clear();
                            parsed[t].chunkReady = false;
                        }
                        cvTaken.notify_all();
                        if (!job) {
                            flushBatch(batch);           // keep input order
                            job = openUnitJob(parameters);
                        }
                        feedUnitJob(job, chunk);
                    }
                    if (job) {
                        feedUnitJob(job, parsed[t].seqs);
                        vector<uint64_t> h; vector<uint32_t> c;
                        finishUnitJob(job, parameters, parsed[t].ref, h, c);
                        references.push_back(std::move(parsed[t].ref));
                    } else {
                        const uint32_t unit = (uint32_t)batch.refs.size();
                        batch.refs.push_back(std::move(parsed[t].ref));
                        for (auto &q : parsed[t].seqs) batch.seqs.push_back(std::move(q));
                        batch.unitOfRecord.insert(batch.unitOfRecord.end(), parsed[t].seqs.size(), unit);
                        batch.bytes += parsed[t].bytes;
                    }
                    vector<mashhost::SeqBuffer>().swap(parsed[t].seqs);
                    { std::lock_guard<std::mutex> lock(mu); consumed = t + 1; }
                    cvRoom.notify_all();
                    if (batchFull(batch, parameters)) flushBatch(batch);
                }
                for (auto &w : workers) w.join();
                i += run - 1;
            } else if (parameters.concatenated) {
                // the unit is parsed on its own; past unitStreamBytes() it streams through a unit job, else it joins the batch
                vector<string> file(1, files[i]);
                Reference ref;
                vector<mashhost::SeqBuffer> seqs;
                vector<uint32_t> unitOfRecord;
                uint64_t bytes = 0;
                mashgpu_unit_job *job = 0;
                DrainFn drain = [&](vector<mashhost::SeqBuffer> &s, vector<uint32_t> &u, uint64_t &b) -> uint64_t {
                    if (!job && b < unitStreamBytes()) return 0;
                    if (!job) {
                        flushBatch(batch);
                        job = openUnitJob(parameters);
                    }
                    feedUnitJob(job, s);
                    u.clear();
                    b = 0;
                    return 0;
                };
                parseUnit(file, parameters, ref, seqs, unitOfRecord, 0, bytes, drain);
                if (job) {
                    vector<uint64_t> h; vector<uint32_t> c;
                    finishUnitJob(job, parameters, ref, h, c);
                    references.push_back(ref);
                } else {
                    const uint32_t unit = (uint32_t)batch.refs.size();
                    batch.refs.push_back(std::move(ref));
                    for (auto &q : seqs) batch.seqs.push_back(std::move(q));
                    batch.unitOfRecord.insert(batch.unitOfRecord.end(), seqs.size(), unit);
                    batch.bytes += bytes;
                }
            } else {
                // one sketch per record (sketchFileBySequence / sketchSequence, reference Sketch.cpp:326-370, 1338-1365)
                gzFile fp = mashhost::FastxReader::openPath(files[i]);
                mashhost::FastxReader reader(fp);
                int l;
                while ((l = reader.read()) >= 0) {
                    if (l < parameters.kmerSize) continue;
                    batch.refs.emplace_back();
                    batch.refs.back().name = reader.name;
                    batch.refs.back().comment = reader.comment;
                    batch.bytes += reader.seq.size();
                    batch.seqs.push_back(std::move(reader.seq));
                    batch.unitOfRecord.push_back((uint32_t)batch.refs.size() - 1);
                    if (batchFull(batch, parameters)) flushBatch(batch);
                }
                gzclose(fp);
                if (l != -1) { cerr << "\nERROR: reading " << files[i] << "." << endl; exit(1); }
            }
            if (batchFull(batch, parameters)) flushBatch(batch);
        }
    }
    flushBatch(batch);
    createIndex();
    return 0;
}

// --------------------------------------------------------------------------------------------------------------
// .msh (Cap'n Proto) I/O -- layout per MinHash.capnp (SURVEY.md 5.1):
//   MinHash: data 3 words {kmerSize u32 @0B, windowSize u32 @4B, minHashesPerWindow u32 @8B, concatenated bit 96,
//            noncanonical bit 97, preserveCase bit 98, error f32 @16B, hashSeed u32 @20B (xor 42)},
//            pointers {0 referenceListOld, 1 locusList, 2 alphabet, 3 referenceList}
//   ReferenceList: 1 pointer (references).  Reference: data 2 words {length u32 @0B, counts32Sorted bit 32,
//            length64 u64 @8B}, pointers {0 sequence, 1 quality, 2 name, 3 comment, 4 hashes32, 5 hashes64, 6 counts32}
//   LocusList: 1 pointer (loci); Locus: data 3 words, no pointers.
// --------------------------------------------------------------------------------------------------------------
namespace {

struct MappedFile {
    void *data = MAP_FAILED;
    size_t size = 0;
    int fd = -1;
    bool open(const char *file)
    {
        fd = ::open(file, O_RDONLY);
        if (fd < 0) return false;
        struct stat info;
        if (fstat(fd, &info) == -1) return false;
        size = info.st_size;
        data = mmap(NULL, size, PROT_READ, MAP_PRIVATE, fd, 0);
        return data != MAP_FAILED;
    }
    ~MappedFile()
    {
        if (data != MAP_FAILED) munmap(data, size);
        if (fd >= 0) close(fd);
    }
};

}  // namespace

uint64_t Sketch::initParametersFromCapnp(const char *file)   // reference Sketch.cpp:255-324
{
    MappedFile m;
    if (!m.open(file)) {
        cerr << "ERROR: could not open \"" << file << "\" for reading." << endl;
        exit(1);
    }
    try {
        capnp_lite::Reader msg(m.data, m.size);
        auto root = msg.root();
        parameters.kmerSize = msg.get<uint32_t>(root, 0);
        parameters.windowSize = msg.get<uint32_t>(root, 4);
        parameters.minHashesPerWindow = msg.get<uint32_t>(root, 8);
        parameters.concatenated = msg.getBit(root, 96);
        parameters.noncanonical = msg.getBit(root, 97);
        parameters.preserveCase = msg.getBit(root, 98);
        parameters.error = msg.get<float>(root, 16);
        parameters.seed = msg.get<uint32_t>(root, 20) ^ 42u;
        auto listNew = msg.getList(msg.getStruct(root, 3), 0);
        auto refs = (listNew.valid && listNew.count) ? listNew : msg.getList(msg.getStruct(root, 0), 0);
        uint64_t referenceCount = refs.valid ? refs.count : 0;
        parameters.counts = referenceCount ? !msg.pointerIsNull(msg.element(refs, 0), 6) : false;
        if (!msg.pointerIsNull(root, 2)) setAlphabetFromString(parameters, msg.getText(root, 2).c_str());
        else setAlphabetFromString(parameters, alphabetNucleotide);
        return referenceCount;
    } catch (const std::exception &e) {
        cerr << "ERROR: \"" << file << "\" is not a valid sketch file (" << e.what() << ")." << endl;
        exit(1);
    }
}

void Sketch::loadCapnp(const char *file)   // reference Sketch.cpp:907-1067
{
    MappedFile m;
    if (!m.open(file)) return;
    try {
        capnp_lite::Reader msg(m.data, m.size);
        auto root = msg.root();
        auto listNew = msg.getList(msg.getStruct(root, 3), 0);
        auto refs = (listNew.valid && listNew.count) ? listNew : msg.getList(msg.getStruct(root, 0), 0);
        uint32_t count = refs.valid ? refs.count : 0;
        size_t base = references.size();
        references.resize(base + count);
        for (uint32_t i = 0; i < count; i++) {
            auto r = msg.element(refs, i);
            Reference &reference = references[base + i];
            reference.name = msg.getText(r, 2);
            reference.comment = msg.getText(r, 3);
            uint64_t length64 = msg.get<uint64_t>(r, 8);
            reference.length = length64 ? length64 : msg.get<uint32_t>(r, 0);
            reference.hashesSorted.setUse64(parameters.use64);
            auto hashes = msg.getList(r, parameters.use64 ? 5 : 4);
            uint64_t hashCount = hashes.valid ? hashes.count : 0;
            if (hashCount > parameters.minHashesPerWindow) hashCount = parameters.minHashesPerWindow;
            reference.hashesSorted.resize((int)hashCount);
            for (uint64_t j = 0; j < hashCount; j++) {
                if (parameters.use64) reference.hashesSorted.set64((int)j, msg.elementU64(hashes, (uint32_t)j));
                else reference.hashesSorted.set32((int)j, msg.elementU32(hashes, (uint32_t)j));
            }
            if (!msg.pointerIsNull(r, 6)) {
                auto counts = msg.getList(r, 6);
                if (!counts.valid || counts.count < hashCount) throw std::runtime_error("counts list shorter than the hash list");
                reference.counts.resize(hashCount);
                for (uint64_t j = 0; j < hashCount; j++) reference.counts[j] = msg.elementU32(counts, (uint32_t)j);
            }
            reference.countsSorted = msg.getBit(r, 32);
        }
    } catch (const std::exception &e) {
        cerr << "ERROR: \"" << file << "\" is not a valid sketch file (" << e.what() << ")." << endl;
        exit(1);
    }
}

int Sketch::writeToCapnp(const char *file) const   // reference Sketch.cpp:384-490, same builder call order
{
    int fd = open(file, O_CREAT | O_WRONLY | O_TRUNC, 0644);
    if (fd < 0) {
        cerr << "ERROR: could not open " << file << " for writing.\n";
        exit(1);
    }
    capnp_lite::Builder b;
    auto rootPtr = b.initRootPointer();
    auto root = b.initStruct(rootPtr, 3, 4);
    auto rootPointers = b.plus(root, 3);
    auto refList = b.initStruct(b.plus(rootPointers, parameters.seed == 42 ? 0 : 3), 0, 1);   // referenceListOld vs referenceList (:397)
    auto refs = b.initStructList(refList, (uint32_t)references.size(), 2, 7);
    for (uint64_t i = 0; i < references.size(); i++) {
        auto r = b.plus(refs, (uint32_t)i * 9);
        auto rp = b.plus(r, 2);
        b.setText(b.plus(rp, 2), references[i].name);
        b.setText(b.plus(rp, 3), references[i].comment);
        b.at(b.plus(r, 1)) = references[i].length;                                           // length64
        const HashList &hashes = references[i].hashesSorted;
        if (hashes.size() != 0) {
            if (parameters.use64) {
                auto h = b.initList(b.plus(rp, 5), 5, (uint32_t)hashes.size());
                for (int j = 0; j != hashes.size(); j++) b.at(b.plus(h, j)) = hashes.at(j).hash64;
            } else {
                auto h = b.initList(b.plus(rp, 4), 4, (uint32_t)hashes.size());
                uint32_t *dst = reinterpret_cast<uint32_t *>(&b.at(h));
                for (int j = 0; j != hashes.size(); j++) dst[j] = hashes.at(j).hash32;
            }
            if (references[i].counts.size() > 0 && parameters.counts) {
                const vector<uint32_t> &counts = references[i].counts;
                auto c = b.initList(b.plus(rp, 6), 4, (uint32_t)counts.size());
                uint32_t *dst = reinterpret_cast<uint32_t *>(&b.at(c));
                for (uint64_t j = 0; j != counts.size(); j++) dst[j] = counts[j];
                b.at(r) |= 1ull << 32;                                                        // counts32Sorted
            }
        }
    }
    auto locusList = b.initStruct(b.plus(rootPointers, 1), 0, 1);
    b.initStructList(locusList, 0, 3, 0);
    // scalars (:472-479): kmerSize, hashSeed (xor default 42), error, minHashesPerWindow, windowSize, flags
    uint32_t w0lo = (uint32_t)parameters.kmerSize, w0hi = (uint32_t)parameters.windowSize;
    b.at(root) = (uint64_t)w0lo | ((uint64_t)w0hi << 32);
    uint64_t flags = (parameters.concatenated ? 1ull : 0) | (parameters.noncanonical ? 2ull : 0) | (parameters.preserveCase ? 4ull : 0);
    b.at(b.plus(root, 1)) = (uint64_t)(uint32_t)parameters.minHashesPerWindow | (flags << 32);
    float error = (float)parameters.error;
    uint32_t errorBits;
    memcpy(&errorBits, &error, 4);
    b.at(b.plus(root, 2)) = (uint64_t)errorBits | ((uint64_t)(parameters.seed ^ 42u) << 32);
    string alphabet;
    getAlphabetAsString(alphabet);
    b.setText(b.plus(rootPointers, 2), alphabet);

    string bytes = b.serialize();
    size_t done = 0;
    while (done < bytes.size()) {
        ssize_t w = write(fd, bytes.data() + done, bytes.size() - done);
        if (w <= 0) { cerr << "ERROR: could not write " << file << endl; exit(1); }
        done += (size_t)w;
    }
    close(fd);
    return 0;
}

void Sketch::toSketchSet(mashgpu_sketch_set &set, vector<uint64_t> &hashes, vector<uint32_t> &n, vector<uint64_t> &lengths) const
{
    uint64_t count = references.size();
    uint64_t stride = 1;
    for (auto &r : references) stride = std::max<uint64_t>(stride, r.hashesSorted.size());
    hashes.assign(count * stride, 0);
    n.resize(count);
    lengths.resize(count);
    for (uint64_t i = 0; i < count; i++) {
        const HashList &list = references[i].hashesSorted;
        n[i] = list.size();
        lengths[i] = references[i].length;
        for (int j = 0; j < list.size(); j++) hashes[i * stride + j] = list.get64() ? list.at(j).hash64 : (uint64_t)list.at(j).hash32;
    }
    set.n = count; set.stride = stride; set.hashes = hashes.data(); set.n_hashes = n.data(); set.length = lengths.data(); set.on_device = 0;
}

}  // namespace mash
