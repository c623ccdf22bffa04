// kj_cli.cpp -- `kaiju-b200`: the reference's command-line surface (src/kaiju.cpp:74-202, usage 430-451) on top of the C ABI.
//   kaiju-b200 -t nodes.dmp -f db.fmi -i reads.fastq [-j reads2.fastq] [-a mem|greedy] [-m -s -e -E -l] [-x|-X] [-o out] [-z N] [-v] [-M kaijux|kaijup]
// Output: "C\t<name>\t<taxid>\n" / "U\t<name>\t0\n" (ConsumerThread.cpp:724-739), in INPUT order.
// Host glue only: option parsing and the string tables; kj_classify_files() reads FASTA/FASTQ(.gz), parses it on the device with the reference's
// name trimming (kaiju.cpp:318-335) and strip() (util.cpp:26-33), classifies and formats every output line.  -z is accepted and ignored (the GPU
// replaces the consumer threads); -p = protein input.  -v prints all seven columns of the reference's -v output (best length/score, taxon ids,
// accessions, fragment strings; KJ_OUT_KAIJU_V), from a device-native index file (no sequence names) columns 1-5 (KJ_OUT_KAIJU_IDS).
// -M kaijux | kaijup (src/kaijux.cpp, kaijup.cpp): the same kernels over an index view that numbers the database sequences (seq_taxon[i] = i + 2
// under one root), so the "taxon id set" of a read is the set of its matching sequences; their names are the label table (KJ_OUT_NAMES, with -v
// KJ_OUT_NAMES_V: the matched fragment strings in the last column).
#include <getopt.h>
#include <unistd.h>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <atomic>
#include <mutex>
#include <stdexcept>
#include <string>
#include <thread>
#include <vector>
#include <algorithm>
#include "kaiju_b200.h"

static uint32_t g_max_read_len = KJ_MAX_READ_LEN;      // -L: longest mate admitted (kj_set_max_read_len)
static uint64_t g_host_bytes = 0;                      // -H: pinned host memory the index may take when it does not fit in HBM (kj_create_tiered)
static bool g_pool = false;                            // -P: one index spread over the HBM of the -d devices (kj_create_group)
static void die(const std::string& m) { fprintf(stderr, "Error: %s\n\n", m.c_str()); exit(EXIT_FAILURE); }
// -l, -s, -m and -e are read as the reference reads them (std::stoi, kaiju.cpp:110-166): the leading number of the argument, which must fit
// in an int.  An argument without one, or out of range, is reported and the option keeps its value.
static bool read_int(const char* s, int& v) {
    try { v = std::stoi(s); return true; } catch (const std::exception&) { return false; }
}
static void usage(const char* prog) {
    fprintf(stderr, "kaiju-b200 (H100-native classification path of Kaiju)\n\nUsage:\n   %s -t nodes.dmp -f kaiju_db.fmi -i reads.fastq [-j reads2.fastq]\n\n"
                    "Mandatory arguments:\n   -t FILENAME   Name of nodes.dmp file\n   -f FILENAME   Name of database (.fmi) file\n   -i FILENAME   Name of input file containing reads in FASTA or FASTQ format (plain, gzip or BGZF;\n                 also a FIFO or pipe, e.g. /dev/stdin or <(zcat r1.fq.gz))\n\n"
                    "Optional arguments:\n   -j FILENAME   Name of second input file for paired-end reads (may be a FIFO or pipe, as -i)\n   -o FILENAME   Name of output file. If not specified, output will be printed to STDOUT\n"
                    "   -z INT        accepted for compatibility (ignored: the GPU replaces the worker threads)\n   -a STRING     Run mode, either \"mem\"  or \"greedy\" (default: greedy)\n"
                    "   -e INT        Number of mismatches allowed in Greedy mode (default: 3)\n   -m INT        Minimum match length (default: 11)\n   -s INT        Minimum match score in Greedy mode (default: 65)\n"
                    "   -E FLOAT      Minimum E-value in Greedy mode (default: 0.01)\n   -x            Enable SEG low complexity filter (enabled by default)\n   -X            Disable SEG low complexity filter\n"
                    "   -w FILENAME   Write the device-native index file for -t/-f and exit; such a file can then be given as -f (no -t needed, no transcode at start-up)\n   -T FILENAME   Also write kaiju2table's summary (reads per taxon of rank -r, default species; needs -N names.dmp) from the counts kept on the GPU\n   -p            Input sequences are protein sequences\n   -L INT        Longest read (bases per mate) to accept, 16383 to 1048575 (default 16383; protein reads: a third of it).  Reads above 16383 bases\n                 run on the long-read kernels, whose per-warp scratch grows with the read length\n   -H GB         Pinned host memory (GiB) the index may take when it does not fit in GPU memory (default 0: GPU memory only); the part\n                 in host memory is read over PCIe, the results are the same\n   -v            Enable verbose output (adds the match length/score, the matching taxon ids, accession numbers and fragment sequences;\n                 with -M the matched fragment sequences)\n   -M STRING     front-end: \"kaijux\" (as kaiju, but reports the names of the matching database sequences; no -t) or \"kaijup\" (the same for protein reads)\n   -d LIST       CUDA device ordinal(s): one number, a comma-separated list, or \"all\" (default 0).  One context (index replica) per listed device.  With at least as many\n                 data sets (-i/-j/-o lists) as devices, the data sets are classified in parallel, each on one device; with fewer, one after\n                 another, each split into batches over all devices (a device may be listed twice: two contexts on one card)\n"
                    "   -P            Pool the GPU memory of the -d devices: one index spread over all of them (for indexes larger than one GPU; the devices\n                 read each other's memory over NVLink) instead of one replica per device; the data sets are classified as without -P.\n                 Not with -H, -w, -M or a device-native index file\n", prog);
    exit(EXIT_FAILURE);
}

int main(int argc, char** argv) {
    kj_params P; P.mode = 1; P.min_fragment_length = 11; P.mismatches = 3; P.min_score = 65; P.seed_length = 7; P.use_evalue = 1; P.min_evalue = 0.01; P.seg = 1; P.input_is_protein = 0; P.name_mode = 0;
    std::string nodes_fn, fmi_fn, in1, in2, out_fn, native_out, table_fn, table_rank = "species", names_fn; bool verbose = false; std::string device_arg = "0", frontend; int c;
    while ((c = getopt(argc, argv, "a:hd:pxXvn:m:e:E:l:t:f:i:j:s:z:o:w:T:r:N:M:L:H:P")) != -1) {
        switch (c) {
            case 'a': if (!strcmp(optarg, "mem")) { P.mode = 0; P.use_evalue = 0; } else if (!strcmp(optarg, "greedy")) P.mode = 1; else { fprintf(stderr, "-a must be a valid mode.\n"); usage(argv[0]); } break;
            case 'h': usage(argv[0]); break;
            case 'd': device_arg = optarg; break;
            case 'P': g_pool = true; break;
            case 'v': verbose = true; break;
            case 'p': P.input_is_protein = 1; break;
            case 'x': P.seg = 1; break;
            case 'X': P.seg = 0; break;
            case 'o': out_fn = optarg; break;
            case 'w': native_out = optarg; break;
            case 'T': table_fn = optarg; break;
            case 'r': table_rank = optarg; break;
            case 'N': names_fn = optarg; break;
            case 'f': fmi_fn = optarg; break;
            case 't': nodes_fn = optarg; break;
            case 'i': in1 = optarg; break;
            case 'j': in2 = optarg; break;
            case 'l': { int v; if (!read_int(optarg, v)) { fprintf(stderr, "Invalid argument in -l %s\n", optarg); break; } if (v < 7) die("Seed length must be >= 7."); P.seed_length = (uint32_t)v; break; }
            case 's': { int v; if (!read_int(optarg, v)) { fprintf(stderr, "Invalid argument in -s %s\n", optarg); break; } if (v <= 0) die("Min Score (-s) must be greater than 0."); P.min_score = (uint32_t)v; break; }
            case 'm': { int v; if (!read_int(optarg, v)) { fprintf(stderr, "Invalid argument in -m %s\n", optarg); break; } if (v <= 0) die("Min fragment length (-m) must be greater than 0."); P.min_fragment_length = (uint32_t)v; break; }
            case 'e': { int v; if (!read_int(optarg, v)) { fprintf(stderr, "Invalid numerical argument in -e %s\n", optarg); break; } if (v < 0) die("Number of mismatches must be >= 0."); P.mismatches = (uint32_t)v; break; }
            case 'E': { P.min_evalue = atof(optarg); if (P.min_evalue <= 0.0) die("E-value threshold must be greater than 0."); break; }
            case 'z': { if (atoi(optarg) <= 0) die("Number of threads (-z) must be greater than 0."); break; }
            case 'n': break;
            case 'M': frontend = optarg; break;
            case 'H': { const double gb = atof(optarg); if (!(gb >= 0.0) || gb > 1e6) die("The host memory budget (-H) must be a number of GB >= 0."); g_host_bytes = (uint64_t)(gb * 1073741824.0); break; }
            case 'L': { const long v = atol(optarg); if (v < KJ_MAX_READ_LEN || v > KJ_MAX_LONG_READ_LEN) die("The read-length limit (-L) must lie between 16383 and 1048575."); g_max_read_len = (uint32_t)v; break; }
            default: usage(argv[0]);
        }
    }
    if (fmi_fn.empty()) { fprintf(stderr, "Error: Please specify the location of the FMI file, using the -f option.\n\n"); usage(argv[0]); }
    { const char* b = strrchr(argv[0], '/'); const std::string prog = b ? b + 1 : argv[0]; if (frontend.empty() && (prog == "kaijux" || prog == "kaijup")) frontend = prog; }
    const bool names = !frontend.empty();
    if (g_pool) {       // a spread index is built from the reference's .fmi, over HBM alone, for the taxon path
        if (g_host_bytes) die("-P cannot be combined with -H: a pooled index lives in GPU memory only.");
        if (!native_out.empty()) die("-P cannot be combined with -w.");
        if (names) die("-P cannot be combined with -M.");
    }
    if (names) {      // -M kaijux | kaijup (or invoked under that name): report the names of the matching database sequences, no taxonomy
        if (frontend != "kaijux" && frontend != "kaijup") die("-M must be kaijux or kaijup");
        if (frontend == "kaijup" && !in2.empty()) die("kaijup takes one input file");
        if (!table_fn.empty()) die("-T cannot be combined with -M: the front-ends report database sequences, not taxa.");
        if (!native_out.empty()) die("-w cannot be combined with -M");
        P.name_mode = 1; P.input_is_protein = frontend == "kaijup" ? 1 : 0;
    }
    // -f may name a device-native index file (written with -w): it holds the taxonomy too, so -t is not needed then
    bool native_in = false;
    { FILE* f = fopen(fmi_fn.c_str(), "rb"); char m[8] = {0}; if (f) { native_in = fread(m, 1, 8, f) == 8 && memcmp(m, "KJB200IX", 8) == 0; fclose(f); } }
    if (g_pool && native_in) die("-P needs the reference's .fmi as -f (device-native index files hold no pooled layout)");
    if (names && native_in) die("-M needs the reference's .fmi as -f (a device-native index file holds no sequence names)");
    if (nodes_fn.empty() && !native_in && !names) { fprintf(stderr, "Error: Please specify the location of the nodes.dmp file, using the -t option.\n\n"); usage(argv[0]); }
    if (!native_out.empty()) {              // -w FILE: transcode .fmi + nodes.dmp into the device-native index file and exit (no GPU needed)
        if (native_in) die("-w needs the reference's .fmi as -f");
        kj_fmi* fmi = nullptr; kj_nodes* nodes = nullptr;
        if (kj_nodes_load(nodes_fn.c_str(), &nodes) != KJ_OK || kj_fmi_load(fmi_fn.c_str(), &fmi) != KJ_OK) die(kj_last_error());
        kj_index_view iv; kj_taxonomy_view tv; kj_fmi_view(fmi, &iv); kj_nodes_view(nodes, &tv);
        if (kj_native_index_write(&iv, &tv, native_out.c_str()) != KJ_OK) die(kj_last_error());
        kj_fmi_free(fmi); kj_nodes_free(nodes);
        return EXIT_SUCCESS;
    }
    if (in1.empty()) { fprintf(stderr, "Error: Please specify the location of the input file, using the -i option.\n\n"); usage(argv[0]); }
    const bool paired = !in2.empty();
    if (paired && P.input_is_protein) { fprintf(stderr, "Error: Protein input only supports one input file.\n\n"); usage(argv[0]); }      // kaiju.cpp:201

    auto split = [](const std::string& v) { std::vector<std::string> out; size_t b = 0; while (b <= v.size()) { size_t e = v.find(',', b); if (e == std::string::npos) e = v.size(); if (e > b) out.push_back(v.substr(b, e - b)); b = e + 1; } return out; };
    const std::vector<std::string> l1 = split(in1), l2 = split(in2), lo = split(out_fn);
    if (l1.empty()) die("Please specify the location of the input file, using the -i option.");
    if (paired && l2.size() != l1.size()) die("Length of input file lists differ");                      // kaiju-multi.cpp:255-258
    if (!lo.empty() && lo.size() != l1.size()) die("Length of input and output file lists differ");
    if (lo.empty() && l1.size() > 1) die("Several input files need a list of output files (-o)");

    // devices: one context (index replica) per listed device.  With at least as many data sets as contexts, each data set goes whole to whichever
    // context is free; with fewer, the data sets run one after another, each one over all contexts (kj_classify_files_multi)
    std::vector<int> devices;
    if (device_arg == "all") { const int nd = kj_device_count(); if (nd <= 0) die("no CUDA device available (this program has no CPU fallback)"); for (int d = 0; d < nd; d++) devices.push_back(d); }
    else for (const std::string& t : split(device_arg)) devices.push_back(atoi(t.c_str()));
    if (devices.empty()) devices.push_back(0);
    if (!g_pool && l1.size() < devices.size() && devices.size() > 8) devices.resize(8);      // one data set over several contexts: at most 8 (kj_classify_files_multi)
    if (g_pool && devices.size() > 8) die("-P pools at most 8 devices.");
    if (!table_fn.empty() && (names_fn.empty() || nodes_fn.empty())) die("The summary table (-T) needs names.dmp (-N) and nodes.dmp (-t).");

    kj_fmi* fmi = nullptr; kj_nodes* nodes = nullptr; kj_index_view iv; kj_taxonomy_view tv;
    std::vector<uint64_t> star_taxon, star_node, star_parent;      // -M: sequences numbered 2.. under the root 1 (ascending id = the front-ends' order)
    if (!native_in) {
        if (!names && kj_nodes_load(nodes_fn.c_str(), &nodes) != KJ_OK) die(kj_last_error());
        if (kj_fmi_load(fmi_fn.c_str(), &fmi) != KJ_OK) die(kj_last_error());
        kj_fmi_view(fmi, &iv);
        if (names) {
            star_taxon.resize((size_t)iv.nseq); star_node.resize((size_t)iv.nseq + 1); star_parent.assign((size_t)iv.nseq + 1, 1);
            star_node[0] = 1; for (int32_t i = 0; i < iv.nseq; i++) { star_taxon[(size_t)i] = (uint64_t)i + 2; star_node[(size_t)i + 1] = (uint64_t)i + 2; }
            iv.seq_taxon = star_taxon.data(); tv.n = star_node.size(); tv.node = star_node.data(); tv.parent = star_parent.data();
        } else kj_nodes_view(nodes, &tv);
    }
    std::vector<kj_ctx*> ctxs(devices.size(), nullptr);
    if (g_pool) {       // one spread index, one context per device; the contexts take the data sets as replicas do
        int rc = kj_create_group(ctxs.data(), (int)devices.size(), devices.data(), &P, &iv, &tv, 1);
        for (size_t d = 0; rc == KJ_OK && d < ctxs.size(); d++) rc = kj_set_max_read_len(ctxs[d], g_max_read_len);
        if (rc != KJ_OK) die(kj_last_error());
    } else {
        // one thread per distinct device; the contexts of one device are created one after another (the construction sizes its temporary
        // buffers from the free HBM it finds, which a second construction running beside it would take away)
        std::vector<std::thread> th; std::mutex mu; std::string err;
        for (size_t d = 0; d < devices.size(); d++) {
            if (std::find(devices.begin(), devices.begin() + (long)d, devices[d]) != devices.begin() + (long)d) continue;
            th.emplace_back([&, d] {
                for (size_t e = d; e < devices.size(); e++) {
                    if (devices[e] != devices[d]) continue;
                    int rc = native_in ? kj_create_from_native(&ctxs[e], devices[e], &P, fmi_fn.c_str()) : kj_create_tiered(&ctxs[e], devices[e], &P, &iv, &tv, 1, g_host_bytes);
                    if (rc == KJ_OK) rc = kj_set_max_read_len(ctxs[e], g_max_read_len);
                    if (rc != KJ_OK) { std::lock_guard<std::mutex> lk(mu); if (err.empty()) err = kj_last_error(); return; }
                }
            });
        }
        for (auto& x : th) x.join();
        if (!err.empty()) die(err);
    }
    // the line format, and the strings it prints: -M the database sequence names by dense taxon index (id i + 2 = sequence i), -v the accessions
    const int fmt = names ? (verbose ? KJ_OUT_NAMES_V : KJ_OUT_NAMES) : !verbose ? KJ_OUT_KAIJU : fmi ? KJ_OUT_KAIJU_V : KJ_OUT_KAIJU_IDS;
    if (fmt == KJ_OUT_KAIJU_V || names) {
        std::string blob; std::vector<uint64_t> off{0};
        if (names) {
            std::vector<uint64_t> ids(kj_counts_size(ctxs[0])), cnt(ids.size());
            if (kj_counts_get(ctxs[0], ids.data(), cnt.data()) != KJ_OK) die(kj_last_error());
            for (size_t k = 0; k + 1 < ids.size(); k++) { if (ids[k] >= 2 && ids[k] - 2 < (uint64_t)iv.nseq) blob += kj_fmi_seq_name(fmi, (int32_t)(ids[k] - 2)); off.push_back(blob.size()); }
        } else {
            uint32_t n_acc = 0;
            if (iv.seq_accession) for (int32_t i = 0; i < iv.nseq; i++) if (iv.seq_accession[i] != 0xffffffffu) n_acc = std::max(n_acc, iv.seq_accession[i] + 1);
            for (uint32_t r = 0; r < n_acc; r++) { const char* a = kj_fmi_accession(fmi, r); if (a) blob += a; off.push_back(blob.size()); }
        }
        for (kj_ctx* ctx : ctxs) if (kj_set_output_strings(ctx, names ? KJ_STR_TAXON : KJ_STR_ACCESSION, blob.data(), off.data(), off.size() - 1) != KJ_OK) die(kj_last_error());
    }
    if (fmi) { kj_fmi_free(fmi); fmi = nullptr; }
    if (nodes) kj_nodes_free(nodes);

    // parsing, classification and output formatting all run on the device; the host moves bytes (kj_ingest.h).
    // Comma-separated lists for -i / -j / -o process several data sets against the index loaded once per device (kaiju-multi.cpp:220-330).
    struct Done { uint64_t n_reads = 0, n_classified = 0, inflated = 0; double secs = 0; std::vector<uint64_t> ids, counts; };
    std::vector<Done> done(l1.size()); std::atomic<size_t> next(0); std::mutex mu; std::string err;
    // data set k on the contexts cs[0, n): its output, and with -T the sum of the contexts' counts (their id lists are the same)
    auto run_set = [&](size_t k, kj_ctx** cs, int n) -> int {
        Done& r = done[k]; int rc = KJ_OK;
        for (int i = 0; rc == KJ_OK && i < n && !table_fn.empty(); i++) rc = kj_counts_reset(cs[i]);
        const auto t0 = std::chrono::steady_clock::now();
        if (rc == KJ_OK) rc = kj_classify_files_multi(cs, n, l1[k].c_str(), paired ? l2[k].c_str() : nullptr, lo.empty() ? nullptr : lo[k].c_str(), fmt, &r.n_reads, &r.n_classified);
        r.secs = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
        r.inflated = kj_files_device_inflated_bytes(cs[0]);
        if (rc == KJ_OK && !table_fn.empty()) {
            r.ids.resize(kj_counts_size(cs[0])); r.counts.assign(r.ids.size(), 0);
            std::vector<uint64_t> ids(r.ids.size()), cnt(r.ids.size());
            for (int i = 0; rc == KJ_OK && i < n; i++) {
                if ((rc = kj_counts_get(cs[i], ids.data(), cnt.data())) != KJ_OK) break;      // (kj_classify_files_multi checked that the vectors have one size)
                if (i == 0) r.ids = ids; else if (ids != r.ids) die("the contexts of -d count different taxa");
                for (size_t t = 0; t < cnt.size(); t++) r.counts[t] += cnt[t];
            }
        }
        return rc;
    };
    if (l1.size() < ctxs.size()) {        // fewer data sets than contexts: each one over every context, in list order
        for (size_t k = 0; k < l1.size(); k++) if (run_set(k, ctxs.data(), (int)ctxs.size()) != KJ_OK) die(kj_last_error());
    } else {
        std::vector<std::thread> workers;
        for (size_t d = 0; d < ctxs.size(); d++) workers.emplace_back([&, d] {
            for (;;) {
                const size_t k = next.fetch_add(1); if (k >= l1.size()) return;
                { std::lock_guard<std::mutex> lk(mu); if (!err.empty()) return; }
                if (run_set(k, &ctxs[d], 1) != KJ_OK) { std::lock_guard<std::mutex> lk(mu); if (err.empty()) err = kj_last_error(); return; }
            }
        });
        for (auto& x : workers) x.join();
        if (!err.empty()) die(err);
    }
    for (size_t k = 0; k < l1.size(); k++) {
        if (!table_fn.empty()) {     // kaiju2table's report from the per-taxon counts kept in HBM (one block of rows per data set, in list order)
            kj_table_opts to; memset(&to, 0, sizeof to); to.rank = table_rank.c_str();
            const std::string label = lo.empty() ? l1[k] : lo[k];
            if (kj_table_write(done[k].ids.data(), done[k].counts.data(), done[k].ids.size(), nodes_fn.c_str(), names_fn.c_str(), label.c_str(), &to, table_fn.c_str(), k > 0) != KJ_OK) die(kj_last_error());
        }
        if (verbose || getenv("KJ_CLI_TIMING")) fprintf(stderr, "%s: %llu reads, %llu classified, %.4f s from the first byte read to the last byte written\n", l1[k].c_str(), (unsigned long long)done[k].n_reads, (unsigned long long)done[k].n_classified, done[k].secs);
        if (getenv("KJ_CLI_TIMING")) fprintf(stderr, "%s: %llu bytes of text inflated on the device (BGZF input; 0: plain text, or gzip inflated by zlib on the host)\n", l1[k].c_str(), (unsigned long long)done[k].inflated);
    }
    for (kj_ctx* ctx : ctxs) kj_destroy(ctx);
    if (fmi) kj_fmi_free(fmi);
    return EXIT_SUCCESS;
}
