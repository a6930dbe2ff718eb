// Drop-in `db_sort` and `set_lcas` executables over libkuq's C ABI — SURVEY.md §8 row f4.
// Built twice from this file: plain → db_sort (db_sort.cpp:41-187), -DTOOL_SET_LCAS → set_lcas (set_lcas.cpp:92-600).
// Same getopt strings, same file side effects; the work itself (minimizer binning + sort, k-mer lookup + LCA update)
// runs on the GPU.  ROUND 1 STATUS: written after the round's GPU budget was spent — compiles, not yet run on
// hardware.  The oracle's CPU statements of both tools are pinned against the reference executables
// (tests/test_oracle_db_build.py).
//
// set_lcas options NOT supported (exit with a message): -I (UIDs).
#include <fcntl.h>
#include <getopt.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <sysexits.h>
#include <unistd.h>

#include <algorithm>
#include <cctype>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <iostream>
#include <map>
#include <mutex>
#include <sstream>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

#include "../../include/kuq.h"
#include "kuq_dbfile.h"
#include "kuq_ranges.h"

using namespace std;

[[noreturn]] static void die(int code, const string &msg, const char *tool) {
  cerr << tool << ": " << msg << endl;
  exit(code);
}

struct Mapped {
  void *p = NULL;
  size_t size = 0;
  void open(const string &path, const char *tool) {
    int fd = ::open(path.c_str(), O_RDONLY);
    if (fd < 0) die(EX_OSERR, "unable to open " + path, tool);
    struct stat sb;
    if (fstat(fd, &sb) < 0) die(EX_OSERR, "unable to fstat " + path, tool);
    size = sb.st_size;
    p = size ? mmap(0, size, PROT_READ, MAP_PRIVATE, fd, 0) : NULL;
    if (size && p == MAP_FAILED) die(EX_OSERR, "unable to mmap " + path, tool);
    ::close(fd);
  }
};

// The devices the tool may use, as classify picks them: KUQ_DEVICES=0,2,3 (or "all"), else KUQ_DEVICE=n alone, else
// every visible sm_90 device.  An ordinal may repeat: several workers on one card.
static vector<int> pick_devices() {
  vector<int> devices;
  const char *dl = getenv("KUQ_DEVICES");
  if (dl && strcmp(dl, "all") != 0) {
    for (const char *q = dl; *q;) { devices.push_back(atoi(q)); while (*q && *q != ',') q++; if (*q) q++; }
  } else if (dl || !getenv("KUQ_DEVICE")) {
    for (int d = 0; d < kuq_device_count(); d++) devices.push_back(d);
  }
  if (devices.empty()) devices.assign(1, getenv("KUQ_DEVICE") ? atoi(getenv("KUQ_DEVICE")) : 0);
  return devices;
}

static void write_file(const string &path, const void *data, size_t size, const char *tool) {
  ofstream out(path.c_str(), ofstream::binary);
  if (!out.is_open()) die(EX_CANTCREAT, "can't write " + path, tool);
  out.write((const char *)data, (streamsize)size);
  out.close();
  if (!out) die(EX_IOERR, "error writing " + path, tool);
}

#ifndef TOOL_SET_LCAS
// ====================================================================================================================
// db_sort
// ====================================================================================================================
static const char *TOOL = "db_sort";
static void usage(int exit_code = EX_USAGE) {
  cerr << "Usage: db_sort [-z] [-M] [-t threads] [-n nt] <-d input db> <-o output db> <-i output idx>\n"
       << "KUQ_DB_SORT_BUDGET (bytes of device memory; default 3/4 of the free memory): a database whose sort does not fit\n"
       << "is sorted in passes over minimizer ranges.\n"
       << "KUQ_DEVICES (0,2,3 or all; default: every visible GPU) or KUQ_DEVICE: the devices that share the passes.\n";
  exit(exit_code);
}

int main(int argc, char **argv) {
  string input, output, index;
  uint32_t nt = 15;                                     // Bin_key_nt, db_sort.cpp:27
  bool zero_vals = false;
  if (argc > 1 && strcmp(argv[1], "-h") == 0) usage(0);
  int opt;
  while ((opt = getopt(argc, argv, "n:d:o:i:t:zM")) != -1) {
    switch (opt) {
      case 'n': {
        long long sig = atoll(optarg);
        if (sig < 1 || sig > 31) die(EX_USAGE, "bin key length out of range", TOOL);
        nt = (uint32_t)sig;
        break;
      }
      case 'd': input = optarg; break;
      case 'o': output = optarg; break;
      case 'i': index = optarg; break;
      case 'M': break;                                  // the images are in memory anyway
      case 't':
        if (atoll(optarg) <= 0) die(EX_USAGE, "can't use nonpositive thread count", TOOL);
        break;
      case 'z': zero_vals = true; break;
      default: usage();
    }
  }
  if (input.empty() || output.empty() || index.empty()) usage();
  if (nt > 15) die(EX_USAGE, "bin key lengths above 15 overflow the reference's own index arithmetic (krakendb.cpp:204)", TOOL);
  cerr << "db_sort: Getting database into memory ...";
  Mapped in;
  in.open(input, TOOL);
  if (in.size < 56) die(EX_DATAERR, "input database too short", TOOL);
  const KdbFile h = kdb_view(in.p);
  vector<char> kdb(h.header_bytes + h.key_ct * h.pair_sz), idx(8 + 8 * ((1ull << (2 * nt)) + 1));
  cerr << "db_sort: Sorting ...";
  char err[512] = "";
  const vector<int> devices = pick_devices();
  uint32_t passes = 0;                                  // budget: KUQ_DB_SORT_BUDGET, else 3/4 of free device memory
  int rc = kuq_db_sort_devices(devices.data(), (uint32_t)devices.size(), in.p, in.size, nt, zero_vals, 0, kdb.data(),
                               idx.data(), &passes, err, sizeof err);
  if (rc) die(rc == KUQ_E_NO_DEVICE ? EX_UNAVAILABLE : EX_DATAERR, err[0] ? err : kuq_strerror(rc), TOOL);
  cerr << "db_sort: " << passes << (passes == 1 ? " pass" : " passes");
  if (passes > 1) cerr << " on " << devices.size() << (devices.size() == 1 ? " device" : " devices");
  cerr << endl;
  cerr << "db_sort: Sorting complete - writing database to disk ..." << endl;
  write_file(index, idx.data(), idx.size(), TOOL);       // make_index, krakendb.cpp:141-147
  write_file(output, kdb.data(), kdb.size(), TOOL);      // db_sort.cpp:69-73
  return 0;
}

#else
// ====================================================================================================================
// set_lcas
// ====================================================================================================================
static const char *TOOL = "set_lcas";
static const size_t SKIP_LEN = 50000;                    // set_lcas.cpp:31
static const uint32_t TID_HUMAN = 9606, TID_MOUSE = 10090;  // host taxa get no sequence taxa, :83-84
static bool Allow_extra_kmers = false, verbose = false, Operate_in_RAM = false, Pretend = false;
static bool Add_taxids_for_sequences = false, Add_taxids_for_assembly = false;   // -a / -A (set_lcas.cpp:528-533)
static uint32_t Minimum_sequence_size = 0;
static uint32_t Lca_flags = 0;                           // -T → KUQ_LCA_FORCE_CONTAMINANT, -R → KUQ_LCA_RESET
static string DB_filename, Index_filename, TaxDB_filename, File_to_taxon_map_filename, ID_to_taxon_map_filename,
    Multi_fasta_filename, Output_DB_filename, Kmer_count_filename;

static void usage(int exit_code = EX_USAGE) {
  cerr << "Usage: set_lcas [options]" << endl << endl
       << "Options: (*mandatory)" << endl
       << "* -d filename      Kraken DB filename" << endl
       << "* -i filename      Kraken DB index filename" << endl
       << "* -b filename      Taxonomy DB file" << endl
       << "  -t #             Number of threads" << endl
       << "  -M               Copy DB to RAM during operation" << endl
       << "  -o filename      Output database to filename, instead of overwriting the input database" << endl
       << "  -x               K-mers not found in DB do not cause errors" << endl
       << "  -f filename      File to taxon map" << endl
       << "  -F filename      Multi-FASTA file with sequence data" << endl
       << "  -m filename      Sequence ID to taxon map" << endl
       << "  -a               Add taxonomy IDs (starting with 1000000001) for sequences to Taxonomy DB" << endl
       << "  -A               Add taxonomy IDs (starting with 1000000001) for assemblies (third column in seqid2taxid.map) to Taxonomy DB" << endl
       << "  -T             When a k-mer appears in a 'synthetic construct' sequence, force the taxID to be the 'synthetic construct' taxID, instead of the LCA." << endl
       << "  -R               Reset the taxIDs of the k-mers of the sequences to 0" << endl
       << "  -E #             Exclude sequences that are shorter than the threshold." << endl
       << "  -c filename      Write k-mer counts per taxon to filename" << endl
       << "  -p               Pretend - do not write database back to disk" << endl
       << "  -v               Verbose output" << endl
       << "  -h               Print this message" << endl << endl
       << "-F and -m must be specified together.  If -f is given, -F/-m are ignored." << endl
       << "(GPU build: -I is not supported)" << endl;
  exit(exit_code);
}

// FastaReader::next_sequence (seqreader.cpp:34-79): header = line after '>', id = its first word, sequence = the
// following lines glued together until the next '>' line
struct Fasta {
  ifstream file;
  string linebuffer;
  bool valid = false;
  explicit Fasta(const string &path) : file(path.c_str()) {
    if (file.rdstate() & ifstream::failbit) die(EX_NOINPUT, "can't open " + path, TOOL);
    valid = true;
  }
  bool next(string &id, string &header, string &seq) {
    id.clear(); header.clear(); seq.clear();
    if (!file.good()) { valid = false; return false; }
    string line;
    if (linebuffer.empty()) getline(file, line);
    else { line = linebuffer; linebuffer.clear(); }
    if (line.empty() || line[0] != '>') {
      cerr << "set_lcas: malformed fasta file - expected header char > not found" << endl;
      valid = false;
      return false;
    }
    header = line.substr(1);
    istringstream ss(header);
    ss >> id;
    while (file.good()) {
      getline(file, line);
      if (!line.empty() && line[0] == '>') { linebuffer = line; break; }
      seq += line;
    }
    return true;
  }
};

struct Batch {
  string bases;
  vector<uint64_t> offs{0};
  vector<uint32_t> taxids;
  uint32_t contaminant = 0;        // the one contaminant taxid (32630 / 81077) this batch holds, 0 = none yet
};
static uint32_t K = 0;
static const uint64_t BATCH_NT = 64ull << 20;

// One context per device entry that owns minimizer ranges: ranges[0] stays staged while the library is read, the
// others are staged after it in turn.  missing: the library's k-mers its ranges lack; code / msg: its first failure.
struct Context {
  kuq_ctx *ctx = NULL;
  vector<pair<uint64_t, uint64_t>> ranges;
  size_t first_range = 0;                                // the plan's index of ranges[0]
  uint64_t missing = 0, batch_missing = 0;
  int code = 0;
  string msg;
  void fail(int c, const string &m) { if (!code) { code = c; msg = m; } }
};
static vector<Context> Ctxs;
static uint64_t Missing_total = 0;
// With a context that owns several ranges every batch is kept to be replayed against its later ranges: the library may
// be a pipe that can be read once (build_db.sh passes -F <(cat_library)).  With at most one range per context the
// library is read once and never held.
static bool Keep_batches = false;
static vector<Batch> Kept;

// f(context) on every context at once, one host thread each (none for a single context); then the first failure ends
// the run
template <typename F>
static void on_contexts(F f) {
  if (Ctxs.size() == 1) {
    f(Ctxs[0]);
  } else {
    vector<thread> th;
    for (Context &c : Ctxs) th.emplace_back([&c, &f] { f(c); });
    for (thread &t : th) t.join();
  }
  for (Context &c : Ctxs)
    if (c.code) die(c.code, c.msg, TOOL);
}

static void lca_batch(Context &c, const Batch &b) {
  c.batch_missing = 0;
  if (kuq_set_lcas_batch(c.ctx, b.bases.data(), b.offs.data(), (uint32_t)b.taxids.size(), b.taxids.data(), Lca_flags, &c.batch_missing))
    c.fail(EX_SOFTWARE, kuq_last_error(c.ctx));
  c.missing += c.batch_missing;
}

static void check_missing() {
  for (Context &c : Ctxs)
    if (c.batch_missing && !Allow_extra_kmers) die(EX_DATAERR, "kmer found in sequence that is not in database", TOOL);   // :441-443
}

// every context looks the batch up in its staged range
static void run_batch(const Batch &b) {
  on_contexts([&](Context &c) { lca_batch(c, b); });
  check_missing();
}

static void flush(Batch &b) {
  if (b.taxids.empty()) return;
  run_batch(b);
  if (Keep_batches) { Kept.push_back(std::move(b)); b = Batch(); return; }
  b.bases.clear(); b.offs.assign(1, 0); b.taxids.clear(); b.contaminant = 0;
}

// the reference's pieces: [i, i + SKIP_LEN + k - 1) for i = 0, SKIP_LEN, ... (set_lcas.cpp:363-364, 399-400)
static void add_sequence(Batch &b, const string &seq, uint32_t taxid) {
  if (taxid == 32630u || taxid == 81077u) {              // TID_CONTAMINANT1/2, set_lcas.cpp:88-89
    // under -T the first contaminant taxid to reach a k-mer stays: keep file order between the two kinds
    if (b.contaminant && b.contaminant != taxid) flush(b);
    b.contaminant = taxid;
  }
  for (size_t i = 0; i < seq.size(); i += SKIP_LEN) {
    const size_t len = min(seq.size() - i, SKIP_LEN + K - 1);
    if (b.bases.size() + len > BATCH_NT || b.taxids.size() >= (1u << 19)) flush(b);
    b.bases.append(seq, i, len);
    b.offs.push_back(b.bases.size());
    b.taxids.push_back(taxid);
  }
}

// ---- the taxonomy as TaxonomyDB holds it (readTaxonomyIndex_, taxdb.hpp:563-605), and the taxa -a / -A add to it ----
struct Taxon {
  uint32_t parent;                 // the row's parent pointer; `linked` false = NULL (the root, an unknown parent, row 0)
  bool linked;
  string name, rank;
};
// One insert per taxDB line in file order (the first line of a taxid wins), then taxid 0 'unclassified'.  The
// insert sequence is the reference's, so iterating this map visits taxids in the reference's order, which decides
// where new taxids start (set_lcas.cpp:219-224).
static unordered_map<uint32_t, Taxon> Taxa;
static uint32_t New_taxid_start = 1000000000;            // set_lcas.cpp:51
static unordered_map<string, uint32_t> Name_to_taxid;   // assembly names and sequence ids share one cache

static void read_taxdb(const string &path) {
  ifstream in(path.c_str());
  if (!in.is_open()) die(EX_NOINPUT, "unable to open taxonomy index file " + path, TOOL);
  string line;
  while (getline(in, line)) {                            // id \t parent \t name \t rank
    size_t a = line.find('\t'), b = a == string::npos ? a : line.find('\t', a + 1);
    if (a == string::npos || b == string::npos) continue;
    const size_t c = line.find('\t', b + 1);
    Taxon t{(uint32_t)strtoul(line.substr(a + 1, b - a - 1).c_str(), NULL, 10), false,
            line.substr(b + 1, c == string::npos ? string::npos : c - b - 1), c == string::npos ? "" : line.substr(c + 1)};
    Taxa.emplace((uint32_t)strtoul(line.substr(0, a).c_str(), NULL, 10), t);
  }
  Taxa.emplace(0u, Taxon{0, false, "unclassified", "no rank"});
  for (auto &kv : Taxa)                                  // createPointers, taxdb.hpp:412-433
    kv.second.linked = kv.second.parent != kv.first && Taxa.count(kv.second.parent);
}

// Parent_map (getParentMap, taxdb.hpp:383-398): the parent pointer's taxid, 0 for none
static uint32_t parent_map(uint32_t taxid) {
  const Taxon &t = Taxa.at(taxid);
  return t.linked ? t.parent : 0;
}

// get_new_taxid (set_lcas.cpp:183-203): the id is used up even when the parent is unknown and nothing is added
static uint32_t new_taxid(const string &name, uint32_t parent, const char *rank) {
  auto it = Name_to_taxid.find(name);
  if (it != Name_to_taxid.end()) return it->second;
  const uint32_t id = ++New_taxid_start;
  if (parent == id) return 0;
  if (!Taxa.count(parent)) {
    cerr << "ERROR with taxon [" << id << ";" << rank << ";" << name << "] - parent taxon " << parent << " not in database!" << endl;
    return 0;
  }
  if (!Taxa.emplace(id, Taxon{parent, true, name, rank}).second) return 0;
  Name_to_taxid[name] = id;
  return id;
}

// writeTaxonomyIndex (taxdb.hpp:533-547): ascending taxids, a row without a parent pointer names itself
static void write_taxdb(const string &path) {
  vector<uint32_t> keys;
  for (auto &kv : Taxa) keys.push_back(kv.first);
  sort(keys.begin(), keys.end());
  string out;
  for (uint32_t id : keys) {
    const Taxon &t = Taxa.at(id);
    out += to_string(id) + '\t' + to_string(t.linked ? t.parent : id) + '\t' + t.name + '\t' + t.rank + '\n';
  }
  write_file(path, out.data(), out.size(), TOOL);
}

// read_seqid_to_taxid_map (set_lcas.cpp:205-266): the first mapping of a sequence id wins.  With -A / -a the
// assembly (third column) and sequence taxa are created here, before any sequence is read, and each mapping is
// printed on stdout.
static unordered_map<string, uint32_t> read_seqid_map(const string &path) {
  cerr << "Reading sequence ID to taxonomy ID mapping ... ";
  unordered_map<string, uint32_t> id_to_taxon;
  ifstream map_file(path.c_str());
  if (map_file.rdstate() & ifstream::failbit) die(EX_NOINPUT, "can't open " + path, TOOL);
  const bool add = Add_taxids_for_assembly || Add_taxids_for_sequences;
  if (add) {
    for (auto &kv : Taxa)
      if (kv.first >= New_taxid_start) New_taxid_start = kv.first + 100;
    cerr << "[starting new taxonomy IDs with " << (New_taxid_start + 1) << ']';
  }
  string line, seq_id, name;
  uint32_t taxid = 0;
  while (map_file.good()) {
    getline(map_file, line);
    if (line.empty()) break;
    istringstream iss(line);
    iss >> seq_id >> taxid;
    if (id_to_taxon.count(seq_id)) continue;
    const uint32_t orig_taxid = taxid;
    if (Add_taxids_for_assembly && iss.good()) {         // one separator, then the rest of the line
      iss.get();
      getline(iss, name);
      if (!name.empty()) taxid = new_taxid(name, taxid, "assembly");
    }
    if (Add_taxids_for_sequences && orig_taxid != TID_HUMAN && orig_taxid != TID_MOUSE)
      taxid = new_taxid(seq_id, taxid, "sequence");
    if (add) cout << seq_id << '\t' << taxid << '\n';
    id_to_taxon[seq_id] = taxid;
  }
  if (id_to_taxon.empty()) cerr << "Error: No ID mappings present!!" << endl;
  cerr << " got " << id_to_taxon.size() << " mappings." << endl;
  return id_to_taxon;
}

// The minimizer ranges of the database, each staged on one context at a time: as few as `budget` bytes of device
// memory allow, 12 bytes per record in HBM.  Together they cover every bin, so that a k-mer whose bin holds no records
// is still counted as missing.  {(0, 0)} = the whole database at once.
static vector<pair<uint64_t, uint64_t>> plan_lca_ranges(const DbFile &f, uint64_t budget) {
  const vector<pair<uint64_t, uint64_t>> whole{{0, 0}};
  vector<pair<uint64_t, uint64_t>> ranges;
  if (!plan_ranges(f.offsets, f.n_bins, budget, 12, ranges)) die(EX_SOFTWARE, "a single minimizer bin exceeds KUQ_SET_LCAS_BUDGET", TOOL);
  if (ranges.size() <= 1) return whole;
  ranges.front().first = 0;                              // bins of ranges without records join the range before them
  for (size_t r = 1; r < ranges.size(); r++) ranges[r - 1].second = ranges[r].first;
  ranges.back().second = f.n_bins;
  return ranges;
}

// A context's default budget (KUQ_SET_LCAS_BUDGET unset): its device's free memory less 1 GiB for the batch and the
// staging buffers, shared among the `sharing` contexts on that device
static uint64_t default_budget(kuq_ctx *ctx, uint32_t sharing) {
  const uint64_t free_b = kuq_device_free_bytes(ctx);
  return (free_b > (2ull << 30) ? free_b - (1ull << 30) : free_b / 2) / sharing;
}

static kuq_ctx *create_context(int device) {
  kuq_config cfg;
  kuq_config_default(&cfg);
  cfg.n_slots = 1;
  cfg.max_bases_per_batch = BATCH_NT + (1 << 20);
  cfg.hll_mode = KUQ_HLL_DENSE_ONLY;                      // no sketches are used here
  cfg.device = device;
  kuq_ctx *ctx = NULL;
  int rc = kuq_create(&cfg, &ctx);
  if (rc) die(EX_UNAVAILABLE, string("libkuq: ") + kuq_strerror(rc), TOOL);
  return ctx;
}

static void stage(Context &c, const Mapped &kdb, const Mapped &idx, const pair<uint64_t, uint64_t> &range) {
  if (kuq_stage_db(c.ctx, kdb.p, kdb.size, idx.p, idx.size, range.first, range.second)) c.fail(EX_DATAERR, kuq_last_error(c.ctx));
}

// the context's staged values, counted by taxid on the device, added to `counts`
static void add_value_counts(Context &c, map<uint32_t, uint64_t> &counts) {
  uint32_t m = 0;
  if (kuq_db_value_counts(c.ctx, NULL, NULL, 0, &m)) return c.fail(EX_SOFTWARE, kuq_last_error(c.ctx));
  vector<uint32_t> t(m);
  vector<uint64_t> n(m);
  if (m && kuq_db_value_counts(c.ctx, t.data(), n.data(), m, &m)) return c.fail(EX_SOFTWARE, kuq_last_error(c.ctx));
  for (uint32_t i = 0; i < m; i++) counts[t[i]] += n[i];
}

int main(int argc, char **argv) {
  if (argc > 1 && strcmp(argv[1], "-h") == 0) usage(0);
  int opt;
  while ((opt = getopt(argc, argv, "f:d:i:t:n:m:F:xMTRvb:aApI:o:Sc:E:")) != -1) {
    switch (opt) {
      case 'f': File_to_taxon_map_filename = optarg; break;
      case 'd': DB_filename = optarg; break;
      case 'i': Index_filename = optarg; break;
      case 'F': Multi_fasta_filename = optarg; break;
      case 'm': ID_to_taxon_map_filename = optarg; break;
      case 't':
        if (atoll(optarg) <= 0) die(EX_USAGE, "can't use nonpositive thread count", TOOL);
        break;
      case 'v': verbose = true; break;
      case 'x': Allow_extra_kmers = true; break;
      case 'b': TaxDB_filename = optarg; break;
      case 'c': Kmer_count_filename = optarg; break;
      case 'M': Operate_in_RAM = true; break;
      case 'o': Output_DB_filename = optarg; break;
      case 'E': Minimum_sequence_size = (uint32_t)atoi(optarg); break;
      case 'p': Pretend = true; break;
      case 'n': case 'S': break;
      case 'T': Lca_flags |= KUQ_LCA_FORCE_CONTAMINANT; break;
      case 'R': Lca_flags |= KUQ_LCA_RESET; break;
      case 'a': Add_taxids_for_sequences = true; break;
      case 'A': Add_taxids_for_assembly = true; break;
      case 'I':
        die(EX_USAGE, string("option -") + (char)opt + " is not supported by the GPU set_lcas", TOOL);
      default: usage();
    }
  }
  if (DB_filename.empty() || Index_filename.empty() || TaxDB_filename.empty()) usage();
  if (File_to_taxon_map_filename.empty() && (Multi_fasta_filename.empty() || ID_to_taxon_map_filename.empty())) usage();
  const bool one_fasta_file = File_to_taxon_map_filename.empty();

  read_taxdb(TaxDB_filename);

  Mapped kdb, idx;
  kdb.open(DB_filename, TOOL);
  idx.open(Index_filename, TOOL);
  DbFile file;
  string parse_err;
  if (parse_db(kdb.p, kdb.size, idx.p, idx.size, file, parse_err)) die(EX_DATAERR, parse_err, TOOL);
  K = file.k;
  // the range plan: from KUQ_SET_LCAS_BUDGET, else from the first device's free memory; when the database takes more
  // than one range and there are more devices, every context's share of its device (the smallest share of all)
  const vector<int> devices = pick_devices();
  const char *budget_env = getenv("KUQ_SET_LCAS_BUDGET");
  const uint64_t given = budget_env ? strtoull(budget_env, NULL, 10) : 0;
  vector<kuq_ctx *> made{create_context(devices[0])};
  vector<pair<uint64_t, uint64_t>> ranges = plan_lca_ranges(file, given ? given : default_budget(made[0], 1));
  if (ranges.size() > 1 && devices.size() > 1) {
    for (size_t g = 1; g < devices.size(); g++) made.push_back(create_context(devices[g]));
    if (!given) {
      uint64_t budget = UINT64_MAX;
      for (size_t g = 0; g < devices.size(); g++)
        budget = min(budget, default_budget(made[g], (uint32_t)count(devices.begin(), devices.end(), devices[g])));
      ranges = plan_lca_ranges(file, budget);
    }
  }
  // one range per context while there are enough contexts (the library is then never kept), else contiguous groups
  // balanced by the bytes each range stages; a context without ranges is let go
  vector<size_t> first{0, ranges.size()};
  if (made.size() > 1 && ranges.size() <= made.size()) {
    first.resize(made.size() + 1);
    for (size_t g = 0; g <= made.size(); g++) first[g] = min(g, ranges.size());
  } else if (made.size() > 1) {
    first = group_ranges((const uint64_t *)((const uint8_t *)idx.p + 8), ranges, (int)made.size(), 12);
  }
  for (size_t g = 0; g < made.size(); g++) {
    if (first[g] == first[g + 1]) { kuq_destroy(made[g]); continue; }
    Ctxs.emplace_back();
    Ctxs.back().ctx = made[g];
    Ctxs.back().ranges.assign(ranges.begin() + first[g], ranges.begin() + first[g + 1]);
    Ctxs.back().first_range = first[g];
  }
  for (Context &c : Ctxs) Keep_batches |= c.ranges.size() > 1;
  if (ranges.size() > 1) {
    cerr << "Database staged in " << ranges.size() << " minimizer ranges over " << Ctxs.size()
         << (Ctxs.size() == 1 ? " context" : " contexts") << " (batches kept: " << (Keep_batches ? "yes" : "no") << ")" << endl;
    // one taxid numbering for every range: the values of all records (as classify -x numbers them).  Each context stages
    // its ranges last to first, so that its first range stays staged for the pass that reads the library.
    vector<vector<uint32_t>> seen(Ctxs.size());
    on_contexts([&](Context &c) {
      vector<uint32_t> &all = seen[&c - Ctxs.data()];
      for (size_t r = c.ranges.size(); r-- > 0 && !c.code;) {
        stage(c, kdb, idx, c.ranges[r]);
        uint32_t m = 0;
        if (c.code) break;
        kuq_db_taxids(c.ctx, NULL, NULL, 0, &m);
        vector<uint32_t> t(m);
        if (m && kuq_db_taxids(c.ctx, t.data(), NULL, m, &m)) c.fail(EX_SOFTWARE, kuq_last_error(c.ctx));
        all.insert(all.end(), t.begin(), t.end());
      }
    });
    vector<uint32_t> all;
    for (auto &v : seen) all.insert(all.end(), v.begin(), v.end());
    sort(all.begin(), all.end());
    all.erase(unique(all.begin(), all.end()), all.end());
    for (Context &c : Ctxs)
      if (kuq_set_db_taxid_universe(c.ctx, all.data(), (uint32_t)all.size())) die(EX_SOFTWARE, kuq_last_error(c.ctx), TOOL);
  } else {
    on_contexts([&](Context &c) { stage(c, kdb, idx, c.ranges[0]); });
  }
  unordered_map<string, uint32_t> id_to_taxon;
  if (one_fasta_file) id_to_taxon = read_seqid_map(ID_to_taxon_map_filename);   // may add taxa
  {
    vector<uint32_t> ids, parents;                        // Parent_map, new taxa included
    for (auto &kv : Taxa) {
      if (kv.first == 0) continue;
      ids.push_back(kv.first);
      parents.push_back(parent_map(kv.first));
    }
    for (Context &c : Ctxs)
      if (kuq_set_taxonomy(c.ctx, ids.data(), parents.data(), (uint32_t)ids.size())) die(EX_SOFTWARE, kuq_last_error(c.ctx), TOOL);
  }

  Batch batch;
  if (one_fasta_file) {                                   // process_single_file, set_lcas.cpp:272-386
    Fasta reader(Multi_fasta_filename);
    const string prefix = "kraken:taxid|";
    uint32_t seqs_processed = 0, seqs_skipped = 0, seqs_no_taxid = 0;
    string id, header, seq;
    while (reader.valid) {
      if (!reader.next(id, header, seq)) break;
      if (seq.empty()) { ++seqs_skipped; continue; }
      uint32_t taxid = 0;
      auto it = id_to_taxon.find(id);
      if (it != id_to_taxon.end()) {
        taxid = it->second;
      } else {                                            // "NC_0001.2" → "NC_0001", :297-313
        size_t pos = id.find_last_of('.');
        bool num = pos != string::npos;
        for (size_t i = pos + 1; num && i < id.size(); ++i) num = isdigit((unsigned char)id[i]) != 0;
        if (num) {
          it = id_to_taxon.find(id.substr(0, pos));
          if (it != id_to_taxon.end()) taxid = it->second;
        }
      }
      if (taxid == 0 && id.size() >= prefix.size() && id.compare(0, prefix.size(), prefix) == 0) {   // :315-323
        taxid = (uint32_t)strtol(id.c_str() + prefix.size(), NULL, 10);
        if (taxid == 0) cerr << "Error: taxonomy ID is zero for sequence '" << id << "'?!" << endl;
        const size_t begin = header.find_first_not_of("\t ");
        if (begin != string::npos) header = header.substr(begin);
      }
      if (taxid == 0) {
        cerr << "Error! Didn't find taxonomy ID mapping for sequence " << id << "!!" << endl;
        ++seqs_skipped;
        continue;
      }
      if (Minimum_sequence_size > 0 && seq.size() < Minimum_sequence_size) {
        cerr << "Skipping sequence " << id << " as it's too short (" << seq.size() << ")" << endl;
        ++seqs_skipped;
        continue;
      }
      if (taxid == 0 || !Taxa.count(taxid)) {             // :336-341
        cerr << "Skipping sequence " << id << " since taxonomy ID " << taxid << " is not in taxonomy database!" << endl;
        ++seqs_skipped;
        continue;
      }
      if (Add_taxids_for_sequences) {                     // the taxon is named after the header line, :344-353
        const uint32_t par = parent_map(taxid);
        if (taxid != TID_HUMAN && par != TID_HUMAN && taxid != TID_MOUSE && par != TID_MOUSE) Taxa.at(taxid).name = header;
      }
      add_sequence(batch, seq, taxid);                    // -T tests the mapped taxid, :344
      ++seqs_processed;
      cerr << "\rProcessed " << seqs_processed << " sequences";
    }
    flush(batch);
    cerr << "\r                                                                            ";
    cerr << "\rFinished processing " << seqs_processed << " sequences (skipping " << seqs_skipped
         << " empty sequences, and " << seqs_no_taxid << " sequences with no taxonomy mapping)" << endl;
  } else {                                                // process_files, :388-411: one single-FASTA file per line
    cerr << "Processing files in " << File_to_taxon_map_filename << endl;
    ifstream map_file(File_to_taxon_map_filename.c_str());
    if (map_file.rdstate() & ifstream::failbit) die(EX_NOINPUT, "can't open " + File_to_taxon_map_filename, TOOL);
    string line;
    uint32_t seqs_processed = 0;
    while (map_file.good()) {
      getline(map_file, line);
      if (line.empty()) break;
      string filename;
      uint32_t taxid = 0;
      istringstream iss(line);
      iss >> filename;
      iss >> taxid;
      Fasta reader(filename);
      string id, header, seq;
      reader.next(id, header, seq);                       // the first sequence only, :414-421
      if (taxid == 0 || !Taxa.count(taxid))
        cerr << "Skipping " << filename << " since taxonomy ID " << taxid << " is not in taxonomy database!" << endl;
      else
        add_sequence(batch, seq, taxid);
      cerr << "\rProcessed " << ++seqs_processed << " sequences";
    }
    flush(batch);
    cerr << "\r                                                       ";
    cerr << "\rFinished processing " << seqs_processed << " sequences" << endl;
  }
  // each context writes its ranges' records into the one image and counts their values (count_taxons,
  // krakendb.cpp:90-113) on the device; contexts with further ranges replay the same batches in the same order against
  // each of them
  vector<char> out((const char *)kdb.p, (const char *)kdb.p + kdb.size);
  const bool want_counts = !Kmer_count_filename.empty();
  vector<map<uint32_t, uint64_t>> counts(Ctxs.size());
  vector<double> count_s(Ctxs.size(), 0);
  mutex progress;
  on_contexts([&](Context &c) {
    const size_t g = &c - Ctxs.data();
    for (size_t r = 0; r < c.ranges.size() && !c.code; r++) {
      if (r) {
        stage(c, kdb, idx, c.ranges[r]);
        for (size_t b = 0; b < Kept.size() && !c.code; b++) {
          lca_batch(c, Kept[b]);
          if (c.batch_missing && !Allow_extra_kmers) c.fail(EX_DATAERR, "kmer found in sequence that is not in database");
        }
        if (c.code) break;
      }
      if (kuq_export_db_values(c.ctx, out.data(), out.size())) c.fail(EX_SOFTWARE, kuq_last_error(c.ctx));
      if (want_counts && !c.code) {
        const auto t0 = chrono::steady_clock::now();
        add_value_counts(c, counts[g]);
        count_s[g] += chrono::duration<double>(chrono::steady_clock::now() - t0).count();
      }
      if (r) {
        lock_guard<mutex> hold(progress);
        cerr << "Finished minimizer range " << (c.first_range + r + 1) << " of " << ranges.size() << endl;
      }
    }
  });
  for (Context &c : Ctxs) Missing_total += c.missing;
  if (verbose && Missing_total) cerr << Missing_total << " k-mers of the library are not in the database" << endl;
  if (want_counts) {                                      // count_taxons → :141-150, in ascending taxid order
    cerr << "Writing kmer counts to " << Kmer_count_filename << "..." << endl;
    map<uint32_t, uint64_t> all;
    double secs = 0;
    for (size_t g = 0; g < Ctxs.size(); g++) {
      for (auto &kv : counts[g]) all[kv.first] += kv.second;
      secs += count_s[g];
    }
    if (getenv("KUQ_TIMING")) cerr << "[timing] value counts " << secs << " s" << endl;
    ofstream ofs(Kmer_count_filename.c_str());
    for (auto &kv : all) ofs << kv.first << '\t' << kv.second << '\n';
  }
  if (!Pretend) {
    // the reference rewrites the memory-mapped input (or the RAM copy under -M) and, with -o, copies it there
    // (:152-169); the net effect with -o is that the OUTPUT holds the new values — and, without -M, so does the input
    const string target = (!Output_DB_filename.empty() && Operate_in_RAM) ? Output_DB_filename : DB_filename;
    if (Operate_in_RAM) cerr << "Writing database from RAM back to " << target << " ..." << endl;
    write_file(target, out.data(), out.size(), TOOL);
    if (!Output_DB_filename.empty() && !Operate_in_RAM) write_file(Output_DB_filename, out.data(), out.size(), TOOL);
  }
  if ((Add_taxids_for_sequences || Add_taxids_for_assembly) && !Pretend) {   // the taxDB is rewritten in place, :171-177
    cerr << "Writing new TaxDB ..." << endl;
    write_taxdb(TaxDB_filename);
  }
  for (Context &c : Ctxs) kuq_destroy(c.ctx);
  return 0;
}
#endif
