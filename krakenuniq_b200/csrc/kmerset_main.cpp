// Drop-in for the Jellyfish 1 call in step 1 of build_db.sh (scripts/build_db.sh:131-132):
//     kmer_set count -m K -s SIZE -C -t N -o PREFIX FILE...
// writes PREFIX_0, which build_db.sh then moves to database.jdb (:138-140), so that
//     krakenuniq-build --jellyfish-bin <this executable> ...
// builds the k-mer set on the GPU (kuq_kmer_set_* of libkuq).  The records are those of `jellyfish count -C` — every
// distinct canonical k-mer with its count — but in ascending key order instead of hash order.  -s and -t are accepted
// and ignored (pass --jellyfish-hash-size to krakenuniq-build to skip its count_unique pass).  Inputs are read
// sequentially (they may be pipes, like build_db.sh's <( cat_library )); several files form one record stream.
#include <fcntl.h>
#include <getopt.h>
#include <sysexits.h>
#include <unistd.h>

#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <iostream>
#include <string>
#include <vector>

#include "../../include/kuq.h"
#include "kuq_dbfile.h"

using namespace std;

static const char *TOOL = "kmer_set";
static const char *VERSION_LINE = "kmer_set 1.1.11 (the `count -C` interface of jellyfish 1, on the GPU with libkuq)";

[[noreturn]] static void die(int code, const string &msg) {
  cerr << TOOL << ": " << msg << endl;
  exit(code);
}

[[noreturn]] static void usage(int code = EX_USAGE) {
  cerr << "Usage: kmer_set count -m K -s SIZE[kKmMgG] -C|--both-strands [-t N] -o PREFIX FILE...\n"
       << "       kmer_set --version\n"
       << "Writes PREFIX_0: every distinct canonical K-mer (K = 1..31) of the FASTA files with its count, in ascending\n"
       << "key order.  -s and -t are accepted and ignored.  KUQ_KMER_SET_BUDGET (bytes of HBM), KUQ_KMER_SET_BATCH\n"
       << "(bases per batch) and KUQ_DEVICE tune the run.\n";
  exit(code);
}

static bool parse_size(const char *s) {       // jellyfish's -s: a number with an optional k/M/G suffix
  char *end = nullptr;
  const unsigned long long v = strtoull(s, &end, 10);
  if (end == s) return false;
  if (*end && strchr("kKmMgG", *end)) end++;
  return *end == 0 && v > 0;
}

// FASTA records in FastaReader::next_sequence form (seqreader.cpp:34-79): a '>' line opens a record, the following
// lines are its sequence, '\r' of CRLF files included (kuq_kmer_set_add treats it as KmerScanner does).  Sequences go to
// the k-mer set in batches.
struct Feeder {
  kuq_kmer_set *h = nullptr;
  string bases;
  vector<uint64_t> offs{0};
  bool open_record = false;
  uint64_t n_records = 0, n_bases = 0;
  double add_s = 0;                                       // time inside kuq_kmer_set_add (staging copies, waits)
  static const uint64_t BATCH = 64ull << 20;

  void submit() {
    const auto t = chrono::steady_clock::now();
    if (offs.size() > 1 && kuq_kmer_set_add(h, bases.data(), offs.data(), (uint32_t)(offs.size() - 1)))
      die(EX_SOFTWARE, kuq_kmer_set_last_error(h));
    add_s += chrono::duration<double>(chrono::steady_clock::now() - t).count();
    bases.clear();
    offs.assign(1, 0);
  }
  void end_record() {
    if (!open_record) return;
    offs.push_back(bases.size());
    open_record = false;
    if (bases.size() >= BATCH || offs.size() > (1u << 20)) submit();
  }
  void line(const char *p, size_t n, const string &path, bool first_line) {
    if (n && p[0] == '>') {
      end_record();
      open_record = true;
      n_records++;
      return;
    }
    if (!open_record) {
      if (first_line && n && p[0] == '@') die(EX_DATAERR, path + ": FASTQ input is not supported (FASTA only)");
      die(EX_DATAERR, path + ": malformed fasta file - expected header char > not found");
    }
    bases.append(p, n);
    n_bases += n;
  }
  // whole file, sequentially (no mmap, no seek: the input may be a pipe)
  void read_file(const string &path) {
    int fd = ::open(path.c_str(), O_RDONLY);
    if (fd < 0) die(EX_NOINPUT, "can't open " + path);
    vector<char> buf(16 << 20);
    string partial;
    bool first = true;
    for (;;) {
      const ssize_t got = ::read(fd, buf.data(), buf.size());
      if (got < 0) die(EX_IOERR, "error reading " + path);
      if (got == 0) break;
      const char *p = buf.data(), *end = p + got;
      while (p < end) {
        const char *nl = (const char *)memchr(p, '\n', end - p);
        if (!nl) { partial.append(p, end - p); break; }
        if (!partial.empty()) {
          partial.append(p, nl - p);
          line(partial.data(), partial.size(), path, first);
          partial.clear();
        } else {
          line(p, nl - p, path, first);
        }
        first = false;
        p = nl + 1;
      }
    }
    if (!partial.empty()) line(partial.data(), partial.size(), path, first);
    ::close(fd);
    end_record();                                         // a record never continues into the next file
  }
};

int main(int argc, char **argv) {
  if (argc > 1 && (strcmp(argv[1], "--version") == 0 || strcmp(argv[1], "-V") == 0)) {
    cout << VERSION_LINE << endl;
    return 0;
  }
  if (argc > 1 && (strcmp(argv[1], "-h") == 0 || strcmp(argv[1], "--help") == 0)) usage(0);
  if (argc < 2 || strcmp(argv[1], "count") != 0) usage();
  int k = 0;
  bool both = false;
  string prefix = "mer_counts";
  static const option longopts[] = {{"mer-len", required_argument, 0, 'm'}, {"size", required_argument, 0, 's'},
                                    {"both-strands", no_argument, 0, 'C'},  {"threads", required_argument, 0, 't'},
                                    {"output", required_argument, 0, 'o'},  {"help", no_argument, 0, 'h'},
                                    {0, 0, 0, 0}};
  optind = 2;
  int opt;
  while ((opt = getopt_long(argc, argv, "m:s:Ct:o:h", longopts, nullptr)) != -1) {
    switch (opt) {
      case 'm': {
        char *end = nullptr;
        const long v = strtol(optarg, &end, 10);
        if (end == optarg || *end || v < 1 || v > 31) die(EX_USAGE, string("k-mer length must be 1..31, got ") + optarg);
        k = (int)v;
        break;
      }
      case 's':
        if (!parse_size(optarg)) die(EX_USAGE, string("invalid hash size ") + optarg);
        break;
      case 'C': both = true; break;
      case 't':
        if (atoll(optarg) <= 0) die(EX_USAGE, "can't use nonpositive thread count");
        break;
      case 'o': prefix = optarg; break;
      case 'h': usage(0);
      default: usage();
    }
  }
  if (!k) die(EX_USAGE, "-m K is required");
  if (!both) die(EX_USAGE, "only canonical counting (-C / --both-strands) is supported, as KrakenUniq needs it");
  if (optind >= argc) die(EX_USAGE, "no input file");
  vector<string> inputs(argv + optind, argv + argc);

  const auto t0 = chrono::steady_clock::now();
  const int dev = getenv("KUQ_DEVICE") ? atoi(getenv("KUQ_DEVICE")) : 0;
  char err[1024] = "";
  Feeder f;
  int rc = kuq_kmer_set_create(dev, (uint32_t)k, 0, &f.h, err, sizeof err);
  if (rc) die(rc == KUQ_E_NO_DEVICE ? EX_UNAVAILABLE : EX_SOFTWARE, err[0] ? err : kuq_strerror(rc));
  const auto t1 = chrono::steady_clock::now();
  for (const string &path : inputs) f.read_file(path);
  f.submit();
  const double input_s = chrono::duration<double>(chrono::steady_clock::now() - t1).count();

  // header (SURVEY App. A16): JFLISTDN, key_bits = 2k, val_len = 4, key_ct at byte 48, every other byte zero
  const uint64_t key_bits = 2 * (uint64_t)k, key_len = kdb_key_len(key_bits), rec = key_len + 4;
  vector<char> header(kdb_header_bytes(key_bits), 0);
  memcpy(header.data(), "JFLISTDN", 8);
  const uint64_t val_len = 4;
  memcpy(header.data() + 8, &key_bits, 8);
  memcpy(header.data() + 16, &val_len, 8);
  const string out_path = prefix + "_0", tmp_path = out_path + ".tmp" + to_string(getpid());
  FILE *out = fopen(tmp_path.c_str(), "wb");
  if (!out) die(EX_CANTCREAT, "can't write " + tmp_path);
  auto fail = [&](int code, const string &msg) {
    fclose(out);
    unlink(tmp_path.c_str());
    die(code, msg);
  };
  if (fwrite(header.data(), 1, header.size(), out) != header.size()) fail(EX_IOERR, "error writing " + tmp_path);
  const uint64_t cap = 1ull << 22;
  vector<char> recs(cap * rec);
  for (;;) {
    uint64_t n = 0;
    rc = kuq_kmer_set_next(f.h, recs.data(), cap, &n);
    if (rc) fail(EX_SOFTWARE, kuq_kmer_set_last_error(f.h));
    if (!n) break;
    if (fwrite(recs.data(), rec, n, out) != n) fail(EX_IOERR, "error writing " + tmp_path);
  }
  uint64_t key_ct = 0;
  uint32_t passes = 0;
  if (kuq_kmer_set_info(f.h, &key_ct, &passes)) fail(EX_SOFTWARE, kuq_kmer_set_last_error(f.h));
  memcpy(header.data() + 48, &key_ct, 8);
  if (fseek(out, 0, SEEK_SET) || fwrite(header.data(), 1, header.size(), out) != header.size() || fclose(out))
    die(EX_IOERR, "error writing " + tmp_path);
  if (rename(tmp_path.c_str(), out_path.c_str())) {
    unlink(tmp_path.c_str());
    die(EX_CANTCREAT, "can't rename " + tmp_path + " to " + out_path);
  }
  kuq_kmer_set_destroy(f.h);
  const double s = chrono::duration<double>(chrono::steady_clock::now() - t0).count();
  cerr << TOOL << ": " << f.n_records << " sequences, " << f.n_bases << " bases, " << key_ct << " distinct " << k
       << "-mers, " << passes << (passes == 1 ? " pass, " : " passes, ") << s << " s (input " << input_s
       << " s, of which parsing " << input_s - f.add_s << " s)" << endl;
  return 0;
}
