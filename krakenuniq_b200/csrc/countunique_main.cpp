// Drop-in for count_unique (src/count_unique.cpp), which krakenuniq-build runs to size Jellyfish's hash when
// --jellyfish-hash-size is not given (scripts/build_db.sh:125-129):
//     count_unique [-k K] [-t N] [-p P] < library
// prints the HyperLogLog estimate of the library's distinct forward k-mers at precision P, computed on the GPU
// (kuq_count_unique_* of libkuq).  stdin may be plain FASTA or gzip.  -t is checked as the reference checks it and
// otherwise ignored.  One difference: a precision outside 4..18 makes the reference abort on an uncaught exception;
// this tool prints the same message and exits EX_USAGE, before it reads stdin or touches a device.
#include <err.h>
#include <sched.h>
#include <sysexits.h>
#include <unistd.h>
#include <zlib.h>

#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <iostream>
#include <string>
#include <vector>

#include "../../include/kuq.h"

using namespace std;

static int K = 31, Hll_precision = 14, Num_threads = 1;

[[noreturn]] static void usage(int code = EX_USAGE) {
  cerr << "Usage: count-unique [options]" << endl
       << "  Estimate the number of k-mer in stdin using HLL." << endl
       << "Options: " << endl
       << "  -k #          Length of k-mers [" << K << "]" << endl
       << "  -t #          Number of threads [" << Num_threads << "]" << endl
       << "  -p INT        HLL precision [" << Hll_precision << "]" << endl
       << "  -h            Print this message" << endl;
  exit(code);
}

// count_unique.cpp:81-122; -t is bounded by the processors this process may run on, as omp_get_num_procs counts them
static void parse_command_line(int argc, char **argv) {
  if (argc > 1 && strcmp(argv[1], "-h") == 0) usage(0);
  int opt;
  long long sig;
  while ((opt = getopt(argc, argv, "t:k:m:p:")) != -1) {
    switch (opt) {
      case 't': {
        sig = atoll(optarg);
        if (sig <= 0) errx(EX_USAGE, "can't use nonpositive thread count");
        cpu_set_t set;
        const long procs = sched_getaffinity(0, sizeof set, &set) == 0 ? CPU_COUNT(&set) : sysconf(_SC_NPROCESSORS_ONLN);
        if (sig > procs) errx(EX_USAGE, "thread count exceeds number of processors");
        Num_threads = (int)sig;
        break;
      }
      case 'k':
        sig = atoll(optarg);
        if (sig <= 0) errx(EX_USAGE, "k can't be <= 0");
        if (sig > 31) errx(EX_USAGE, "k can't be > 31");
        K = (int)sig;
        break;
      case 'p': Hll_precision = atoi(optarg); break;
      default: usage();
    }
  }
}

// FastaReader::next_sequence (seqreader.cpp:34-79) over stdin: the first line must open a record with '>' (else the
// reader warns and stops), each following '>' line opens the next, and every other line is appended to the open
// record's sequence ('\r' of CRLF lines included).  Records go to the sketch in batches.
struct Feeder {
  kuq_count_unique *h = nullptr;
  string bases;
  vector<uint64_t> offs{0};
  bool open_record = false, stopped = false;
  double add_s = 0;                                      // time inside kuq_count_unique_add
  uint64_t n_records = 0, n_bases = 0;
  static const uint64_t BATCH = 64ull << 20;

  void submit() {
    const auto t = chrono::steady_clock::now();
    if (offs.size() > 1 && kuq_count_unique_add(h, bases.data(), offs.data(), (uint32_t)(offs.size() - 1)))
      errx(EX_SOFTWARE, "%s", kuq_count_unique_last_error(h));
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
  void line(const char *p, size_t n, bool first) {
    if (n && p[0] == '>') {
      end_record();
      open_record = true;
      n_records++;
      return;
    }
    if (first) {
      warnx("malformed fasta file - expected header char > not found");
      stopped = true;
      return;
    }
    bases.append(p, n);
    n_bases += n;
  }
  void read(gzFile in) {
    vector<char> buf(16 << 20);
    string partial;
    bool first = true;
    for (;;) {
      const int got = gzread(in, buf.data(), (unsigned)buf.size());
      if (got < 0) errx(EX_IOERR, "error reading stdin");
      if (got == 0) break;
      const char *p = buf.data(), *end = p + got;
      while (p < end && !stopped) {
        const char *nl = (const char *)memchr(p, '\n', end - p);
        if (!nl) { partial.append(p, end - p); break; }
        if (!partial.empty()) {
          partial.append(p, nl - p);
          line(partial.data(), partial.size(), first);
          partial.clear();
        } else {
          line(p, nl - p, first);
        }
        first = false;
        p = nl + 1;
      }
      if (stopped) break;
    }
    if (!stopped && (first || !partial.empty())) line(partial.data(), partial.size(), first);   // empty input: no '>'
    end_record();
    submit();
  }
};

int main(int argc, char **argv) {
  parse_command_line(argc, argv);
  // HyperLogLogPlusMinus takes the precision as uint8_t (hyperloglogplus.cpp:428-433)
  const unsigned p = (uint8_t)Hll_precision;
  if (p < 4 || p > 18) {
    cerr << "precision (number of register = 2^precision) must be between 4 and 18" << endl;
    return EX_USAGE;
  }
  const auto t0 = chrono::steady_clock::now();
  gzFile in = gzdopen(dup(0), "rb");
  if (!in) err(EX_NOINPUT, "can't open /dev/fd/0");
  gzbuffer(in, 1 << 20);
  const int dev = getenv("KUQ_DEVICE") ? atoi(getenv("KUQ_DEVICE")) : 0;
  char msg[1024] = "";
  Feeder f;
  const int rc = kuq_count_unique_create(dev, (uint32_t)K, p, 0, &f.h, msg, sizeof msg);
  if (rc) errx(rc == KUQ_E_NO_DEVICE ? EX_UNAVAILABLE : EX_SOFTWARE, "%s", msg[0] ? msg : kuq_strerror(rc));
  const auto t1 = chrono::steady_clock::now();
  f.read(in);
  gzclose(in);
  uint64_t estimate = 0, n_observed = 0;
  if (kuq_count_unique_result(f.h, &estimate, &n_observed, nullptr)) errx(EX_SOFTWARE, "%s", kuq_count_unique_last_error(f.h));
  cout << estimate << endl;
  if (getenv("KUQ_COUNT_UNIQUE_STATS")) {                // measurement aid: timings on stderr
    double sketch_ms = 0;
    uint64_t windows = 0, bases = 0;
    kuq_count_unique_stats(f.h, &sketch_ms, &windows, &bases);
    const auto t2 = chrono::steady_clock::now();
    fprintf(stderr, "count_unique: %llu sequences, %llu bases, %llu windows, total %.6f s, setup %.6f s, input %.6f s "
            "(parsing %.6f s), sketch kernel %.3f ms\n", (unsigned long long)f.n_records, (unsigned long long)f.n_bases,
            (unsigned long long)windows, chrono::duration<double>(t2 - t0).count(), chrono::duration<double>(t1 - t0).count(),
            chrono::duration<double>(t2 - t1).count(), chrono::duration<double>(t2 - t1).count() - f.add_s, sketch_ms);
  }
  kuq_count_unique_destroy(f.h);
  return 0;
}
