// classify_main.cpp — drop-in `classify` executable over libkuq.so (SURVEY.md §8(b), rows f1/f2).
//
// Same argv, file formats and text outputs as the reference driver (src/classify.cpp:150-346,1068-1189), so that
// scripts/krakenuniq:240-248 can call it unchanged; the per-read work (classify_sequence, :897-1012) happens on the
// GPU behind include/kuq.h.  Host-side pieces restated here, each citing what it mirrors:
//   FASTA/FASTQ readers            src/seqreader.cpp:34-129 (gz through zlib instead of bxzstr)
//   work-unit loop                 src/classify.cpp:506-559 (batches hold whole work units, DESIGN.md §4): kuq_batches.h
//   Kraken output lines            src/classify.cpp:980-1010, hitlist_string :826-861
//   stats / progress lines         src/classify.cpp:361-375, 555-558
//   taxDB reader, genome sizes     src/taxdb.hpp:563-605, 850-885
//   report (clades, sorting, cols) src/taxdb.hpp:928-1123, src/classify.cpp:286-328
//   --paired / --check-names       scripts/read_merger.pl (what scripts/krakenuniq:230-237 runs before classify): the
//                                  mates are merged during the ingest; the one deviation is the exit status, EX_DATAERR
//                                  where the merger stopped at a malformed record or a name mismatch (the wrapper
//                                  ignores the merger's status and exits 0)
//   --extract                      scripts/krakenuniq-extract-reads run on our Kraken lines and inputs: the reads of the
//                                  chosen taxa are written while the batch is formatted (INTEGRATION.md)
//   --mpa-report / --translate-out scripts/krakenuniq-mpa-report and scripts/krakenuniq-translate run on our Kraken
//                                  lines: booked while the batch is formatted, the table written after the last sample
//   --sample-sheet                 no counterpart: one process stages the database(s) once and classifies every row of
//                                  the sheet as a separate run would, with kuq_reset_counts between the samples; a
//                                  streamed database's passes are shared among the rows (classify_streamed)
// Not supported (exit with a message): -I uid mapping, -x together with several -d databases (the reference's own loop
// for that combination queries database 0 in every pass, classify.cpp:585-632).
#include <fcntl.h>
#include <getopt.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <sys/time.h>
#include <sysexits.h>
#include <unistd.h>
#include <zlib.h>

#include <dlfcn.h>
#include <omp.h>
#include <atomic>
#include <condition_variable>
#include <deque>
#include <mutex>
#include <thread>

#include <algorithm>
#include <cinttypes>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <iomanip>
#include <iostream>
#include <map>
#include <memory>
#include <set>
#include <sstream>
#include <string>
#include <unordered_map>
#include <unordered_set>
#include <vector>

#include "../../include/kuq.h"
#include "kuq_batches.h"
#include "kuq_dbfile.h"
#include "kuq_ranges.h"

using namespace std;

static vector<string> DB_filenames, Index_filenames;
static uint32_t Minimum_hit_count = 1;        // -m (classify.cpp:45)
static bool Quick_mode = false, Print_classified = false, Print_unclassified = false, Print_kraken = true;
static bool Populate_memory = false, Only_classified_kraken_output = false, Print_sequence = false, Map_UIDs = false;
static bool Paired = false, Check_names = false;  // --paired / --check-names: argv holds one pair of mate files
static string Pair_error;                         // what read_merger.pl would have died with (the run exits EX_DATAERR)
static string Sample_sheet;                       // --sample-sheet: the samples of the run, each with its own outputs
static string Sample_label;                       // the sample being classified (sheet runs), named in error messages
static bool Filter = false;                       // --threshold: the Kraken lines krakenuniq-filter makes of ours
static double Threshold = 0;
// --extract: the reads krakenuniq-extract-reads [-t taxDB] [-i] [-f] [-p] TAXIDS out.kraken reads would print
static bool Extract = false, Extract_subtree = false, Extract_invert = false, Extract_fasta = false, Extract_others = false;
static bool Extract_now = false;                  // this sample writes an extraction (a sheet row may leave it out)
static string Extract_list, Extract_output_file;
static vector<uint32_t> Extract_taxa;             // the list's decimal taxids ("-1" is Extract_others)
// --mpa-report: one krakenuniq-mpa-report table over the Kraken lines of every sample of the run; --translate-out: the
// lines krakenuniq-translate [--mpa-format] prints from a sample's Kraken lines (both with -a's taxDB)
static bool Mpa = false, Mpa_show_zeros = false, Mpa_header_line = false, Mpa_intermediate = false, Translate_mpa = false;
static bool Translate_now = false;                // this sample writes a translation (a sheet row may leave it out)
static string Mpa_output_file, Translate_output_file;
static uint64_t Populate_memory_size = 0;
static string Classified_output_file, Unclassified_output_file, Kraken_output_file, Report_output_file, TaxDB_file;
static size_t Work_unit_size = 500000;      // DEF_WORK_UNIT_SIZE, classify.cpp:38
// Preloaded runs: a batch closes at a unit boundary once it holds this many work units, the rows of the library's dense
// (unit, taxon) table (kuq_unit_table_rows).  The per-batch hash map then only holds candidate pairs (at most one per
// 1025 bases), far below its 2 Mi pairs whatever the units hit.  Small -u with tens of thousands of taxa gives smaller
// batches; everything else is cut by size first.
static size_t Max_units_per_batch = SIZE_MAX;
static int Num_threads = 1;
static int HLL_PRECISION = 14;              // readcounts.hpp:29 (only selects report columns, classify.cpp:289)
static unsigned long long total_classified = 0, total_sequences = 0, total_bases = 0;

[[noreturn]] static void die(int code, const string &msg) {
  cerr << "classify: " << (Sample_label.empty() ? "" : "sample " + Sample_label + ": ") << msg << endl;
  exit(code);
}

static void usage(int exit_code = EX_USAGE) {
  cerr << "Usage: classify [options] <fasta/fastq file(s)>" << endl
       << endl
       << "Options: (*mandatory)" << endl
       << "* -d filename      Kraken DB filename" << endl
       << "* -i filename      Kraken DB index filename" << endl
       << "  -o filename      Output file for Kraken output" << endl
       << "  -r filename      Output file for Kraken report output" << endl
       << "  -a filename      TaxDB" << endl
       << "  -I filename      UID to TaxId map" << endl
       << "  -p #             Precision for unique k-mer counting, between 10 and 18" << endl
       << "  -t #             Number of threads" << endl
       << "  -u #             Thread work unit size (in bp)" << endl
       << "  -q               Quick operation" << endl
       << "  -m #             Minimum hit count (ignored w/o -q)" << endl
       << "  -C filename      Print classified sequences" << endl
       << "  -U filename      Print unclassified sequences" << endl
       << "  -c               Only include classified reads in output" << endl
       << "  -M               Preload database files" << endl
       << "  -x size          Preload database files using x amount of RAM (e.g. 10G)" << endl
       << "  -s               Print read sequence in Kraken output" << endl
       << "  --paired         The two files are mates of paired-end reads: each pair is classified as one" << endl
       << "                   sequence mate1 + 'N' + mate2, named after mate 1 (what read_merger.pl writes)" << endl
       << "  --check-names    With --paired: stop at the first pair whose names differ (exit status 65)" << endl
       << "  --sample-sheet f Classify every sample of the tab-separated sheet f against one staging of the database:" << endl
       << "                   columns input (files separated by ','), input2 (the mates, with --paired), output," << endl
       << "                   report, classified_out, unclassified_out (as -o -r -C -U; empty = not written), name" << endl
       << "  --threshold T    Write the Kraken lines that krakenuniq-filter --threshold T makes of them: each call moves" << endl
       << "                   up the taxonomy until a fraction T of the read's unambiguous k-mers lies in the clade," << endl
       << "                   with that fraction as a P= column (-a's taxDB is the filter's taxonomy)" << endl
       << "  --extract L      Write the reads that krakenuniq-extract-reads L <Kraken output> <input> prints: L is a" << endl
       << "                   comma-separated taxid list (-1 = every other line, 0 = unclassified), to --extract-out f" << endl
       << "                   ('-' = stdout, .gz = gzip; a --sample-sheet column extract_out instead)" << endl
       << "  --extract-subtree  with the children of the taxa in -a's taxDB (the script's -t)" << endl
       << "  --extract-invert   every read not selected (-i)       --extract-fasta  FASTQ reads as FASTA (-f)" << endl
       << "  --mpa-report f   Write the table krakenuniq-mpa-report prints from the Kraken lines to f, one count column" << endl
       << "                   per sample ('-' = stdout, .gz = gzip; needs -a; a --sample-sheet writes one table)" << endl
       << "  --mpa-show-zeros, --mpa-header-line, --mpa-intermediate-ranks   the script's --show-zeros," << endl
       << "                   --header-line (sample ids = the Kraken output files) and --intermediate-ranks" << endl
       << "  --translate-out f  Write what krakenuniq-translate prints from the Kraken lines (read id, lineage) to f" << endl
       << "                   ('-' = stdout, .gz = gzip; needs -a; a --sample-sheet column translate_out instead)" << endl
       << "  --translate-mpa-format  lineages in the script's --mpa-format" << endl
       << "  -h              Print this message" << endl
       << endl
       << "Kraken output is to standard output by default." << endl;
  exit(exit_code);
}

static vector<string> split(const string &s, char sep) {
  vector<string> v;
  for (size_t a = 0;;) {
    const size_t b = s.find(sep, a);
    v.push_back(s.substr(a, b == string::npos ? string::npos : b - a));
    if (b == string::npos) return v;
    a = b + 1;
  }
}

// parse_human_readable_size, krakenutil.cpp:30-55
static uint64_t parse_human_readable_size(const char *s) {
  char *endp = NULL;
  errno = 0;
  uint64_t x = strtoumax(s, &endp, 10);
  if (errno || endp == s) return 0;
  int sh;
  switch (*endp) {
    case 'k': case 'K': sh = 10; break;
    case 'm': case 'M': sh = 20; break;
    case 'g': case 'G': sh = 30; break;
    case 0: sh = 0; break;
    default: return 0;
  }
  if (x > SIZE_MAX >> sh) return 0;
  return x << sh;
}

static void parse_command_line(int argc, char **argv) {
  int opt;
  long long sig;
  if (argc > 1 && strcmp(argv[1], "-h") == 0) usage(0);
  enum { OPT_PAIRED = 256, OPT_CHECK_NAMES, OPT_SAMPLE_SHEET, OPT_THRESHOLD, OPT_EXTRACT, OPT_EXTRACT_OUT, OPT_EXTRACT_SUBTREE,
         OPT_EXTRACT_INVERT, OPT_EXTRACT_FASTA, OPT_MPA_REPORT, OPT_MPA_SHOW_ZEROS, OPT_MPA_HEADER_LINE, OPT_MPA_INTERMEDIATE,
         OPT_TRANSLATE_OUT, OPT_TRANSLATE_MPA };
  static const struct option long_opts[] = {{"paired", no_argument, NULL, OPT_PAIRED},
                                            {"check-names", no_argument, NULL, OPT_CHECK_NAMES},
                                            {"sample-sheet", required_argument, NULL, OPT_SAMPLE_SHEET},
                                            {"threshold", required_argument, NULL, OPT_THRESHOLD},
                                            {"extract", required_argument, NULL, OPT_EXTRACT},
                                            {"extract-out", required_argument, NULL, OPT_EXTRACT_OUT},
                                            {"extract-subtree", no_argument, NULL, OPT_EXTRACT_SUBTREE},
                                            {"extract-invert", no_argument, NULL, OPT_EXTRACT_INVERT},
                                            {"extract-fasta", no_argument, NULL, OPT_EXTRACT_FASTA},
                                            {"mpa-report", required_argument, NULL, OPT_MPA_REPORT},
                                            {"mpa-show-zeros", no_argument, NULL, OPT_MPA_SHOW_ZEROS},
                                            {"mpa-header-line", no_argument, NULL, OPT_MPA_HEADER_LINE},
                                            {"mpa-intermediate-ranks", no_argument, NULL, OPT_MPA_INTERMEDIATE},
                                            {"translate-out", required_argument, NULL, OPT_TRANSLATE_OUT},
                                            {"translate-mpa-format", no_argument, NULL, OPT_TRANSLATE_MPA}, {NULL, 0, NULL, 0}};
  while ((opt = getopt_long(argc, argv, "d:i:t:u:n:m:o:qcC:U:Ma:r:sI:p:x:", long_opts, NULL)) != -1) {
    switch (opt) {
      case OPT_PAIRED: Paired = true; break;
      case OPT_CHECK_NAMES: Check_names = true; break;           // ignored without --paired (krakenuniq:281-283)
      case OPT_SAMPLE_SHEET: Sample_sheet = optarg; break;
      case OPT_THRESHOLD: {
        char *end = NULL;
        Threshold = strtod(optarg, &end);
        if (end == optarg || *end) die(EX_USAGE, string("--threshold: not a number: '") + optarg + "'");
        if (!(Threshold >= 0 && Threshold <= 1)) die(EX_USAGE, "threshold must be in the interval [0,1].");   // krakenuniq-filter:55-58
        Filter = true;
        break;
      }
      case OPT_EXTRACT: Extract = true; Extract_list = optarg; break;
      case OPT_EXTRACT_OUT: Extract_output_file = optarg; break;
      case OPT_EXTRACT_SUBTREE: Extract_subtree = true; break;
      case OPT_EXTRACT_INVERT: Extract_invert = true; break;
      case OPT_EXTRACT_FASTA: Extract_fasta = true; break;
      case OPT_MPA_REPORT: Mpa = true; Mpa_output_file = optarg; break;
      case OPT_MPA_SHOW_ZEROS: Mpa_show_zeros = true; break;
      case OPT_MPA_HEADER_LINE: Mpa_header_line = true; break;
      case OPT_MPA_INTERMEDIATE: Mpa_intermediate = true; break;
      case OPT_TRANSLATE_OUT: Translate_output_file = optarg; break;
      case OPT_TRANSLATE_MPA: Translate_mpa = true; break;
      case 'd': DB_filenames.push_back(optarg); break;
      case 'i': Index_filenames.push_back(optarg); break;
      case 't':
        sig = atoll(optarg);
        if (sig <= 0) die(EX_USAGE, "can't use nonpositive thread count");
        if (sig > omp_get_num_procs()) die(EX_USAGE, "thread count exceeds number of processors");   // classify.cpp:1087-1088
        Num_threads = (int)sig;                  // host threads: parallel FASTA/FASTQ parsing and text formatting
        break;
      case 'p': HLL_PRECISION = atoi(optarg); break;
      case 'q': Quick_mode = true; break;
      case 'm':
        sig = atoll(optarg);
        if (sig <= 0) die(EX_USAGE, "can't use nonpositive minimum hit count");
        Minimum_hit_count = (uint32_t)sig;
        break;
      case 'c': Only_classified_kraken_output = true; break;
      case 'C': Print_classified = true; Classified_output_file = optarg; break;
      case 'U': Print_unclassified = true; Unclassified_output_file = optarg; break;
      case 'o': Kraken_output_file = optarg; break;
      case 'r': Report_output_file = optarg; break;
      case 's': Print_sequence = true; break;
      case 'a': TaxDB_file = optarg; break;
      case 'u':
        sig = atoll(optarg);
        if (sig <= 0) die(EX_USAGE, "can't use nonpositive work unit size");
        Work_unit_size = sig;
        break;
      case 'M': Populate_memory = true; break;
      case 'x': Populate_memory = true; Populate_memory_size = parse_human_readable_size(optarg); break;
      case 'I': Map_UIDs = true; break;
      default: usage(); break;
    }
  }
  // the filter keeps five columns of a Kraken line (krakenuniq-filter:131): the sequence column would silently go
  if (Filter && Print_sequence) die(EX_USAGE, "--threshold cannot be combined with -s");
  if (!Extract && (!Extract_output_file.empty() || Extract_subtree || Extract_invert || Extract_fasta))
    die(EX_USAGE, "--extract-out, --extract-subtree, --extract-invert and --extract-fasta need --extract");
  if (Extract) {
    // the script's list (:62): entries compare as strings with the line's decimal taxid, so only canonical decimals
    // can match; "-1" takes every line no other entry matched (:116-118)
    for (const string &e : split(Extract_list, ',')) {
      if (e == "-1") { Extract_others = true; continue; }
      const bool canonical = !e.empty() && e.size() <= 10 && all_of(e.begin(), e.end(), ::isdigit) && (e == "0" || e[0] != '0');
      if (canonical && strtoull(e.c_str(), NULL, 10) <= UINT32_MAX) Extract_taxa.push_back((uint32_t)strtoull(e.c_str(), NULL, 10));
    }
    if (Extract_subtree && TaxDB_file.empty()) die(EX_USAGE, "--extract-subtree takes the children from the taxDB: give it with -a");
    if (!Sample_sheet.empty() && !Extract_output_file.empty())
      die(EX_USAGE, "--sample-sheet takes the extraction's file from the sheet: --extract-out is its column extract_out");
    if (Sample_sheet.empty() && Extract_output_file.empty()) die(EX_USAGE, "--extract needs --extract-out");
  }
  if (!Mpa && (Mpa_show_zeros || Mpa_header_line || Mpa_intermediate))
    die(EX_USAGE, "--mpa-show-zeros, --mpa-header-line and --mpa-intermediate-ranks need --mpa-report");
  if (!Sample_sheet.empty() && !Translate_output_file.empty())
    die(EX_USAGE, "--sample-sheet takes the translation's file from the sheet: --translate-out is its column translate_out");
  if (Sample_sheet.empty() && Translate_mpa && Translate_output_file.empty()) die(EX_USAGE, "--translate-mpa-format needs --translate-out");
  if (DB_filenames.empty()) { cerr << "Missing mandatory option -d" << endl; usage(); }
  if (Index_filenames.empty()) { cerr << "Missing mandatory option -i" << endl; usage(); }
  if (!Sample_sheet.empty()) {                      // the sheet names every sample's inputs and outputs
    if (optind < argc) die(EX_USAGE, "--sample-sheet takes the inputs from the sheet: no input files on the command line");
    if (!Kraken_output_file.empty() || !Report_output_file.empty() || Print_classified || Print_unclassified)
      die(EX_USAGE, "--sample-sheet takes the outputs from the sheet: -o, -r, -C and -U are its columns");
    return;
  }
  if (Paired && argc - optind != 2) die(EX_USAGE, "--paired requires exactly two filenames");   // krakenuniq:160-161
  if (optind == argc && !Populate_memory) cerr << "No sequence data files specified" << endl;
}

// ---- samples: the command line's one, or the rows of --sample-sheet ---------------------------------------------
// A sample's inputs are classified as one run, the inputs of a separate `classify` call: each a file, or with --paired
// a pair of mate files.  The outputs are the values of -o -r -C -U ("" = the option was not given).
struct Sample {
  string name;
  vector<pair<string, string>> inputs;
  string kraken, report, classified, unclassified, extract, translate;
};

static vector<pair<const char *, const char *>> files_of(const Sample &s) {
  vector<pair<const char *, const char *>> in;
  for (auto &f : s.inputs) in.emplace_back(f.first.c_str(), f.second.empty() ? NULL : f.second.c_str());
  return in;
}

// What two paths share when they name one file: device and inode of an existing file, else the absolute path
static string path_key(const string &p) {
  struct stat sb;
  if (stat(p.c_str(), &sb) == 0) return "i" + to_string(sb.st_dev) + ":" + to_string(sb.st_ino);
  const size_t slash = p.rfind('/');
  const string dir = slash == string::npos ? "." : slash == 0 ? "/" : p.substr(0, slash);
  char *real = realpath(dir.c_str(), NULL);
  const string key = "p" + (real ? string(real) : dir) + "/" + p.substr(slash == string::npos ? 0 : slash + 1);
  free(real);
  return key;
}

// The sheet: tab-separated, a header line naming the columns, then one sample per line; blank lines and lines that start
// with '#' are skipped.  Every check runs here, before a database is opened, so a bad sheet writes nothing.
static vector<Sample> read_sample_sheet(const string &path) {
  ifstream in(path);
  if (!in.is_open()) die(EX_NOINPUT, "can't open the sample sheet " + path);
  static const set<string> known = {"input", "input2", "output", "report", "classified_out", "unclassified_out", "name",
                                    "extract_out", "translate_out"};
  map<string, size_t> col;
  vector<Sample> samples;
  map<string, string> written;                     // path_key -> which sample writes it
  set<string> read_keys{path_key(path)};
  string line;
  for (size_t line_no = 1; getline(in, line); line_no++) {
    if (!line.empty() && line.back() == '\r') line.pop_back();
    if (line.empty() || line[0] == '#') continue;
    const vector<string> f = split(line, '\t');
    const string at = path + ":" + to_string(line_no) + ": ";
    if (col.empty()) {
      for (size_t i = 0; i < f.size(); i++) {
        if (!known.count(f[i])) die(EX_USAGE, at + "unknown column '" + f[i] + "' (columns: input input2 output report classified_out unclassified_out name extract_out translate_out)");
        if (!col.emplace(f[i], i).second) die(EX_USAGE, at + "column '" + f[i] + "' named twice");
      }
      if (!col.count("input")) die(EX_USAGE, at + "the header has no input column");
      if (Paired && !col.count("input2")) die(EX_USAGE, at + "--paired needs an input2 column with the second mates");
      if (!Paired && col.count("input2")) die(EX_USAGE, at + "an input2 column needs --paired");
      if (Extract && !col.count("extract_out")) die(EX_USAGE, at + "--extract needs an extract_out column");
      if (!Extract && col.count("extract_out")) die(EX_USAGE, at + "an extract_out column needs --extract");
      if (Translate_mpa && !col.count("translate_out")) die(EX_USAGE, at + "--translate-mpa-format needs a translate_out column");
      continue;
    }
    if (f.size() > col.size()) die(EX_USAGE, at + "more cells than the header has columns");
    auto cell = [&](const char *c) { auto it = col.find(c); return it != col.end() && it->second < f.size() ? f[it->second] : string(); };
    Sample s;
    s.name = cell("name").empty() ? to_string(samples.size() + 1) : cell("name");
    const vector<string> in1 = split(cell("input"), ','), in2 = split(cell("input2"), ',');
    if (cell("input").empty()) die(EX_USAGE, at + "sample " + s.name + " has no input");
    if (Paired && (in1.size() != 1 || in2.size() != 1 || in2[0].empty()))
      die(EX_USAGE, at + "sample " + s.name + ": with --paired, input and input2 each hold one file");
    for (size_t i = 0; i < in1.size(); i++) {
      vector<string> files{in1[i]};
      if (Paired) files.push_back(in2[i]);
      for (const string &p : files) {
        if (p.empty()) die(EX_USAGE, at + "sample " + s.name + ": an empty input file name");
        struct stat sb;
        if (access(p.c_str(), R_OK) != 0 || stat(p.c_str(), &sb) != 0 || S_ISDIR(sb.st_mode))
          die(EX_NOINPUT, at + "sample " + s.name + ": can't read input " + p);
        read_keys.insert(path_key(p));
      }
      s.inputs.emplace_back(in1[i], Paired ? in2[i] : string());
    }
    // an empty cell: that output is not written (-o off); Kraken lines never go to standard output
    s.kraken = cell("output").empty() || cell("output") == "-" ? "off" : cell("output");
    s.report = cell("report");
    s.classified = cell("classified_out");
    s.unclassified = cell("unclassified_out");
    s.extract = cell("extract_out");                // empty: nothing is extracted from this sample
    s.translate = cell("translate_out");            // empty: this sample's reads are not translated
    for (const string *o : {&s.kraken, &s.report, &s.classified, &s.unclassified, &s.extract, &s.translate}) {
      if (o->empty() || *o == "off" || *o == "-") continue;
      auto w = written.emplace(path_key(*o), s.name);
      if (!w.second) die(EX_USAGE, at + "samples " + w.first->second + " and " + s.name + " both write " + *o);
    }
    samples.push_back(s);
  }
  if (col.empty()) die(EX_USAGE, path + ": no header line");
  if (samples.empty()) die(EX_USAGE, path + ": no samples");
  for (auto &w : written)
    if (read_keys.count(w.first)) die(EX_USAGE, "sample " + w.second + " writes to one of the inputs");
  return samples;
}

// ---- output streams: plain file, ".gz" → gzip, "-" → stdout (cout_or_file, classify.cpp:133-148) ---------------
struct OutStream {
  FILE *f = NULL;
  gzFile gz = NULL;
  bool is_stdout = false;
  void open(const string &path, bool append = false) {
    if (path == "-") { f = stdout; is_stdout = true; return; }
    if (path.size() >= 3 && path.compare(path.size() - 3, 3, ".gz") == 0) {
      gz = gzopen(path.c_str(), "wb");
      if (!gz) die(EX_CANTCREAT, "can't open " + path);
    } else {
      f = fopen(path.c_str(), append ? "ab" : "wb");
      if (!f) die(EX_CANTCREAT, "can't open " + path);
    }
  }
  void write(const char *p, size_t n) {
    if (gz) gzwrite(gz, p, (unsigned)n);
    else if (f) fwrite(p, 1, n, f);
  }
  void write(const string &s) { write(s.data(), s.size()); }
  void close() {
    if (gz) gzclose(gz);
    else if (f && !is_stdout) fclose(f);
    else if (f) fflush(f);
    f = NULL; gz = NULL;
  }
};

// ---- input: FASTA / FASTQ through zlib (plain or gzip), semantics of src/seqreader.cpp -------------------------
struct Read {
  string header_line, quals;
  uint64_t seq_off, seq_len;          // into the batch's bases buffer
};

// bzip2 input (the reference reads it through bxzstr when built with libbz2, seqreader.hpp:24,48).  The image has the
// runtime library but not its header, so the three entry points of the high-level API are bound with dlopen.
struct Bz2Api {
  void *(*open)(const char *, const char *) = NULL;
  int (*read)(void *, void *, int) = NULL;
  void (*close)(void *) = NULL;
  bool load() {
    if (open) return true;
    void *h = NULL;
    for (const char *name : {"libbz2.so.1.0", "libbz2.so.1", "libbz2.so"}) if ((h = dlopen(name, RTLD_NOW))) break;
    if (!h) return false;
    open = (void *(*)(const char *, const char *))dlsym(h, "BZ2_bzopen");
    read = (int (*)(void *, void *, int))dlsym(h, "BZ2_bzread");
    close = (void (*)(void *))dlsym(h, "BZ2_bzclose");
    return open && read && close;
  }
};
static Bz2Api Bz2;

static bool is_bzip2(const unsigned char *magic3) { return magic3[0] == 'B' && magic3[1] == 'Z' && magic3[2] == 'h'; }

struct LineReader {     // std::ifstream + std::getline state semantics (eofbit / failbit), over zlib / libbz2
  gzFile gz = NULL;
  void *bz = NULL;
  vector<char> buf;
  size_t pos = 0, end = 0;
  bool eofbit = false, failbit = false;
  bool open(const char *path) {
    unsigned char magic[3] = {0, 0, 0};
    if (FILE *f = fopen(path, "rb")) { size_t got = fread(magic, 1, 3, f); (void)got; fclose(f); }
    buf.resize(8 << 20);
    if (is_bzip2(magic)) {
      if (!Bz2.load()) die(EX_UNAVAILABLE, string("bzip2 input needs libbz2.so.1.0, which could not be loaded: ") + path);
      bz = Bz2.open(path, "rb");
      return bz != NULL;
    }
    gz = gzopen(path, "rb");
    if (!gz) return false;
    gzbuffer(gz, 1 << 20);
    return true;
  }
  void close() {
    if (gz) gzclose(gz);
    if (bz) Bz2.close(bz);
    gz = NULL; bz = NULL;
  }
  bool fill() {           // false at end of data
    int n = bz ? Bz2.read(bz, buf.data(), (int)buf.size()) : gzread(gz, buf.data(), (unsigned)buf.size());
    if (n <= 0) return false;
    pos = 0; end = (size_t)n;
    return true;
  }
  bool good() const { return !eofbit && !failbit; }
  // std::getline: extracts up to '\n'; hitting the end of the data sets eofbit, extracting nothing sets failbit
  bool getline(string &line) {
    line.clear();
    if (!good()) { failbit = true; return false; }
    bool extracted = false;
    for (;;) {
      if (pos == end && !fill()) {
        eofbit = true;
        if (!extracted) failbit = true;
        return extracted;
      }
      char *nl = (char *)memchr(buf.data() + pos, '\n', end - pos);
      if (nl) {
        line.append(buf.data() + pos, nl - (buf.data() + pos));
        pos = (nl - buf.data()) + 1;
        return true;
      }
      line.append(buf.data() + pos, end - pos);
      extracted = extracted || end > pos;
      pos = end;
    }
  }
  int peek() {
    if (pos == end && !fill()) return -1;
    return (unsigned char)buf[pos];
  }
};

// --extract: a record's lines as they are in the file (a FASTQ record's four lines, a FASTA record's sequence lines), each
// with its '\n' where the file has one
static void keep_line(string *raw, const string &line, const LineReader &in) {
  if (!raw) return;
  raw->append(line);
  if (!in.eofbit) *raw += '\n';
}

struct SeqReader {
  LineReader in;
  bool fastq = false, valid = true;
  string linebuffer;
  bool have_linebuffer = false;
  string *raw = NULL;                    // --extract: the record's lines are appended here
  string *log = NULL;                    // where the messages go (NULL: stderr at once)
  void note(const string &msg) {
    if (log) *log += "classify: " + msg + "\n";
    else fprintf(stderr, "classify: %s\n", msg.c_str());
  }
  // next_sequence(): FASTA seqreader.cpp:34-79, FASTQ :93-129.  Appends the sequence to `bases`.
  bool next(Read &r, string &bases) {
    r.quals.clear();
    if (fastq) {
      if (!valid || !in.good()) { valid = false; return false; }
      string line;
      in.getline(line);
      if (line.empty()) { valid = false; return false; }            // :101-104
      if (line[0] != '@') {
        if (line[0] != '\r') note("malformed fastq file - sequence header (" + line + ")");
        valid = false;
        return false;
      }
      r.header_line = line.substr(1);
      keep_line(raw, line, in);
      string seq;
      in.getline(seq);
      keep_line(raw, seq, in);
      in.getline(line);
      if (line.empty() || line[0] != '+') {
        if (line.empty() || line[0] != '\r') note("malformed fastq file - quality header (" + line + ")");
        valid = false;
        return false;
      }
      keep_line(raw, line, in);
      in.getline(r.quals);
      keep_line(raw, r.quals, in);
      r.seq_off = bases.size();
      r.seq_len = seq.size();
      bases += seq;
      return true;
    }
    if (!in.good()) { valid = false; return false; }                 // seqreader.cpp:37-40
    string line;
    if (have_linebuffer) { line = linebuffer; have_linebuffer = false; }
    else in.getline(line);
    if (line.empty() || line[0] != '>') {
      note("malformed fasta file - expected header char > not found");
      valid = false;
      return false;
    }
    r.header_line = line.substr(1);
    r.seq_off = bases.size();
    while (in.good()) {
      in.getline(line);
      if (!line.empty() && line[0] == '>') { linebuffer = line; have_linebuffer = true; break; }
      bases += line;
      keep_line(raw, line, in);
    }
    r.seq_len = bases.size() - r.seq_off;
    return true;
  }
};

// ---- paired-end input (--paired): the records scripts/read_merger.pl writes, merged during the ingest ------------
// Both readers (MateFile + PairReader for the serial path, process_file_parallel for plain files) take their record
// order from MergeOrder and their ids from mate_id, so the merger's rules live here.

// The length of a mate's id: the run of non-space characters right after the '>' / '@' (h is the header line without
// it), -1 when there is none (malformed, read_merger.pl:145-148,162-170); then s/[\/_.][12]$// (:182).  The id is a
// prefix of h.
static long mate_id(const char *h, size_t n) {
  size_t k = 0;
  while (k < n && !isspace((unsigned char)h[k])) k++;
  if (k == 0) return -1;
  if (k >= 2 && (h[k - 2] == '/' || h[k - 2] == '_' || h[k - 2] == '.') && (h[k - 1] == '1' || h[k - 1] == '2')) k -= 2;
  return (long)k;
}

// The order of the merged records (read_merger.pl:102-127).  `read(k)` takes the next record of mate file k: 1 a
// record, 0 the file has ended, -1 malformed.  `same()` compares the ids of the last record of each file.
struct MergeOrder {
  enum Kind { END, PAIR, ONLY1, ONLY2, EMPTY_N, MALFORMED, MISMATCH };
  enum { PAIRS, REST1, REST2, DONE } phase = PAIRS;
  template <class ReadMate, class Same> Kind next(ReadMate read, Same same) {
    int a, b;
    switch (phase) {
      case PAIRS:
        if ((a = read(0)) < 0) return fail(MALFORMED);
        if ((b = read(1)) < 0) return fail(MALFORMED);
        if (a == 0 && b == 0) { phase = DONE; return END; }
        if (a == 0) { warn(2); phase = REST2; return ONLY2; }
        if (b == 0) { warn(1); phase = REST1; return ONLY1; }
        if (Check_names && !same()) return fail(MISMATCH);
        return PAIR;
      case REST1:
        // after the rest of file 1 the loop falls through with both mates undefined and writes ">" + "N" (:104-118)
        if ((a = read(0)) < 0) return fail(MALFORMED);
        if (a == 0) { phase = DONE; return EMPTY_N; }
        return ONLY1;
      case REST2:
        if ((b = read(1)) < 0) return fail(MALFORMED);
        if (b == 0) { phase = DONE; return END; }
        return ONLY2;
      default:
        return END;
    }
  }
  Kind fail(Kind k) { phase = DONE; return k; }
  static void warn(int longer) {
    fprintf(stderr, "classify: mismatched sequence counts - file %d has more reads\n\n  Outputting the further reads unpaired\n", longer);
  }
};

static string mismatch_message(const char *a, size_t na, const char *b, size_t nb) {     // :114-116
  return "mismatched mate pair names ('" + string(a, na) + "' & '" + string(b, nb) + "')";
}

// read_sequence (read_merger.pl:136-183) over one mate file: the format is file 1's, whatever this file holds
struct MateFile {
  LineReader in;
  bool fasta = false;
  string buffer, id, seq;                  // buffer: the next record's header line, when have_line
  bool have_line = false, line_nl = false, ended = false;
  bool keep = false;                       // --extract: raw = the record's four FASTQ lines as in the file
  string raw;
  int read(string &err) {
    if (ended) return 0;
    if (!have_line) {
      if (!in.getline(buffer)) { ended = true; return 0; }
      have_line = true;
      line_nl = !in.eofbit;
    }
    const long k = buffer.empty() || buffer[0] != (fasta ? '>' : '@') ? -1 : mate_id(buffer.data() + 1, buffer.size() - 1);
    if (k < 0) {
      if (!fasta && buffer.empty()) { ended = true; return 0; }    // a blank line ends a FASTQ file (:165-167)
      err = string(fasta ? "malformed fasta file" : "malformed fastq file") + " (line = '" + buffer + (line_nl ? "\n" : "") + "')";
      return -1;
    }
    id.assign(buffer, 1, (size_t)k);
    have_line = false;
    seq.clear();
    if (fasta) {                                                   // every line up to the next '>' line, '\n' removed
      string line;
      while (in.getline(line)) {
        if (!line.empty() && line[0] == '>') { buffer.swap(line); have_line = true; line_nl = !in.eofbit; break; }
        seq += line;
      }
    } else {                                                       // line 2; lines 3 and 4 are skipped unchecked
      string skip;
      string *r = keep ? &raw : NULL;
      if (r) { raw.assign(buffer); if (line_nl) raw += '\n'; }
      in.getline(seq);
      keep_line(r, seq, in);
      in.getline(skip);
      keep_line(r, skip, in);
      in.getline(skip);
      keep_line(r, skip, in);
    }
    return 1;
  }
};

// The merged records of two mate files, with SeqReader::next's interface (the serial path: compressed files and pipes)
struct PairReader {
  MateFile m[2];
  MergeOrder order;
  bool valid = true;
  string *raw = NULL;                      // --extract: mate 1's lines, then mate 2's (raw_n2 bytes)
  uint32_t raw_n2 = 0;
  bool raw_visited = true;                 // the script reads the record: it has a mate 1 (PAIR, ONLY1)
  string *error = &Pair_error;              // where the merger's stop is recorded
  // "" or why a mate file cannot be opened
  string open(const char *f1, const char *f2) {
    const char *names[2] = {f1, f2};
    for (int k = 0; k < 2; k++) {
      struct stat sb;
      const bool regular = stat(names[k], &sb) == 0 && S_ISREG(sb.st_mode);
      unsigned char magic[3] = {0, 0, 0};
      if (regular)                                                 // determine_file_type (:199-216)
        if (FILE *f = fopen(names[k], "rb")) { size_t got = fread(magic, 1, 3, f); (void)got; fclose(f); }
      if (!m[k].in.open(names[k])) return string("can't open ") + names[k];
      const bool known = magic[0] == '@' || magic[0] == '>' || is_bzip2(magic) || (magic[0] == 0x1f && magic[1] == 0x8b && magic[2] == 8);
      if (regular && !known) { stop(string("Unknown input file type for ") + names[k]); return ""; }
    }
    const int c = m[0].in.peek();                                  // the format: file 1's first line (:66-75)
    if (c != '>' && c != '@') { stop(string("Unknown file format for ") + f1); return ""; }
    m[0].fasta = m[1].fasta = c == '>';
    return "";
  }
  void stop(const string &why) { *error = why; valid = false; }
  void close() { m[0].in.close(); m[1].in.close(); }
  bool next(Read &r, string &bases) {
    if (!valid) return false;
    string err;
    m[0].keep = m[1].keep = raw != NULL;
    auto kind = order.next([&](int k) { return m[k].read(err); }, [&] { return m[0].id == m[1].id; });
    if (raw) {
      raw_visited = kind == MergeOrder::PAIR || kind == MergeOrder::ONLY1;
      raw_n2 = kind == MergeOrder::PAIR ? (uint32_t)m[1].raw.size() : 0;
      if (raw_visited) *raw += m[0].raw;
      if (raw_n2) *raw += m[1].raw;
    }
    r.quals.clear();
    r.seq_off = bases.size();
    switch (kind) {
      case MergeOrder::PAIR: r.header_line = m[0].id; bases += m[0].seq; bases += 'N'; bases += m[1].seq; break;
      case MergeOrder::ONLY1: r.header_line = m[0].id; bases += m[0].seq; break;
      case MergeOrder::ONLY2: r.header_line = m[1].id; bases += m[1].seq; break;
      case MergeOrder::EMPTY_N: r.header_line.clear(); bases += 'N'; break;
      case MergeOrder::MALFORMED: stop(err); return false;
      case MergeOrder::MISMATCH: stop(mismatch_message(m[0].id.data(), m[0].id.size(), m[1].id.data(), m[1].id.size())); return false;
      case MergeOrder::END: valid = false; return false;
    }
    r.seq_len = bases.size() - r.seq_off;
    return true;
  }
};

// The records of one input of process_file / BatchReader: a FASTA / FASTQ file, or two mate files merged (--paired)
struct InputReader {
  SeqReader single;
  PairReader pair;
  bool paired = false;
  // "" or why the input cannot be opened
  string open(const char *filename, const char *mate2) {
    paired = mate2 != NULL;
    if (paired) return pair.open(filename, mate2);
    if (!single.in.open(filename)) return string("can't open ") + filename;
    single.fastq = single.in.peek() == '@';                        // determine_input_file_type, :377-388
    return "";
  }
  bool fastq() const { return !paired && single.fastq; }          // merged records are FASTA
  bool valid() const { return paired ? pair.valid : single.valid; }
  bool next(Read &r, string &bases) { return paired ? pair.next(r, bases) : single.next(r, bases); }
  void close() { if (paired) pair.close(); else single.in.close(); }
  void keep_raw(string *raw) { single.raw = pair.raw = raw; }
  uint32_t raw_n2() const { return paired ? pair.raw_n2 : 0; }
  bool raw_visited() const { return !paired || pair.raw_visited; }
};

// ---- taxonomy (taxdb.hpp:563-605) + report (taxdb.hpp:928-1123) ------------------------------------------------
struct TaxEntry {
  uint32_t id = 0;
  int parent = -1;                    // index into entries, -1 = NULL
  string name, rank;
  vector<int> children;
  uint64_t genomeSize = 0, genomeSizeOfChildren = 0;
};
struct TaxDB {
  vector<TaxEntry> e;
  unordered_map<uint32_t, int> idx;
  vector<uint32_t> row_ids, row_parents;   // every row in file order (krakenuniq-filter's parent map, kuq_set_threshold)
  bool keep_text = false;                  // also every row's name and rank (krakenuniq-mpa-report / -translate's maps)
  vector<string> row_names, row_ranks;
  void read(const string &path) {
    ifstream in(path);
    if (!in.is_open()) die(EX_NOINPUT, "unable to open taxonomy index file " + path);
    vector<uint32_t> parents;
    string line;
    while (getline(in, line)) {
      if (line.empty()) continue;
      size_t a = line.find('\t'), b = a == string::npos ? a : line.find('\t', a + 1);
      if (a == string::npos || b == string::npos) continue;
      size_t c = line.find('\t', b + 1);
      TaxEntry t;
      t.id = (uint32_t)strtoul(line.substr(0, a).c_str(), NULL, 10);
      uint32_t par = (uint32_t)strtoul(line.substr(a + 1, b - a - 1).c_str(), NULL, 10);
      if (t.id > 1 && t.id == par) die(1, "ERROR: the parent of " + to_string(t.id) + " is itself. Should not happend for taxa other than the root.");
      row_ids.push_back(t.id);
      row_parents.push_back(par);
      t.name = line.substr(b + 1, c == string::npos ? string::npos : c - b - 1);
      t.rank = c == string::npos ? "" : line.substr(c + 1);
      if (keep_text) {                                              // split(/\t/): the rank is the fourth field
        row_names.push_back(t.name);
        row_ranks.push_back(c == string::npos ? "" : line.substr(c + 1, line.find('\t', c + 1) - c - 1));
      }
      if (idx.count(t.id)) continue;                                // entries.insert keeps the first
      idx[t.id] = (int)e.size();
      e.push_back(t);
      parents.push_back(par);
    }
    if (!idx.count(0)) {                                            // taxdb.hpp:596
      TaxEntry z; z.id = 0; z.name = "unclassified"; z.rank = "no rank";
      idx[0] = (int)e.size(); e.push_back(z); parents.push_back(0);
    }
    for (size_t i = 0; i < e.size(); i++) {                          // createPointers, :411-433
      if (e[i].id == parents[i]) continue;
      auto it = idx.find(parents[i]);
      if (it == idx.end()) continue;
      e[i].parent = it->second;
      e[it->second].children.push_back((int)i);
    }
  }
  // getParentMap, :383-398
  void parent_map(vector<uint32_t> &ids, vector<uint32_t> &parents) const {
    for (auto &t : e) {
      if (t.id == 0) continue;
      ids.push_back(t.id);
      parents.push_back(t.parent < 0 ? 0 : e[t.parent].id);
    }
  }
  void set_genome_size(uint32_t taxid, uint64_t size) {               // :850-866
    auto it = idx.find(taxid);
    if (it == idx.end()) { cerr << "No taxonomy entry for " << taxid << "!!" << endl; return; }
    int i = it->second;
    e[i].genomeSize += size;
    while (e[i].parent >= 0) { i = e[i].parent; e[i].genomeSizeOfChildren += size; }
  }
};

struct Clade { uint64_t reads = 0, kmers = 0, unique = 0; };

static bool Exact_partitioned = false;   // classifyExact: the contexts hold the exact set's k-mer parts (kuq_exact_partition)
#ifdef EXACT_COUNTING
static bool Exact_union_needed = false;  // classifyExact: taxon 0 has children, so the report needs the whole set on one card
#endif
static bool Exact_settled = false;       // classifyExact: this sample's set spilled to host memory and was settled by part

static void print_report(kuq_ctx *ctx, TaxDB &tax, ostream &out) {
  uint32_t n = 0;
  if (kuq_counts_size(ctx, &n)) die(EX_SOFTWARE, kuq_last_error(ctx));
  vector<uint32_t> t(n);
  vector<uint64_t> nr(n), nk(n), uq(n);
  if (n && kuq_read_counts(ctx, t.data(), nr.data(), nk.data(), uq.data(), NULL, n)) die(EX_SOFTWARE, kuq_last_error(ctx));
  unordered_map<uint32_t, size_t> row;
  for (uint32_t i = 0; i < n; i++) row[t[i]] = i;
  // TaxReport ctor (:928-982): every counted taxon with an entry is a member of each ancestor's clade
  cerr << "Setting values in the taxonomy tree ...";
  map<int, vector<uint32_t>> members;
  for (uint32_t i = 0; i < n; i++) {
    auto it = tax.idx.find(t[i]);
    if (it == tax.idx.end()) { cerr << "No entry for " << t[i] << " in database!" << endl; continue; }
    for (int x = it->second; x >= 0; x = tax.e[x].parent) members[x].push_back(t[i]);
  }
  unordered_map<int, Clade> clade;
  // A handful of clades: one merge per clade.  A real taxonomy (thousands of rows): all clades in one call — the
  // library walks its own copy of the tree, which is this one as long as nothing hangs below the "unclassified" entry.
  size_t batch_min = 32;
  if (const char *v = getenv("KUQ_REPORT_BATCH_MIN")) batch_min = (size_t)strtoull(v, NULL, 10);
  bool batch = getenv("KUQ_REPORT_PER_CLADE") == NULL && members.size() >= batch_min;
  {
    auto z = tax.idx.find(0);
    if (z != tax.idx.end() && !tax.e[z->second].children.empty()) batch = false;
  }
  // an exact set partitioned over contexts has no member-list unions: every clade comes from the roll-up (the run kept
  // the union when taxon 0 has children, so the library's tree is this one)
  if (Exact_partitioned || Exact_settled) batch = true;
  if (batch) {
    vector<uint32_t> ids;
    vector<int> node;
    for (auto &kv : members) { ids.push_back(tax.e[kv.first].id); node.push_back(kv.first); }
    vector<uint64_t> r(ids.size()), k(ids.size()), u(ids.size());
    if (kuq_clade_counts_tree(ctx, ids.data(), (uint32_t)ids.size(), r.data(), k.data(), u.data())) die(EX_SOFTWARE, kuq_last_error(ctx));
    for (size_t i = 0; i < ids.size(); i++) { Clade c; c.reads = r[i]; c.kmers = k[i]; c.unique = u[i]; clade[node[i]] = c; }
  } else {
    for (auto &kv : members) {
      Clade c;
      if (kuq_clade_counts(ctx, kv.second.data(), (uint32_t)kv.second.size(), &c.reads, &c.kmers, &c.unique))
        die(EX_SOFTWARE, kuq_last_error(ctx));
      clade[kv.first] = c;
    }
  }
  cerr << " done" << endl;
  cerr << "Printing classification report ... ";
  uint64_t total = 0;
  for (uint32_t root : {0u, 1u, 0xFFFFFFFFu}) {
    auto it = tax.idx.find(root);
    if (it != tax.idx.end() && clade.count(it->second)) total += clade[it->second].reads;
  }
  if (total == 0) { cerr << "total number of reads is zero - not creating a report!" << endl; return; }
  const bool hll_cols = HLL_PRECISION > 0;
  out << (hll_cols ? "%\treads\ttaxReads\tkmers\tdup\tcov\ttaxID\trank\ttaxName\n" : "%\treads\ttaxReads\ttaxID\trank\ttaxName\n");
  // printReport(tax, depth), :1040-1076 (explicit stack instead of recursion)
  struct Item { int node; unsigned depth; };
  for (uint32_t root : {0u, 1u, 0xFFFFFFFFu}) {
    auto rit = tax.idx.find(root);
    if (rit == tax.idx.end()) continue;
    vector<Item> stack{{rit->second, 0}};
    while (!stack.empty()) {
      Item it = stack.back();
      stack.pop_back();
      auto cit = clade.find(it.node);
      if (cit == clade.end() || cit->second.reads == 0) continue;
      const TaxEntry &e = tax.e[it.node];
      const Clade &c = cit->second;
      auto r = row.find(e.id);
      // printLine, :1078-1123
      out << setprecision(4) << 100.0 * c.reads / total << '\t' << c.reads << '\t' << (r != row.end() ? nr[r->second] : 0) << '\t';
      if (hll_cols) {
        double genome_size = double(e.genomeSize + e.genomeSizeOfChildren);
        out << c.unique << '\t' << setprecision(3) << (double(c.kmers) / c.unique) << '\t';
        if (genome_size == 0) out << "NA"; else out << setprecision(4) << (c.unique / genome_size);
        out << '\t';
      }
      out << (e.id == 0xFFFFFFFFu ? -1 : (int32_t)e.id) << '\t' << e.rank << '\t' << string(2 * it.depth, ' ') + e.name << '\n';
      // children that have a clade, sorted descending by (reads, kmers) — ReadCounts::operator<, readcounts.hpp:90-98
      vector<int> ch;
      for (int k : e.children) if (clade.count(k)) ch.push_back(k);
      stable_sort(ch.begin(), ch.end(), [&](int a, int b) {
        const Clade &x = clade[a], &y = clade[b];
        return y.reads < x.reads || (y.reads == x.reads && y.kmers < x.kmers);
      });
      for (auto k = ch.rbegin(); k != ch.rend(); ++k) stack.push_back({*k, it.depth + 1});
    }
  }
  cerr << " done" << endl;
}

// ---- --mpa-report / --translate-out: the rules of scripts/krakenuniq-mpa-report and scripts/krakenuniq-translate ----
// Both scripts read the taxDB the same way (load_taxonomy): every row split on tabs, the name and the rank of a taxid
// from its last row.  mpa-report's child lists get one entry per row whose parent differs from its taxid, in file order
// (a taxid with two rows is listed, summed and printed twice); translate's parent map F is the one of krakenuniq-filter.
// Both take a Kraken line's fields as Perl's split on whitespace does: a line with an empty read id ("C\t\t562\t150...")
// has the taxon as its second field and the length as its third, which the scripts read as read id and taxid.
static char rank_code(const string &rank) {        // rank_code, mpa-report:168-182 / translate:115-128
  static const char *const ranks[] = {"species", "genus", "family", "order", "class", "phylum", "superkingdom", "kingdom"};
  static const char codes[] = "SGFOCPDK";
  for (int i = 0; i < 8; i++) if (rank == ranks[i]) return codes[i];
  return '-';
}

struct ScriptTax {
  unordered_map<uint32_t, uint32_t> last_row;     // name_map / rank_map: the taxid's last row
  vector<string> names, ranks;                    // per row
  unordered_map<uint32_t, vector<uint32_t>> children;
  unordered_map<uint32_t, uint32_t> F;
  // translate's lineage of every taxid with an F entry, computed the first time a line needs it (by any formatting
  // thread: `ready` 0 = not yet, 1 = being computed, 2 = done), and the node where its walk stops
  unordered_map<uint32_t, uint32_t> node;          // taxid -> slot
  vector<uint32_t> node_taxid, stop;
  vector<string> lineage;
  std::unique_ptr<std::atomic<uint8_t>[]> ready;
  bool mpa_format = false;

  const string &name(uint32_t t) const { static const string none; auto it = last_row.find(t); return it == last_row.end() ? none : names[it->second]; }
  const string &rank(uint32_t t) const { static const string none; auto it = last_row.find(t); return it == last_row.end() ? none : ranks[it->second]; }

  // false when F has a cycle (the script's walk never ends)
  bool build(const TaxDB &tax, bool translate) {
    names = tax.row_names;
    ranks = tax.row_ranks;
    for (uint32_t i = 0; i < tax.row_ids.size(); i++) {
      const uint32_t t = tax.row_ids[i], p = tax.row_parents[i];
      last_row[t] = i;
      if (p != t) { children[p].push_back(t); F[t] = p; }
    }
    if (!translate) return true;
    for (auto &kv : F) { node.emplace(kv.first, (uint32_t)node_taxid.size()); node_taxid.push_back(kv.first); }
    const size_t n = node_taxid.size();
    stop.assign(n, 0);
    lineage.assign(n, string());
    ready.reset(new std::atomic<uint8_t>[n]);
    vector<uint8_t> state(n, 0);                   // 1 = on the current walk, 2 = its stop is known
    vector<uint32_t> path;
    for (uint32_t i = 0; i < n; i++) {
      ready[i].store(0, std::memory_order_relaxed);
      path.clear();
      uint32_t x = node_taxid[i];
      for (auto it = node.find(x); it != node.end() && state[it->second] != 2; it = node.find(x)) {
        if (state[it->second] == 1) return false;
        state[it->second] = 1;
        path.push_back(it->second);
        x = F[x];
      }
      auto it = node.find(x);
      const uint32_t end = it == node.end() ? x : stop[it->second];
      for (uint32_t k : path) { stop[k] = end; state[k] = 2; }
    }
    return true;
  }

  // get_taxonomy_str's walk (translate:89-113): the names from the taxon up to the first node without an F entry,
  // which is left out; with --mpa-format only nodes with a rank code, as code__name with spaces turned into '_'
  string walk(uint32_t x) const {
    vector<string> parts;
    for (auto it = F.find(x); it != F.end(); x = it->second, it = F.find(x)) {
      if (!mpa_format) { parts.push_back(name(x)); continue; }
      const char code = rank_code(rank(x));
      if (code == '-') continue;
      string s = string(1, (char)tolower(code)) + "__" + name(x);
      replace(s.begin(), s.end(), ' ', '_');
      parts.push_back(s);
    }
    if (parts.empty()) return mpa_format ? "root" : "";
    string out;
    for (size_t k = parts.size(); k-- > 0;) { out += parts[k]; if (k) out += mpa_format ? '|' : ';'; }
    return out;
  }
  const string &lineage_at(uint32_t i) {
    if (ready[i].load(std::memory_order_acquire) == 2) return lineage[i];
    uint8_t z = 0;
    if (ready[i].compare_exchange_strong(z, 1, std::memory_order_acq_rel)) {
      lineage[i] = walk(node_taxid[i]);
      ready[i].store(2, std::memory_order_release);
    }
    while (ready[i].load(std::memory_order_acquire) != 2) std::this_thread::yield();
    return lineage[i];
  }
  const string &empty_lineage() const { static const string root = "root", none; return mpa_format ? root : none; }

  // krakenuniq-mpa-report (:95-125) over the lines per taxid of each sample, in sample order
  string mpa_table(const vector<unordered_map<uint64_t, uint64_t>> &taxo_counts, const vector<string> &ids,
                   bool show_zeros, bool header_line, bool intermediate) const {
    vector<unordered_map<uint64_t, uint64_t>> clade(taxo_counts);
    unordered_set<uint64_t> hit;
    for (auto &counts : clade) {
      // dfs_summation(1) (:184-194): after each child's own summation, the child's sum is added to the node's
      struct Frame { uint64_t node; size_t next; };
      vector<Frame> st{{1, 0}};
      while (!st.empty()) {
        const uint64_t x = st.back().node;
        auto it = x <= UINT32_MAX ? children.find((uint32_t)x) : children.end();
        if (it == children.end() || st.back().next == it->second.size()) {
          st.pop_back();
          if (!st.empty()) { auto c = counts.find(x); counts[st.back().node] += c == counts.end() ? 0 : c->second; }
          continue;
        }
        st.push_back({it->second[st.back().next++], 0});
      }
      for (auto &kv : counts) if (kv.second) hit.insert(kv.first);
    }
    // dfs_report(1) (:127-158): rows grouped by rank code in the order D K P C O F G S (X)
    const string order = intermediate ? "DKPCOFGSX" : "DKPCOFGS";
    vector<string> rows(order.size());
    struct Visit { uint32_t node; bool named; string name; };
    vector<Visit> st{{1, false, ""}};
    while (!st.empty()) {
      Visit v = std::move(st.back());
      st.pop_back();
      if (!show_zeros && !hit.count(v.node)) continue;
      char code = rank_code(rank(v.node));
      if (code != '-' || intermediate) {
        if (code == '-') code = 'X';
        string nm = name(v.node);
        nm.erase(remove_if(nm.begin(), nm.end(), [](char c) { return c == '|' || c == '.'; }), nm.end());
        replace(nm.begin(), nm.end(), ' ', '_');
        v.name = (v.named ? v.name + "|" : string()) + (char)tolower(code) + "__" + nm;
        v.named = true;
        string &out = rows[order.find(code)];
        out += v.name;
        for (auto &counts : clade) {
          auto c = counts.find(v.node);
          out += '\t';
          out += to_string(c == counts.end() ? 0 : c->second);
        }
        out += '\n';
      }
      auto it = children.find(v.node);
      if (it != children.end())
        for (auto k = it->second.rbegin(); k != it->second.rend(); ++k) st.push_back({*k, v.named, v.name});
    }
    string table;
    if (header_line) {
      table = "#Sample ID";
      for (auto &id : ids) table += "\t" + id;
      table += '\n';
    }
    for (auto &r : rows) table += r;
    return table;
  }
};
static ScriptTax Script_tax;

// What one formatting part adds to the two scripts' outputs.  Translate lines whose taxon has an F entry are written
// with their lineage; a line whose taxon has none prints the lineage most recently stored under that taxon (the script
// stores each lineage under the node where its walk stopped): when this part stored one earlier, it is written here,
// else the line is a hole that book_script fills from what the earlier parts stored.
struct ScriptPart {
  unordered_map<uint64_t, uint64_t> counts;        // mpa-report: lines per (script) taxid
  string translate;
  vector<pair<size_t, uint64_t>> holes;            // (offset in translate, taxid)
  unordered_map<uint64_t, uint32_t> last;          // stopping node -> slot of the last lineage stored under it
  void clear() { counts.clear(); translate.clear(); holes.clear(); last.clear(); }
};

// One Kraken line of the run (written or not): its code is 'C' when `shown` is not 0, its id is the header's first
// whitespace-delimited token
static void book_line(ScriptPart &p, const char *hdr, size_t hdr_len, uint64_t len, uint32_t shown) {
  size_t x = 0;
  while (x < hdr_len && isspace((unsigned char)hdr[x])) x++;
  size_t y = x;
  while (y < hdr_len && !isspace((unsigned char)hdr[y])) y++;
  const uint64_t taxid = y > x ? shown : len;       // split: an empty id moves the fields left
  if (Mpa) p.counts[taxid]++;
  if (!Translate_now || !shown) return;             // translate prints the lines that start with C
  if (y > x) p.translate.append(hdr + x, y - x);
  else p.translate += to_string(shown);
  p.translate += '\t';
  auto it = taxid <= UINT32_MAX ? Script_tax.node.find((uint32_t)taxid) : Script_tax.node.end();
  if (it != Script_tax.node.end()) {
    p.translate += Script_tax.lineage_at(it->second);
    p.last[Script_tax.stop[it->second]] = it->second;
  } else {
    auto l = p.last.find(taxid);
    if (l != p.last.end()) p.translate += Script_tax.lineage_at(l->second);
    else p.holes.emplace_back(p.translate.size(), taxid);
  }
  p.translate += '\n';
}

// ---- mmap helper ----------------------------------------------------------------------------------------------
struct Mapped {
  void *p = NULL;
  size_t size = 0;
  void open(const string &path) {
    int fd = ::open(path.c_str(), O_RDONLY);
    if (fd < 0) die(EX_OSERR, "unable to open " + path);
    struct stat sb;
    if (fstat(fd, &sb) < 0) die(EX_OSERR, "unable to fstat " + path);
    size = sb.st_size;
    p = mmap(0, size, PROT_READ, MAP_PRIVATE, fd, 0);
    if (p == MAP_FAILED) die(EX_OSERR, "unable to mmap " + path);
    madvise(p, size, MADV_SEQUENTIAL);
    ::close(fd);
  }
};

static double now_s() { struct timeval t; gettimeofday(&t, NULL); return t.tv_sec + t.tv_usec / 1e6; }
static const bool Timing = getenv("KUQ_TIMING") != NULL;
#define TICK(label) do { if (Timing) { double t__ = now_s(); fprintf(stderr, "\n[timing] %-28s %.3f s\n", label, t__ - T0__); T0__ = t__; } } while (0)
static double get_seconds(struct timeval a, struct timeval b) {
  return (b.tv_sec - a.tv_sec) + (b.tv_usec - a.tv_usec) / 1e6;
}

// ---- batches and their output ------------------------------------------------------------------------------------
// --extract: where a read's lines lie in Batch::raw (mate 1's or the only record's n1 bytes, then mate 2's n2)
struct RawRec { uint64_t off; uint32_t n1, n2; bool visited; };

struct Batch {
  string bases;
  vector<uint64_t> offs{0};
  vector<Read> reads;
  vector<uint32_t> units;             // the reads' work units (kuq_batches.h)
  bool fastq = false;
  string raw;                         // --extract only: the reads' lines as in the file
  vector<RawRec> raw_recs;
  size_t sample = 0;                  // the sample whose reads these are (streamed sheet runs)
  void clear() { bases.clear(); offs.assign(1, 0); reads.clear(); units.clear(); raw.clear(); raw_recs.clear(); }
};

static const uint64_t SLOT_NT = 280ull << 20;   // the longest read of the resident paths, below the slot capacity (288 MiB)

// The limits of a batch (kuq_batches.h) with the work units of this run.  Resident databases: a batch fills one slot,
// and KUQ_BATCH_READS closes it at the first unit boundary after that many reads (tests: small batches).
static BatchLimits batch_limits(uint64_t batch_nt, bool aligned, bool resident) {
  BatchLimits l;
  l.batch_nt = batch_nt;
  l.max_units = Max_units_per_batch;
  l.unit_size = Work_unit_size;
  l.aligned = aligned;
  l.slot_nt = resident ? SLOT_NT : 0;
  const char *v = getenv("KUQ_BATCH_READS");
  if (resident && v) l.batch_reads = std::min<size_t>(l.batch_reads, std::max<size_t>(1, strtoull(v, NULL, 10)));
  return l;
}

static OutStream Kraken_out, Classified_out, Unclassified_out, Extract_out, Translate_out;

// One read as the output sees it: the header line without its '>' / '@', the bases and (FASTQ) the qualities
struct ReadView {
  const char *hdr; size_t hdr_len;
  const char *seq; uint64_t len;
  const char *qual; size_t qual_len;
};

// The Kraken lines (classify.cpp:980-1010, hitlist_string :826-861) and the -C / -U records (print_sequence, :794-805)
// of reads [a, b); read i's results are at i - res0 of `res`.  The Kraken text goes into one buffer sized up front.
// `sp` (--mpa-report / --translate-out only) books every line the run writes, or would write with -o FILE.
template <class ViewOf>
static void format_reads(ViewOf view_of, size_t a, size_t b, const kuq_batch_result &res, size_t res0, bool fastq,
                         string &kraken, string &classified, string &unclassified, ScriptPart *sp = NULL) {
  const size_t at = kraken.size();
  if (Print_kraken) {
    size_t need = 0;
    for (size_t i = a; i < b; i++) {
      const ReadView v = view_of(i);
      need += 2 + v.hdr_len + 1 + 10 + 1 + 20 + 1 + 4 + 22ull * res.run_count[i - res0] + 1 + (Print_sequence ? v.len + 1 : 0) +
              (Filter ? 16 : 0);
    }
    kraken.resize(at + need);
  }
  char *o = Print_kraken ? &kraken[at] : NULL;
  auto put = [&](auto v) {
    char buf[20];
    int k = 0;
    do { buf[k++] = (char)('0' + v % 10); v /= 10; } while (v);
    while (k) *o++ = buf[--k];
  };
  for (size_t i = a; i < b; i++) {
    const ReadView v = view_of(i);
    const size_t r = i - res0;
    const uint32_t call = res.call[r];
    if ((Print_unclassified && !call) || (Print_classified && call)) {
      string &oo = call ? classified : unclassified;
      oo += fastq ? '@' : '>';
      oo.append(v.hdr, v.hdr_len); oo += '\n';
      oo.append(v.seq, v.len); oo += '\n';
      if (fastq) { oo += "+\n"; oo.append(v.qual, v.qual_len); oo += '\n'; }
    }
    if (sp && (call || !Only_classified_kraken_output)) book_line(*sp, v.hdr, v.hdr_len, v.len, Filter ? res.filtered_call[r] : call);
    if (!Print_kraken) continue;
    if (!call && Only_classified_kraken_output) continue;            // :986-988
    // --threshold: krakenuniq-filter's line (:131-133), "%s\t<id>\t<new taxon>\t<len>\tP=%0.3f\t<hit list>\n"
    const uint32_t shown = Filter ? res.filtered_call[r] : call;
    *o++ = shown ? 'C' : 'U'; *o++ = '\t';
    {   // id = first whitespace-delimited token of the header line
      size_t x = 0;
      while (x < v.hdr_len && isspace((unsigned char)v.hdr[x])) x++;
      size_t y = x;
      while (y < v.hdr_len && !isspace((unsigned char)v.hdr[y])) y++;
      memcpy(o, v.hdr + x, y - x); o += y - x;
    }
    *o++ = '\t';
    put(shown);
    *o++ = '\t';
    put(v.len);
    *o++ = '\t';
    if (Filter) {
      const uint32_t den = res.filter_total[r];
      o += snprintf(o, 12, "P=%.3f\t", den ? (double)res.filter_hits[r] / den : 0.0);
    }
    if (Quick_mode) { *o++ = 'Q'; *o++ = ':'; put(res.run_count[r]); }   // :989-990
    else if (res.run_count[r] == 0) { *o++ = '0'; *o++ = ':'; *o++ = '0'; }   // :994-995
    for (uint32_t j = 0; !Quick_mode && j < res.run_count[r]; j++) {
      const kuq_run &run = res.runs[res.run_start[r] + j];
      if (j) *o++ = ' ';
      if (run.code == KUQ_CODE_AMBIG) *o++ = 'A'; else put(run.code);
      *o++ = ':';
      put(run.count);
    }
    if (Print_sequence) { *o++ = '\t'; memcpy(o, v.seq, v.len); o += v.len; }
    *o++ = '\n';
  }
  if (Print_kraken) kraken.resize(o - &kraken[0]);
}

// ---- --extract: krakenuniq-extract-reads (:139-217) over the records as they are in the input ---------------------
// One record as the script reads it: `hdr` the header line without its '@' / '>' (the FASTQ record's first line for
// paired reads), `kid` the header our Kraken line takes its id from, m1 / m2 the lines the script prints (a FASTQ
// record's four lines, a FASTA record's sequence lines; m2 = the second mate's four lines).  visited: the script reaches
// the record (records of mate file 2 that have no mate 1 are never read).
struct XRec {
  const char *hdr; size_t hdr_len;
  const char *kid; size_t kid_len;
  const char *m1; size_t n1;
  const char *m2; size_t n2;
  bool visited;
};

// the length of the id the script looks up (:142-150): the line's first word without its '@' / '>' (a prefix of h),
// and one trailing /1 /2 .1 .2
static size_t script_id(const char *h, size_t n) {
  size_t k = 0;
  while (k < n && h[k] != '\n' && !isspace((unsigned char)h[k])) k++;
  if (k >= 2 && (h[k - 2] == '/' || h[k - 2] == '.') && (h[k - 1] == '1' || h[k - 1] == '2')) k -= 2;
  return k;
}

// whether our Kraken line's id (format_reads: the header's first whitespace-delimited token) is id[0, k)
static bool kraken_id_is(const char *h, size_t n, const char *id, size_t k) {
  size_t x = 0;
  while (x < n && isspace((unsigned char)h[x])) x++;
  size_t y = x;
  while (y < n && !isspace((unsigned char)h[y])) y++;
  return y - x == k && memcmp(h + x, id, k) == 0;
}

// the second line of a FASTQ record's text, with its '\n' when it has one
static void append_line2(string &o, const char *m, size_t n) {
  const char *nl = (const char *)memchr(m, '\n', n);
  if (!nl) return;
  const char *s = nl + 1, *e = (const char *)memchr(s, '\n', m + n - s);
  o.append(s, e ? e + 1 - s : m + n - s);
}

// What the script prints for reads [a, b): a read is printed when its Kraken line is selected (extract_sel bit 0 holds
// selected XOR --extract-invert) and the script's id of the record is that line's id; where the ids differ (a header
// ending in /1 .1 ...), the script finds no line for the record, so it prints the record only with --extract-invert.
template <class XOf>
static void extract_reads(XOf x_of, size_t a, size_t b, const kuq_batch_result &res, size_t res0, bool fasta, string &out) {
  for (size_t i = a; i < b; i++) {
    // a read whose line is not selected is written exactly with --extract-invert, whichever id it has; one whose line
    // is selected is written when the script finds the line under the record's id, and with --extract-invert when not
    const bool selected = ((res.extract_sel[i - res0] & 1) != 0) != Extract_invert;
    if (!selected && !Extract_invert) continue;
    const XRec x = x_of(i);
    if (!x.visited) continue;
    const size_t k = script_id(x.hdr, x.hdr_len);
    if (selected && kraken_id_is(x.kid, x.kid_len, x.hdr, k) == Extract_invert) continue;
    const string id(x.hdr, k);
    if (fasta) {                                                   // -a (:162-177)
      out += '>'; out += id; out += '\n';
      out.append(x.m1, x.n1);
    } else if (Extract_fasta) {                                    // -f (:162-190)
      out += '>'; out += id; out += '\n';
      append_line2(out, x.m1, x.n1);
      if (Paired) { out += '>'; out += id; out += '\n'; append_line2(out, x.m2, x.n2); }
    } else {                                                       // the four lines, then mate 2's (:191-204)
      out.append(x.m1, x.n1);
      out.append(x.m2, x.n2);
    }
  }
}

// The script prints nothing when no line is selected (:127), even with -i.  Text written before the sample's first
// selected read is held back (only --extract-invert writes such text) and dropped if no read is ever selected.
static string Extract_pending;
static uint64_t Extract_selected = 0;      // selected reads of the sample so far
static void write_extract(const string &text, bool selected_so_far) {
  if (!selected_so_far) { Extract_pending += text; return; }
  if (!Extract_pending.empty()) { Extract_out.write(Extract_pending); string().swap(Extract_pending); }
  Extract_out.write(text);
}

// A part's booking, in output order: its counts join the sample's column, its translate text is written with the holes
// filled from what the sample's earlier parts stored (batches and input files included), then its own stores are added.
static vector<unordered_map<uint64_t, uint64_t>> Mpa_counts;   // per sample of the run
static vector<string> Mpa_ids;                                  // the samples' ids (--mpa-header-line)
static unordered_map<uint64_t, uint32_t> Translate_stored;      // the sample's last lineage per stopping node
static bool scripts_now() { return Mpa || Translate_now; }
static void book_script(const ScriptPart &p) {
  if (Mpa) {
    auto &c = Mpa_counts.back();
    for (auto &kv : p.counts) c[kv.first] += kv.second;
  }
  if (!Translate_now) return;
  size_t at = 0;
  for (auto &h : p.holes) {
    Translate_out.write(p.translate.data() + at, h.first - at);
    auto it = Translate_stored.find(h.second);
    Translate_out.write(it == Translate_stored.end() ? Script_tax.empty_lineage() : Script_tax.lineage_at(it->second));
    at = h.first;
  }
  Translate_out.write(p.translate.data() + at, p.translate.size() - at);
  for (auto &kv : p.last) Translate_stored[kv.first] = kv.second;
}

// The output of reads [a, b) of a batch, whose results start at read a (the whole batch, or a GPU's share of it)
static void write_reads(const Batch &bt, const kuq_batch_result &res, size_t a, size_t b) {
  string kraken, classified, unclassified;
  auto view_of = [&](size_t i) {
    const Read &r = bt.reads[i];
    return ReadView{r.header_line.data(), r.header_line.size(), bt.bases.data() + r.seq_off, r.seq_len, r.quals.data(), r.quals.size()};
  };
  static ScriptPart sp;
  sp.clear();
  format_reads(view_of, a, b, res, a, bt.fastq, kraken, classified, unclassified, scripts_now() ? &sp : NULL);
  if (scripts_now()) book_script(sp);
  Kraken_out.write(kraken);
  Classified_out.write(classified);
  Unclassified_out.write(unclassified);
  if (!Extract_now) return;
  Extract_selected += res.n_extract;
  if (!res.n_extract && !Extract_invert) return;
  const bool fasta = !bt.fastq && !Paired;
  auto x_of = [&](size_t i) {
    const Read &r = bt.reads[i];
    const RawRec &q = bt.raw_recs[i];
    const char *m1 = bt.raw.data() + q.off;
    const char *h = fasta ? r.header_line.data() : m1 + 1;
    const size_t hn = fasta ? r.header_line.size() : (q.n1 ? q.n1 - 1 : 0);
    return XRec{h, hn, r.header_line.data(), r.header_line.size(), m1, q.n1, m1 + q.n1, q.n2, q.visited && (fasta || q.n1)};
  };
  string x;
  extract_reads(x_of, a, b, res, a, fasta, x);
  write_extract(x, Extract_selected > 0);
}

// A batch's totals (report_stats, classify.cpp:361-375) and the progress line (:555-558)
static void book_batch(uint64_t reads, uint64_t bases, uint64_t classified) {
  total_classified += classified;
  total_sequences += reads;
  total_bases += bases;
  fprintf(stderr, "\r Processed %llu sequences (%.2f%% classified)", total_sequences, total_classified * 100.0 / total_sequences);
}

// The records per taxid of the databases `ctx` has staged, added to `into` (kuq_db_taxids: count, then fetch)
static int db_taxids(kuq_ctx *ctx, map<uint32_t, uint64_t> &into) {
  uint32_t m = 0;
  int rc = kuq_db_taxids(ctx, NULL, NULL, 0, &m);
  vector<uint32_t> t(m);
  vector<uint64_t> c(m);
  if (!rc && m) rc = kuq_db_taxids(ctx, t.data(), c.data(), m, &m);
  for (uint32_t i = 0; !rc && i < m; i++) into[t[i]] += c[i];
  return rc;
}

// A piece of database `db` staged on a context: bins [bin_lo, bin_hi); (0, 0) is the whole database, lo == hi != 0 an
// empty slice
struct Slice { size_t db; uint64_t bin_lo, bin_hi; };

// Context g stages slices[g] in order, one thread per context.  join: each slice joins what the context holds
// (kuq_stage_db_append_range); else each replaces the last (kuq_stage_db), for a group of ranges that does not fit at
// once.  db_counts[d] (the .counts files) gets the records per taxid that database d's slices add: the context's
// db_taxids after a slice minus those before it (none before it when slices replace).  replicas: every context stages
// the same slices, so context 0 alone counts.
static void stage_slices(const vector<kuq_ctx *> &ctxs, const vector<Mapped> &kdbs, const vector<Mapped> &idxs,
                         const vector<vector<Slice>> &slices, bool join, bool replicas, vector<map<uint32_t, uint64_t>> &db_counts) {
  const int G = (int)ctxs.size();
  vector<vector<map<uint32_t, uint64_t>>> added(G, vector<map<uint32_t, uint64_t>>(db_counts.size()));
  vector<int> rcs(G, 0);
#pragma omp parallel for num_threads(G) schedule(static, 1)
  for (int g = 0; g < G; g++) {
    map<uint32_t, uint64_t> before, after;
    for (size_t i = 0; i < slices[g].size() && !rcs[g]; i++) {
      const Slice &s = slices[g][i];
      const Mapped &kdb = kdbs[s.db], &idx = idxs[s.db];
      rcs[g] = join ? kuq_stage_db_append_range(ctxs[g], kdb.p, kdb.size, idx.p, idx.size, s.bin_lo, s.bin_hi)
                    : kuq_stage_db(ctxs[g], kdb.p, kdb.size, idx.p, idx.size, s.bin_lo, s.bin_hi);
      if (rcs[g] || (replicas && g)) continue;
      after.clear();
      if ((rcs[g] = db_taxids(ctxs[g], after))) continue;
      for (auto &kv : after) {
        const auto b = before.find(kv.first);
        const uint64_t was = b == before.end() ? 0 : b->second;
        if (kv.second > was) added[g][s.db][kv.first] += kv.second - was;
      }
      if (join) before.swap(after);
    }
  }
  for (int g = 0; g < G; g++) if (rcs[g]) die(EX_DATAERR, kuq_last_error(ctxs[g]));
  for (int g = 0; g < G; g++)
    for (size_t d = 0; d < db_counts.size(); d++)
      for (auto &kv : added[g][d]) db_counts[d][kv.first] += kv.second;
}

// Contexts that each hold a part of the databases (shards, streamed groups): every one numbers the taxids of every
// database and range (kuq_set_db_taxid_universe), and may store into the others' id buffers (peer access)
static void share_taxa(const vector<kuq_ctx *> &ctxs, const vector<map<uint32_t, uint64_t>> &db_counts) {
  set<uint32_t> all;
  for (auto &c : db_counts) for (auto &kv : c) all.insert(kv.first);
  const vector<uint32_t> u(all.begin(), all.end());
  for (kuq_ctx *c : ctxs)
    if (kuq_set_db_taxid_universe(c, u.data(), (uint32_t)u.size())) die(EX_SOFTWARE, kuq_last_error(c));
  for (kuq_ctx *c : ctxs)
    for (kuq_ctx *p : ctxs) if (p != c && kuq_enable_peer_access(c, p)) die(EX_SOFTWARE, kuq_last_error(c));
}

// background writer: formatted text is handed over batch by batch and written in order while the next batch is
// being gathered / classified / formatted
struct OutJob { vector<string> kraken, classified, unclassified, extract; vector<ScriptPart> script; bool extract_selected = false; };
struct Writer {
  std::mutex m;
  std::condition_variable cv;
  std::deque<OutJob> q;
  std::deque<OutJob> spare;              // written jobs, recycled so that their string buffers stay mapped
  bool done = false;
  std::thread th;
  void start() { th = std::thread([this] { run(); }); }
  void push(OutJob &&j) { { std::lock_guard<std::mutex> l(m); q.push_back(std::move(j)); } cv.notify_one(); }
  OutJob take(size_t parts) {
    OutJob j;
    { std::lock_guard<std::mutex> l(m); if (!spare.empty()) { j = std::move(spare.front()); spare.pop_front(); } }
    j.kraken.resize(parts); j.classified.resize(parts); j.unclassified.resize(parts); j.extract.resize(parts);
    for (auto &x : j.kraken) x.clear();
    for (auto &x : j.classified) x.clear();
    for (auto &x : j.unclassified) x.clear();
    for (auto &x : j.extract) x.clear();
    j.script.resize(scripts_now() ? parts : 0);
    for (auto &x : j.script) x.clear();
    return j;
  }
  void finish() { { std::lock_guard<std::mutex> l(m); done = true; } cv.notify_one(); if (th.joinable()) th.join(); }
  void run();
};

void Writer::run() {
  for (;;) {
    OutJob j;
    {
      std::unique_lock<std::mutex> l(m);
      cv.wait(l, [this] { return done || !q.empty(); });
      if (q.empty()) return;
      j = std::move(q.front());
      q.pop_front();
    }
    for (auto &x : j.kraken) Kraken_out.write(x);
    for (auto &x : j.classified) Classified_out.write(x);
    for (auto &x : j.unclassified) Unclassified_out.write(x);
    if (Extract_now) for (auto &x : j.extract) write_extract(x, j.extract_selected);
    for (auto &x : j.script) book_script(x);
    { std::lock_guard<std::mutex> l(m); if (spare.size() < 3) spare.push_back(std::move(j)); }
  }
}

// ---- parallel ingest for plain (uncompressed) files --------------------------------------------------------------
// The file is mmap'ed and cut into chunks at record boundaries; every chunk is parsed by its own thread into
// zero-copy views (FASTQ) with exactly the record semantics of src/seqreader.cpp; a sequential pass over the read
// lengths then cuts work units and batches like process_file (classify.cpp:506-521); sequence text is gathered into
// pinned buffers and the Kraken lines are formatted by all threads.
struct View {
  const char *hdr; uint32_t hdr_len;      // header line without the leading '>' / '@'
  const char *seq; uint32_t seq_len;      // FASTQ / single-line FASTA: points into the file
  const char *qual; uint32_t qual_len;
  int64_t owned;                          // >= 0: index into the chunk's arena (multi-line FASTA)
};
struct ChunkParse {
  vector<View> reads;
  vector<string> arena;
  bool stopped = false;                   // parser hit the end-of-input condition of the reference reader
  string warning;
};

static inline const char *line_end(const char *p, const char *end) {
  const char *nl = (const char *)memchr(p, '\n', end - p);
  return nl ? nl : end;
}

// FASTQ records [p, end): FastqReader::next_sequence, seqreader.cpp:93-129
static void parse_fastq_chunk(const char *p, const char *end, const char *file_end, ChunkParse &out) {
  while (p < end) {
    const char *e0 = line_end(p, file_end);
    if (e0 == p) { out.stopped = true; return; }                                  // empty line (:101-104)
    if (*p != '@') {
      if (*p != '\r') out.warning = "malformed fastq file - sequence header (" + string(p, e0 - p) + ")";
      out.stopped = true;
      return;
    }
    const char *s = e0 < file_end ? e0 + 1 : file_end;
    const char *e1 = line_end(s, file_end);
    const char *pl = e1 < file_end ? e1 + 1 : file_end;
    const char *e2 = line_end(pl, file_end);
    if (e2 == pl || *pl != '+') {
      if (e2 == pl || *pl != '\r') out.warning = "malformed fastq file - quality header (" + string(pl, e2 - pl) + ")";
      out.stopped = true;
      return;
    }
    const char *q = e2 < file_end ? e2 + 1 : file_end;
    const char *e3 = line_end(q, file_end);
    View v;
    v.hdr = p + 1; v.hdr_len = (uint32_t)(e0 - p - 1);
    v.seq = s; v.seq_len = (uint32_t)(e1 - s);
    v.qual = q; v.qual_len = (uint32_t)(e3 - q);
    v.owned = -1;
    out.reads.push_back(v);
    p = e3 < file_end ? e3 + 1 : file_end;
  }
}

// FASTA records [p, end): FastaReader::next_sequence, seqreader.cpp:34-79.  `p` is at a '>' line start.
static void parse_fasta_chunk(const char *p, const char *end, const char *file_end, ChunkParse &out) {
  while (p < end) {
    const char *e0 = line_end(p, file_end);
    if (*p != '>') { out.warning = "malformed fasta file - expected header char > not found"; out.stopped = true; return; }
    // a last header line that is not newline-terminated sets eofbit while being read into the line buffer, and the
    // reader then reports !good() before using it (seqreader.cpp:37-40,62-66): that record is never produced
    if (e0 == file_end) { out.stopped = true; return; }
    View v;
    v.hdr = p + 1; v.hdr_len = (uint32_t)(e0 - p - 1);
    v.qual = NULL; v.qual_len = 0; v.owned = -1;
    const char *s = e0 < file_end ? e0 + 1 : file_end;
    // sequence lines until the next line that starts with '>'
    const char *first = s, *first_end = line_end(s, file_end);
    const char *nxt = first_end < file_end ? first_end + 1 : file_end;
    if (s >= file_end) { v.seq = s; v.seq_len = 0; out.reads.push_back(v); return; }
    if (*s == '>') { v.seq = s; v.seq_len = 0; out.reads.push_back(v); p = s; continue; }
    if (nxt >= file_end || *nxt == '>') {                                          // single-line sequence: zero copy
      v.seq = first; v.seq_len = (uint32_t)(first_end - first);
      out.reads.push_back(v);
      p = nxt;
      continue;
    }
    string acc(first, first_end - first);
    const char *q = nxt;
    while (q < file_end && *q != '>') {
      const char *qe = line_end(q, file_end);
      acc.append(q, qe - q);
      q = qe < file_end ? qe + 1 : file_end;
    }
    v.owned = (int64_t)out.arena.size();
    v.seq = NULL; v.seq_len = (uint32_t)acc.size();
    out.arena.push_back(std::move(acc));
    out.reads.push_back(v);
    p = q;
  }
}

// start of the first record at or after `p` (chunk boundary search)
static const char *next_record_start(const char *p, const char *file_begin, const char *file_end, bool fastq) {
  if (p <= file_begin) return file_begin;
  // move to the start of the next line
  const char *nl = (const char *)memchr(p - 1, '\n', file_end - (p - 1));
  if (!nl) return file_end;
  p = nl + 1;
  while (p < file_end) {
    const char *e0 = line_end(p, file_end);
    if (!fastq) { if (*p == '>') return p; }
    else if (*p == '@') {
      // a header is followed two lines later by the '+' line; a quality line that starts with '@' is not
      const char *l1 = e0 < file_end ? e0 + 1 : file_end;
      const char *e1 = line_end(l1, file_end);
      const char *l2 = e1 < file_end ? e1 + 1 : file_end;
      if (l2 < file_end && *l2 == '+' && l1 < file_end && *l1 != '@') return p;
    }
    p = e0 < file_end ? e0 + 1 : file_end;
  }
  return file_end;
}

struct Stage { char *bases = NULL; uint64_t cap = 0; uint64_t *offs = NULL; size_t offs_cap = 0; size_t begin = 0, end = 0; };
// pinned staging of one batch; prepare_stage() is also called up front, while the database is being staged
static vector<Stage> Prealloc_stages;
static void prepare_stage(Stage &s, uint64_t bases, size_t reads) {
  if (s.cap < bases + 64) {
    if (s.bases) kuq_host_free(s.bases);
    s.cap = std::max<uint64_t>(bases + 64, 160ull << 20);
    s.bases = (char *)kuq_host_alloc(s.cap);
    if (!s.bases) die(EX_OSERR, "pinned allocation failed");
  }
  if (s.offs_cap < reads + 2) {
    if (s.offs) kuq_host_free(s.offs);
    s.offs_cap = std::max<size_t>(reads + 2, (1u << 20) + 8);
    s.offs = (uint64_t *)kuq_host_alloc(s.offs_cap * 8);
    if (!s.offs) die(EX_OSERR, "pinned allocation failed");
  }
}

// Several GPUs (replicas: every device holds the database): batches go round-robin over the contexts; results come back
// in submission order, so the Kraken output stays in file order whatever the number of devices.
static vector<kuq_ctx *> All_ctx;

// A plain file (regular, uncompressed) mapped and cut into chunks at record boundaries, every chunk parsed by its own
// thread
struct PlainInput {
  const char *base = NULL, *fend = NULL;
  size_t size = 0;
  vector<const char *> cut;
  vector<ChunkParse> parsed;
  bool map(const char *filename) {
    int fd = ::open(filename, O_RDONLY);
    if (fd < 0) return false;
    struct stat sb;
    if (fstat(fd, &sb) < 0 || !S_ISREG(sb.st_mode) || sb.st_size < 2) { ::close(fd); return false; }
    size = sb.st_size;
    base = (const char *)mmap(0, size, PROT_READ, MAP_PRIVATE, fd, 0);
    ::close(fd);
    if (base == MAP_FAILED) { base = NULL; return false; }
    if (((unsigned char)base[0] == 0x1f && (unsigned char)base[1] == 0x8b) || (size >= 3 && is_bzip2((const unsigned char *)base))) {
      unmap();                                                      // gzip / bzip2: the serial reader decompresses
      return false;
    }
    madvise((void *)base, size, MADV_WILLNEED);
    fend = base + size;
    return true;
  }
  void unmap() { if (base) munmap((void *)base, size); base = NULL; }
  void parse(bool fastq, int T) {
    const int n_chunks = (int)std::min<size_t>((size_t)T * 4, std::max<size_t>(1, size / (1 << 20)));
    cut.assign(n_chunks + 1, NULL);
    cut[0] = base; cut[n_chunks] = fend;
    for (int c = 1; c < n_chunks; c++) cut[c] = next_record_start(base + size * c / n_chunks, base, fend, fastq);
    for (int c = 1; c <= n_chunks; c++) if (cut[c] < cut[c - 1]) cut[c] = cut[c - 1];
    parsed.assign(n_chunks, ChunkParse());
#pragma omp parallel for schedule(dynamic, 1) num_threads(T)
    for (int c = 0; c < n_chunks; c++) {
      if (cut[c] >= cut[c + 1]) continue;
      if (fastq) parse_fastq_chunk(cut[c], cut[c + 1], fend, parsed[c]);
      else parse_fasta_chunk(cut[c], cut[c + 1], fend, parsed[c]);
    }
  }
};

static string malformed_message(bool fasta, char marker, const char *line, size_t n, bool newline) {   // :149,170
  return string(fasta ? "malformed fasta file" : "malformed fastq file") + " (line = '" + (marker ? string(1, marker) : "") +
         string(line, n) + (newline ? "\n" : "") + "')";
}

// Where a merged record's bases come from: s1, then 'N' and s2 when the record joins two mates
struct MateSeqs { const char *s1, *s2; uint32_t n1, n2; bool joined; };

// The records of two parsed mate files, merged (MergeOrder, mate_id): each view is named by the stripped id of its mate
// (a prefix of that mate's header).  False where the chunk parsers and read_merger.pl part ways (a FASTQ record without
// its '+' line, a file that does not start with a header, a FASTA header on the last line without a newline): the
// serial PairReader then reads the pair.
static bool merge_parsed(const PlainInput (&in)[2], bool fastq, int T, vector<View> &merged, vector<MateSeqs> &mates) {
  struct Rec { const View *v; const char *seq; long id; };
  vector<Rec> recs[2];
  for (int k = 0; k < 2; k++) {
    const vector<ChunkParse> &parsed = in[k].parsed;
    int last_chunk = (int)parsed.size();
    for (int c = 0; c < (int)parsed.size(); c++) {
      if (!parsed[c].stopped) continue;
      // a blank line where a FASTQ header should be ends the file for both; any other stop differs
      const vector<View> &rs = parsed[c].reads;
      const char *p = rs.empty() ? in[k].cut[c] : rs.back().qual + rs.back().qual_len + 1;
      if (!fastq || p >= in[k].fend || *p != '\n') return false;
      last_chunk = c + 1;
      break;
    }
    vector<size_t> first_of(last_chunk + 1, 0);
    for (int c = 0; c < last_chunk; c++) first_of[c + 1] = first_of[c] + parsed[c].reads.size();
    recs[k].resize(first_of[last_chunk]);
#pragma omp parallel for schedule(dynamic, 1) num_threads(T)
    for (int c = 0; c < last_chunk; c++) {
      size_t i = first_of[c];
      for (const View &v : parsed[c].reads)
        recs[k][i++] = {&v, v.owned >= 0 ? parsed[c].arena[v.owned].data() : v.seq, mate_id(v.hdr, v.hdr_len)};
    }
  }
  auto pair_view = [](const Rec &a, const Rec &b, View &m, MateSeqs &s) {
    m.hdr = a.v->hdr; m.hdr_len = (uint32_t)a.id;
    m.qual = NULL; m.qual_len = 0; m.owned = -1; m.seq = NULL;
    s = {a.seq, b.seq, a.v->seq_len, b.v->seq_len, true};
    const uint64_t len = (uint64_t)s.n1 + 1 + s.n2;
    m.seq_len = (uint32_t)std::min<uint64_t>(len, UINT32_MAX);
    return len;
  };
  // Every pair before the first one that stops the merger (a malformed header, a name mismatch) is merged as a pair
  // (PAIRS in MergeOrder): those are merged in parallel, and MergeOrder goes on from the first stop.
  const size_t n_pair = std::min(recs[0].size(), recs[1].size());
  size_t first_stop = n_pair;
#pragma omp parallel for schedule(static) num_threads(T) reduction(min : first_stop)
  for (size_t i = 0; i < n_pair; i++) {
    const Rec &a = recs[0][i], &b = recs[1][i];
    if (a.id < 0 || b.id < 0 || (Check_names && (a.id != b.id || memcmp(a.v->hdr, b.v->hdr, a.id) != 0))) first_stop = std::min(first_stop, i);
  }
  merged.resize(first_stop);
  mates.resize(first_stop);
  uint64_t longest = 0;
#pragma omp parallel for schedule(static) num_threads(T) reduction(max : longest)
  for (size_t i = 0; i < first_stop; i++) longest = std::max(longest, pair_view(recs[0][i], recs[1][i], merged[i], mates[i]));
  if (longest > (280ull << 20)) die(EX_DATAERR, "a single sequence is longer than 280 Mbp: not supported");
  size_t next_of[2] = {first_stop, first_stop};
  const Rec *cur[2] = {NULL, NULL};
  int last_read = 0;
  auto read = [&](int k) {
    if (next_of[k] >= recs[k].size()) return 0;
    cur[k] = &recs[k][next_of[k]++];
    last_read = k;
    return cur[k]->id < 0 ? -1 : 1;
  };
  auto same = [&] { return cur[0]->id == cur[1]->id && memcmp(cur[0]->v->hdr, cur[1]->v->hdr, cur[0]->id) == 0; };
  MergeOrder order;
  for (;;) {
    const MergeOrder::Kind kind = order.next(read, same);
    if (kind == MergeOrder::END) break;
    if (kind == MergeOrder::MALFORMED) {
      const View &v = *cur[last_read]->v;
      Pair_error = malformed_message(!fastq, fastq ? '@' : '>', v.hdr, v.hdr_len, v.hdr + v.hdr_len < in[last_read].fend);
      break;
    }
    if (kind == MergeOrder::MISMATCH) {
      Pair_error = mismatch_message(cur[0]->v->hdr, cur[0]->id, cur[1]->v->hdr, cur[1]->id);
      break;
    }
    View m;
    MateSeqs s;
    uint64_t len;
    if (kind == MergeOrder::PAIR) {
      len = pair_view(*cur[0], *cur[1], m, s);
    } else {
      const Rec *a = kind == MergeOrder::ONLY2 ? cur[1] : cur[0];
      m.hdr = kind == MergeOrder::EMPTY_N ? "" : a->v->hdr;
      m.hdr_len = kind == MergeOrder::EMPTY_N ? 0 : (uint32_t)a->id;
      m.qual = NULL; m.qual_len = 0; m.owned = -1; m.seq = NULL;
      s = kind == MergeOrder::EMPTY_N ? MateSeqs{NULL, NULL, 0, 0, true} : MateSeqs{a->seq, NULL, a->v->seq_len, 0, false};
      len = m.seq_len = s.n1 + s.joined;
    }
    if (len > (280ull << 20)) die(EX_DATAERR, "a single sequence is longer than 280 Mbp: not supported");
    merged.push_back(m);
    mates.push_back(s);
  }
  return true;
}

// --extract over the mapped files: the lines of the FASTQ record whose sequence line starts at `seq`
static void fastq_record_at(const char *seq, const PlainInput &f, const char *&m, size_t &n) {
  const char *a = seq - 1;                                         // the header line's '\n'
  while (a > f.base && a[-1] != '\n') a--;
  const char *e = seq;
  for (int k = 0; k < 3 && e < f.fend; k++) { e = line_end(e, f.fend); if (e < f.fend) e++; }
  m = a; n = (size_t)(e - a);
}

// One mapped record as extract_reads reads it.  Merged mates (pair != NULL) take both records from the mapped files; a
// record with no mate 1 (mate file 2's rest, the lone "N") is never visited.
static XRec mapped_record(const View &v, const MateSeqs *pair, const PlainInput (&in)[2], bool fastq) {
  XRec x{v.hdr, v.hdr_len, v.hdr, v.hdr_len, NULL, 0, NULL, 0, true};
  const PlainInput &f = in[0];
  if (pair) {
    if (!pair->s1 || pair->s1 < f.base || pair->s1 >= f.fend + 1) { x.visited = false; return x; }
    fastq_record_at(pair->s1, f, x.m1, x.n1);
    if (pair->joined) fastq_record_at(pair->s2, in[1], x.m2, x.n2);
    x.hdr = x.m1 + 1; x.hdr_len = x.n1 - 1;
  } else if (fastq) {
    x.m1 = v.hdr - 1;
    const char *e = v.qual + v.qual_len;
    x.n1 = (size_t)((e < f.fend ? e + 1 : e) - x.m1);
  } else {                                                         // the sequence lines up to the next '>' line
    const char *a = v.hdr + v.hdr_len < f.fend ? v.hdr + v.hdr_len + 1 : f.fend, *e = a;
    while (e < f.fend && *e != '>') { e = line_end(e, f.fend); if (e < f.fend) e++; }
    x.m1 = a; x.n1 = (size_t)(e - a);
  }
  return x;
}

static bool process_file_parallel(kuq_ctx *ctx0, const char *filename, const char *mate2) {
  const vector<kuq_ctx *> ctxs = All_ctx.empty() ? vector<kuq_ctx *>{ctx0} : All_ctx;
  const int G = (int)ctxs.size();
  PlainInput in[2];
  if (!in[0].map(filename)) return false;
  // mate files: both plain, both starting with a header (determine_file_type, read_merger.pl:199-216)
  auto header_first = [](const PlainInput &f) { return f.base[0] == '>' || f.base[0] == '@'; };
  if (mate2 && (!in[1].map(mate2) || !header_first(in[0]) || !header_first(in[1]))) {
    in[0].unmap(); in[1].unmap();
    return false;
  }
  const bool fastq_records = in[0].base[0] == '@';                   // determine_input_file_type; mate files: :66-75
  const bool fastq = fastq_records && !mate2;                        // merged records are FASTA
  const int T = std::max(1, Num_threads);
  double T0__ = now_s();
  for (int k = 0; k < (mate2 ? 2 : 1); k++) in[k].parse(fastq_records, T);
  vector<ChunkParse> &parsed = in[0].parsed;
  const int n_chunks = (int)parsed.size();
  TICK("parse");
  vector<View> merged;
  vector<MateSeqs> mates;
  if (mate2 && !merge_parsed(in, fastq_records, T, merged, mates)) {
    in[0].unmap(); in[1].unmap();
    return false;
  }
  // the reference stops at the first record its reader rejects
  size_t n_total = 0;
  int last_chunk = mate2 ? 0 : n_chunks;
  for (int c = 0; c < last_chunk; c++) {
    n_total += parsed[c].reads.size();
    if (parsed[c].stopped) {
      if (!parsed[c].warning.empty()) fprintf(stderr, "classify: %s\n", parsed[c].warning.c_str());
      last_chunk = c + 1;
      break;
    }
  }
  vector<size_t> first_of(last_chunk + 1, 0);
  for (int c = 0; c < last_chunk; c++) first_of[c + 1] = first_of[c] + parsed[c].reads.size();
  n_total = mate2 ? merged.size() : first_of[last_chunk];
  // flat views of all reads + cumulative sequence length (parallel per chunk, chunk bases from a short serial scan)
  vector<const View *> rv(n_total);
  vector<uint64_t> cum(n_total + 1);
  if (mate2) {
    cum[0] = 0;
    for (size_t i = 0; i < n_total; i++) { rv[i] = &merged[i]; cum[i + 1] = cum[i] + merged[i].seq_len; }
  } else {
    vector<uint64_t> chunk_nt(last_chunk + 1, 0);
#pragma omp parallel for schedule(dynamic, 1) num_threads(T)
    for (int c = 0; c < last_chunk; c++) {
      uint64_t nt = 0;
      for (const View &v : parsed[c].reads) nt += v.seq_len;
      chunk_nt[c + 1] = nt;
    }
    for (int c = 0; c < last_chunk; c++) chunk_nt[c + 1] += chunk_nt[c];
#pragma omp parallel for schedule(dynamic, 1) num_threads(T)
    for (int c = 0; c < last_chunk; c++) {
      uint64_t run = chunk_nt[c];
      size_t i = first_of[c];
      for (const View &v : parsed[c].reads) { rv[i] = &v; cum[i] = run; run += v.seq_len; i++; }
    }
    cum[n_total] = chunk_nt[last_chunk];
  }
  auto chunk_of = [&](size_t i) { return (int)(std::upper_bound(first_of.begin(), first_of.end(), i) - first_of.begin()) - 1; };
  // work units and batches (kuq_batches.h): batches end at unit boundaries
  struct Cut { size_t begin, end; };
  vector<Cut> batches;
  {
    BatchCutter cutter(batch_limits(96ull << 20, true, true));
    size_t begin = 0;
    for (size_t i = 0; i < n_total; i++) {
      const uint64_t len = cum[i + 1] - cum[i];
      if (len > SLOT_NT) die(EX_DATAERR, "a single sequence is longer than 280 Mbp: not supported");
      const BatchCutter::Step st = cutter.next(len);
      if (st.before) { batches.push_back({begin, i}); begin = i; }
      if (st.after) { batches.push_back({begin, i + 1}); begin = i + 1; }
    }
    const size_t end = n_total - cutter.drop();
    if (end > begin) batches.push_back({begin, end});
  }
  TICK("units+batches");
  // ---- pipeline: a filler thread gathers batch b + 2 into pinned memory and submits it while the GPUs classify batch
  // b + 1 and this thread formats batch b.  Batch b runs on device b % G in slot (b / G) % NS and is staged in
  // st[b % (NS * G)]; a slot (and its staging set) is reused only after its batch has been formatted, because the
  // results live in the slot's pinned buffers until then.
  const int NS = 3;
  // Worker teams of the pipeline: more than ~32 OpenMP threads spinning at their barriers starve the thread that talks
  // to the CUDA driver (OMP_WAIT_POLICY=passive avoids it too), and the formatting is not the bottleneck beyond that.
  const int Tf = std::min(8, std::max(1, T / 4)), Te = std::min(24, std::max(1, T - Tf));
  // staging sets live for the whole process: pinned allocations cost tens of ms each, the second input file reuses them
  static vector<Stage> st;
  if (st.empty() && !Prealloc_stages.empty()) st.swap(Prealloc_stages);
  if (st.size() < (size_t)NS * G) st.resize((size_t)NS * G);
  double t_fill = 0, t_emit = 0, t_wait = 0, t_submit = 0;
  auto fill = [&](Stage &s, const Cut &b) {
    s.begin = b.begin; s.end = b.end;
    const size_t n = b.end - b.begin;
    prepare_stage(s, cum[b.end] - cum[b.begin], n);
    const uint64_t c0 = cum[b.begin];
#pragma omp parallel for schedule(static) num_threads(Tf)
    for (size_t i = 0; i < n; i++) {
      const View &v = *rv[b.begin + i];
      s.offs[i] = cum[b.begin + i] - c0;
      if (mate2) {                                                   // seq1 . "N" . seq2 (read_merger.pl:187-191)
        const MateSeqs &m = mates[b.begin + i];
        char *d = s.bases + s.offs[i];
        memcpy(d, m.s1, m.n1);
        if (m.joined) { d[m.n1] = 'N'; memcpy(d + m.n1 + 1, m.s2, m.n2); }
        continue;
      }
      const char *src = v.owned >= 0 ? parsed[chunk_of(b.begin + i)].arena[v.owned].data() : v.seq;
      memcpy(s.bases + s.offs[i], src, v.seq_len);
    }
    s.offs[n] = cum[b.end] - c0;
  };
  Writer writer;
  writer.start();
  auto emit = [&](Stage &s, const kuq_batch_result &res) {
    const size_t n = s.end - s.begin;
    const int parts = Te;
    OutJob job = writer.take(parts);
    auto view_of = [&](size_t i) {
      const View &v = *rv[s.begin + i];
      return ReadView{v.hdr, v.hdr_len, s.bases + s.offs[i], v.seq_len, v.qual, v.qual_len};
    };
    if (Extract_now) Extract_selected += res.n_extract;
    const bool extract = Extract_now && (res.n_extract || Extract_invert);
    job.extract_selected = Extract_selected > 0;
    auto x_of = [&](size_t i) { return mapped_record(*rv[s.begin + i], mate2 ? &mates[s.begin + i] : NULL, in, fastq_records); };
#pragma omp parallel for schedule(static, 1) num_threads(Te)
    for (int pi = 0; pi < parts; pi++) {
      format_reads(view_of, n * pi / parts, n * (pi + 1) / parts, res, 0, fastq, job.kraken[pi], job.classified[pi], job.unclassified[pi],
                   job.script.empty() ? NULL : &job.script[pi]);
      if (extract) extract_reads(x_of, n * pi / parts, n * (pi + 1) / parts, res, 0, !fastq_records, job.extract[pi]);
    }
    writer.push(std::move(job));
    book_batch(n, s.offs[n], res.n_classified);
  };
  // batch bi: device bi % G, slot (bi / G) % NS, staging set bi % (NS * G)
  std::mutex pm;
  std::condition_variable pcv;
  size_t submitted = 0, collected = 0;
  string filler_error;
  std::thread filler([&] {
    for (size_t bi = 0; bi < batches.size(); bi++) {
      {
        std::unique_lock<std::mutex> l(pm);
        pcv.wait(l, [&] { return bi - collected < (size_t)(NS * G); });        // the slot's previous batch is formatted
      }
      const int k = (int)(bi % ((size_t)NS * G));
      kuq_ctx *c = ctxs[bi % G];
      double a = now_s();
      fill(st[k], batches[bi]);
      double b = now_s();
      if (kuq_submit_batch(c, (uint32_t)((bi / G) % NS), st[k].bases, st[k].offs, (uint32_t)(st[k].end - st[k].begin), NULL, 0)) {
        std::lock_guard<std::mutex> l(pm);
        filler_error = kuq_last_error(c);
        submitted = batches.size() + 1;
        pcv.notify_all();
        return;
      }
      t_fill += b - a; t_submit += now_s() - b;
      { std::lock_guard<std::mutex> l(pm); submitted = bi + 1; }
      pcv.notify_all();
    }
  });
  for (size_t bj = 0; bj < batches.size(); bj++) {
    {
      std::unique_lock<std::mutex> l(pm);
      pcv.wait(l, [&] { return submitted > bj; });
      if (!filler_error.empty()) { l.unlock(); filler.join(); die(EX_SOFTWARE, filler_error); }
    }
    const int k = (int)(bj % ((size_t)NS * G));
    kuq_ctx *c = ctxs[bj % G];
    kuq_batch_result res;
    double c0 = now_s();
    if (kuq_wait_batch(c, (uint32_t)((bj / G) % NS), &res)) { filler.detach(); die(EX_SOFTWARE, kuq_last_error(c)); }
    double d = now_s();
    emit(st[k], res);
    t_wait += d - c0; t_emit += now_s() - d;
    { std::lock_guard<std::mutex> l(pm); collected = bj + 1; }
    pcv.notify_all();
  }
  filler.join();
  TICK("pipeline");
  { double w0 = now_s(); writer.finish(); if (Timing) fprintf(stderr, "\n[timing] writer drain %.3f s\n", now_s() - w0); }
  if (Timing) fprintf(stderr, "\n[timing] fill %.3f submit %.3f (filler thread, %d threads) | wait %.3f emit %.3f s (%d threads) over %zu batches on %d device(s)\n",
                      t_fill, t_submit, Tf, t_wait, t_emit, Te, batches.size(), G);
  for (kuq_ctx *c : ctxs) if (kuq_finish(c)) die(EX_SOFTWARE, kuq_last_error(c));
  TICK("kuq_finish (harvest)");
  // tearing down a multi-GB mapping takes ~0.1 s of page-table work nobody has to wait for
  std::thread([b0 = in[0].base, s0 = in[0].size, b1 = in[1].base, s1 = in[1].size] {
    munmap((void *)b0, s0);
    if (b1) munmap((void *)b1, s1);
  }).detach();
  TICK("unmap (detached)");
  (void)ctx0;
  return true;
}

// The batches of the inputs, file after file, read one at a time and cut by kuq_batches.h.  A read that closes a batch
// before itself is held over and starts the next batch.  `extract`: the batches keep the reads' lines (--extract).  The
// merger's stop goes to *pair_error and the messages of a malformed record to *log (NULL: stderr at once).  An input that
// cannot be opened ends the batches: `fail` is then EX_NOINPUT, with the message in fail_msg.
struct BatchReader {
  vector<pair<const char *, const char *>> files;
  size_t fi = 0;
  bool open = false, held = false, extract;
  string *pair_error, *log;
  int fail = 0;
  string fail_msg;
  InputReader reader;
  BatchCutter cutter;
  Read r;
  BatchCutter::Step step;
  string held_bases, held_raw;
  RawRec rr{0, 0, 0, true};
  BatchReader(const vector<pair<const char *, const char *>> &f, const BatchLimits &lim, bool extract, string *pair_error = &Pair_error,
              string *log = NULL)
      : files(f), extract(extract), pair_error(pair_error), log(log), cutter(lim) {}
  void push(Batch &b) {
    b.reads.push_back(r);
    b.offs.push_back(b.bases.size());
    b.units.push_back(step.unit);
    if (extract) b.raw_recs.push_back(rr);
  }
  bool next(Batch &b) {
    b.clear();
    if (held) {
      held = false;
      b.fastq = reader.fastq();
      r.seq_off = 0;
      b.bases += held_bases;
      b.raw += held_raw;
      rr.off = 0;
      push(b);
      if (step.after) return true;
    }
    for (; fi < files.size(); fi++) {
      if (!open) {
        reader = InputReader();
        reader.single.log = log;
        reader.pair.error = pair_error;
        fail_msg = reader.open(files[fi].first, files[fi].second);
        if (!fail_msg.empty()) {
          fail = EX_NOINPUT;
          fi = files.size();
          return false;
        }
        open = true;
      }
      b.fastq = reader.fastq();
      reader.keep_raw(extract ? &b.raw : NULL);
      for (;;) {
        const size_t x0 = b.raw.size();
        if (!reader.valid() || !reader.next(r, b.bases)) break;
        rr = RawRec{x0, (uint32_t)(b.raw.size() - x0 - reader.raw_n2()), reader.raw_n2(), reader.raw_visited()};
        if (cutter.lim.slot_nt && r.seq_len > cutter.lim.slot_nt) die(EX_DATAERR, "a single sequence is longer than 280 Mbp: not supported");
        step = cutter.next(r.seq_len);
        if (step.before) {
          held_bases.assign(b.bases, r.seq_off, r.seq_len);
          b.bases.resize(r.seq_off);
          held_raw.assign(b.raw, rr.off, string::npos);
          b.raw.resize(rr.off);
          held = true;
          return true;
        }
        push(b);
        if (step.after) return true;
      }
      const size_t keep = b.reads.size() - cutter.drop();     // the end of the file
      b.bases.resize(b.offs[keep]);
      b.reads.resize(keep);
      b.offs.resize(keep + 1);
      b.units.resize(keep);
      if (extract) b.raw_recs.resize(keep);
      cutter.next_file();
      reader.close();
      open = false;
      if (keep) { fi++; return true; }
    }
    return false;
  }
};

static void process_file(kuq_ctx *ctx, const char *filename, const char *mate2) {
  if (!getenv("KUQ_SERIAL_INGEST") && process_file_parallel(ctx, filename, mate2)) return;   // plain files: parallel path
  BatchReader br({{filename, mate2}}, batch_limits(96ull << 20, true, true), Extract_now);
  Batch batches[2];
  int inflight = -1;
  auto wait_write = [&](int which) {
    const Batch &b = batches[which];
    kuq_batch_result res;
    if (kuq_wait_batch(ctx, (uint32_t)which, &res)) die(EX_SOFTWARE, kuq_last_error(ctx));
    write_reads(b, res, 0, b.reads.size());
    book_batch(b.reads.size(), b.bases.size(), res.n_classified);
  };
  // batch `cur` is read while the other one is classified
  for (int cur = 0; br.next(batches[cur]); cur ^= 1) {
    const Batch &b = batches[cur];
    if (kuq_submit_batch(ctx, (uint32_t)cur, b.bases.data(), b.offs.data(), (uint32_t)b.reads.size(), NULL, 0))
      die(EX_SOFTWARE, kuq_last_error(ctx));
    if (inflight >= 0) wait_write(inflight);
    inflight = cur;
  }
  if (br.fail) die(br.fail, br.fail_msg);
  if (inflight >= 0) wait_write(inflight);
  if (kuq_finish(ctx)) die(EX_SOFTWARE, kuq_last_error(ctx));     // work units do not span input files
}

// ---- one sample's run: begin_sample, the layout's classification of its inputs, end_sample --------------------------
// The resident and sharded layouts run one sample at a time; the streamed layout calls both from inside its rounds,
// which may hold the batches of several samples.
struct SheetRun {
  vector<Sample> samples;
  bool sheet = false;
  TaxDB *tax = NULL;
  vector<map<uint32_t, uint64_t>> db_counts;     // records per taxid of each database (the .counts files)
  bool genome_sizes_read = false;
  int status = 0;
  struct timeval tv1;
};
static SheetRun Run;

// The "classify: sample" line, a clean slate on every context (the staged database(s) serve the next sample), the
// sample's outputs and its totals
static void begin_sample(size_t si) {
  const Sample &sample = Run.samples[si];
  if (Run.sheet) {
    cerr << "classify: sample " << sample.name << " (" << si + 1 << " of " << Run.samples.size() << ")" << endl;
    Sample_label = sample.name;
    Kraken_output_file = sample.kraken;
    Report_output_file = sample.report;
    Classified_output_file = sample.classified;
    Unclassified_output_file = sample.unclassified;
    Print_classified = !sample.classified.empty();
    Print_unclassified = !sample.unclassified.empty();
    Print_kraken = true;
  }
  if (si) {
    double T0__ = now_s();
    for (kuq_ctx *c : All_ctx) if (kuq_reset_counts(c)) die(EX_SOFTWARE, kuq_last_error(c));
    TICK("reset_counts");
  }
  total_classified = total_sequences = total_bases = 0;
  Extract_now = Extract && !sample.extract.empty();
  Extract_selected = 0;
  if (Extract_now) Extract_out.open(sample.extract);
  Translate_now = !sample.translate.empty();
  Translate_stored.clear();
  if (Translate_now) Translate_out.open(sample.translate);
  if (Mpa) {                                                      // the script names a column after its Kraken file
    Mpa_counts.emplace_back();
    const string &k = Run.sheet ? sample.kraken : Kraken_output_file;
    Mpa_ids.push_back(!k.empty() && k != "off" && k != "-" ? k : Run.sheet ? sample.name : "-");
  }
  if (Print_classified) Classified_out.open(Classified_output_file);
  if (Print_unclassified) Unclassified_out.open(Unclassified_output_file);
  if (!Kraken_output_file.empty()) {
    if (Kraken_output_file == "off" || Kraken_output_file == "-") Print_kraken = false;   // classify.cpp:233-235
    else { cerr << "Writing Kraken output to " << Kraken_output_file << endl; Kraken_out.open(Kraken_output_file); }
  } else {
    Kraken_out.open("-");
  }
  gettimeofday(&Run.tv1, NULL);
}

// The per-taxon state of every context finished and joined, the stats block, the report, the outputs closed and the
// merger's stop turned into the exit status
static void end_sample(size_t si) {
  const Sample &sample = Run.samples[si];
  kuq_ctx *ctx = All_ctx[0];
  for (kuq_ctx *c : All_ctx) if (kuq_finish(c)) die(EX_SOFTWARE, kuq_last_error(c));
  // the other devices' per-taxon state joins the first one's (classify.cpp:542-544 across GPUs)
  {
    double T0__ = now_s();
#ifdef EXACT_COUNTING
    // a set that spilled to host memory (KUQ_EXACT_HOST_BUDGET) is counted part by part on every context instead
    uint64_t spills = 0, spilled = 0;
    for (kuq_ctx *c : All_ctx) {
      uint64_t s = 0, p = 0;
      if (kuq_exact_spill_info(c, &s, &p)) die(EX_SOFTWARE, kuq_last_error(c));
      spills += s;
      spilled += p;
    }
    Exact_settled = spilled > 0;
    if (Exact_partitioned || Exact_settled) {
      for (size_t g = 1; g < All_ctx.size(); g++)
        if (kuq_merge_counters_into(ctx, All_ctx[g])) die(EX_SOFTWARE, kuq_last_error(ctx));
    }
    if (Exact_settled) {
      double S0 = now_s();
      if (kuq_exact_settle(All_ctx.data(), (uint32_t)All_ctx.size())) die(EX_SOFTWARE, kuq_last_error(ctx));
      fprintf(stderr, "classifyExact: the exact k-mer set spilled to host memory %llu times (%llu pairs held there at the end "
                      "of the run) and was counted by k-mer part\n", (unsigned long long)spills, (unsigned long long)spilled);
      if (Timing) fprintf(stderr, "[timing] exact set settled from host memory in %.3f s\n", now_s() - S0);
    } else if (Exact_partitioned) {
      if (kuq_exact_partition(All_ctx.data(), (uint32_t)All_ctx.size())) die(EX_SOFTWARE, kuq_last_error(ctx));
    }
    for (size_t g = 1; g < All_ctx.size() && !Exact_partitioned && !Exact_settled; g++)
      if (kuq_merge_into(ctx, All_ctx[g])) die(EX_SOFTWARE, kuq_last_error(ctx));
#else
    for (size_t g = 1; g < All_ctx.size(); g++)
      if (kuq_merge_into(ctx, All_ctx[g])) die(EX_SOFTWARE, kuq_last_error(ctx));
#endif
    if (All_ctx.size() > 1) TICK("merge");
#ifdef EXACT_COUNTING
    for (size_t g = 0; g < All_ctx.size() && Timing; g++) {
      uint64_t slots = 0, pairs = 0, grown = 0;
      if (kuq_exact_info(All_ctx[g], &slots, &pairs, &grown)) die(EX_SOFTWARE, kuq_last_error(All_ctx[g]));
      fprintf(stderr, "[timing] exact set of context %zu: %llu slots, %llu pairs, grown %llu times\n", g, (unsigned long long)slots,
              (unsigned long long)pairs, (unsigned long long)grown);
    }
#endif
  }
  struct timeval tv1 = Run.tv1, tv2;
  gettimeofday(&tv2, NULL);
  {                                                                 // report_stats, classify.cpp:361-375
    double seconds = get_seconds(tv1, tv2);
    cerr << "\r";
    fprintf(stderr, "%llu sequences (%.2f Mbp) processed in %.3fs (%.1f Kseq/m, %.2f Mbp/m).\n", total_sequences,
            total_bases / 1.0e6, seconds, total_sequences / 1.0e3 / (seconds / 60), total_bases / 1.0e6 / (seconds / 60));
    fprintf(stderr, "  %llu sequences classified (%.2f%%)\n", total_classified, total_classified * 100.0 / total_sequences);
    fprintf(stderr, "  %llu sequences unclassified (%.2f%%)\n", total_sequences - total_classified,
            (total_sequences - total_classified) * 100.0 / total_sequences);
  }

  if (!Report_output_file.empty() && Report_output_file != "off") {
    gettimeofday(&tv1, NULL);
    cerr << "Writing report file to " << Report_output_file << "  ..\n";
    TaxDB &tax = *Run.tax;
    // the genome sizes are read (and .counts written) once per process, as by the first separate run
    for (size_t d = 0; d < DB_filenames.size() && !Run.genome_sizes_read; d++) {   // classify.cpp:262-285, once per database
      const string fname = DB_filenames[d] + ".counts";
      bool counts_ok = false;
      {
        ifstream ifs(fname);
        if (ifs.good()) {
          if (ifs.peek() == ifstream::traits_type::eof()) cerr << "Kmer counts file is empty - trying to regenerate ..." << endl;
          else counts_ok = true;
        }
      }
      if (!counts_ok) {                                               // classify.cpp:275-284 via kuq_db_taxids
        cerr << "Writing kmer counts to " << fname << "... [only once for this database, may take a while] " << endl;
        ofstream ofs(fname);
        for (auto &kv : Run.db_counts[d]) ofs << kv.first << '\t' << kv.second << '\n';
      }
      {
        cerr << "Reading genome sizes from " << fname << " ...";
        ifstream in(fname);
        // readGenomeSizes, taxdb.hpp:868-885, loop kept literally: `while (!eof) { in >> id >> size; set(...) }` counts
        // the last line of a newline-terminated file twice (the failed extraction leaves the variables unchanged);
        // the reference's `cov` column depends on it, so the drop-in reproduces it.
        uint32_t taxid = 0;
        uint64_t size = 0;
        while (!in.eof()) {
          in >> taxid >> size;
          tax.set_genome_size(taxid, size);
        }
        cerr << " done" << endl;
      }
    }
    Run.genome_sizes_read = true;
    ostringstream rep;
    double T0__ = now_s();
    print_report(ctx, tax, rep);
    TICK("print_report");
    OutStream ro;
    ro.open(Report_output_file, true);                              // appended to the wrapper's 2 header lines
    ro.write(rep.str());
    ro.close();
    gettimeofday(&tv2, NULL);
    fprintf(stderr, "Report finished in %.3f seconds.\n", get_seconds(tv1, tv2));
  }
  cerr << "Finishing up ..." << endl;
  Kraken_out.close();
  Classified_out.close();
  Unclassified_out.close();
  string().swap(Extract_pending);                                  // no read was selected: nothing is written
  Extract_out.close();
  Translate_out.close();
  // the records before the merger's stop are classified and written, like the wrapper's run on its partial output; the
  // samples after it still run
  if (!Pair_error.empty()) {
    cerr << "classify: " << (Run.sheet ? "sample " + sample.name + ": " : "") << Pair_error << endl;
    Run.status = EX_DATAERR;
    Pair_error.clear();
  }
}

// ---- chunked mode: `-x size` with a database that does not fit (process_file_with_db_chunk, classify.cpp:566-791) --
// Ranges of minimizer bins whose records (12 bytes each in HBM) + index slice fit the budget: kuq_ranges.h.
static vector<pair<uint64_t, uint64_t>> plan_ranges(const uint64_t *offsets, uint64_t n_bins, uint64_t budget) {
  vector<pair<uint64_t, uint64_t>> ranges;
  if (!plan_ranges(offsets, n_bins, budget, 12, ranges)) die(EX_SOFTWARE, "a single minimizer bin exceeds the chunk budget; raise -x");
  return ranges;
}

// ---- databases that do not fit the HBM budget: streamed through two range buffers ----------------------------------
// One database larger than the budget (the -x path, process_file_with_db_chunk, classify.cpp:566-791), or several
// databases that do not fit it together (`-d a -d b`, classify.cpp:928-936), on the run's G >= 1 contexts.  Every
// database keeps the ranges plan_ranges cuts at the chunk budget, whatever G, and GPU g streams a contiguous group of
// them (kuq_ranges.h, group_ranges) over its own host link (kuq_stream_*: the next range travels while the current one is
// looked up).  The input is read in rounds that stay in HBM next to the two range buffers: every GPU holds every batch
// of a round, and each batch has one owner that alone holds its per-window ids (5 bytes per base + 8 per read, + 4 per
// read of unit ids, on one GPU), as many batches as fit the tightest context and at least one.  Each round goes through
// the databases in command-line order, and every GPU stores its hits straight into the owner's buffer (peer stores when
// the owner is another GPU).  The first database writes its hits, a stored zero as KUQ_CODE_FOUND_ZERO; the later ones
// only fill the windows that no earlier database answered (KUQ_LOOKUP_FILL_EMPTY).  Then the owners resolve the round's
// batches, written in input order.  One database keeps the -x rule (one sketch per taxon; batches need not hold whole
// work units); several take the per-work-unit rule of the preloaded path, which is the reference's rule for `-d a -d b`
// without -x.  stage_streamed runs once per process: the ranges, the taxids of every record and the pinned registration
// of the mapped files; it returns the first context that staged a range (a GPU's group may be empty).
// classify_streamed runs once per process: the rounds of reads of every sample, each through every range.
struct Streamed {
  struct Plan {
    DbFile f;
    vector<pair<uint64_t, uint64_t>> ranges;
    vector<size_t> group;                                          // GPU g streams ranges [group[g], group[g + 1])
  };
  vector<Plan> plans;
  vector<kuq_ctx *> ctxs;
  bool unit_rule = false;
  uint64_t max_rec = 1, max_bins = 1, round_bytes = 0, batch_nt = 1;
  uint64_t tail_bytes = 0;                                         // a round's batches held past an end of a sample
  vector<const void *> pinned;                                     // registered mappings, unregistered at the end
  vector<uint32_t> open_nt, open_type;                             // per context: what its range buffers are open for
};

static int stage_streamed(Streamed &sm, const vector<kuq_ctx *> &ctxs, const vector<int> &ctx_devices, const vector<Mapped> &kdbs,
                          const vector<Mapped> &idxs, const vector<DbFile> &files, uint64_t range_budget, uint64_t hbm_budget,
                          vector<map<uint32_t, uint64_t>> &db_counts) {
  const size_t n_db = kdbs.size();
  const int G = (int)ctxs.size();
  const bool unit_rule = sm.unit_rule = n_db > 1;
  sm.ctxs = ctxs;
  sm.open_nt.assign(G, 0);
  sm.open_type.assign(G, 0);
  vector<Streamed::Plan> &plans = sm.plans;
  plans.resize(n_db);
  uint64_t &max_rec = sm.max_rec, &max_bins = sm.max_bins;
  for (size_t d = 0; d < n_db; d++) {
    Streamed::Plan &pl = plans[d];
    pl.f = files[d];
    pl.ranges = plan_ranges(pl.f.offsets, pl.f.n_bins, range_budget);
    pl.group = group_ranges(pl.f.offsets, pl.ranges, G, 12);
    for (auto &rg : pl.ranges) {
      max_rec = std::max<uint64_t>(max_rec, pl.f.offsets[rg.second] - pl.f.offsets[rg.first]);
      max_bins = std::max<uint64_t>(max_bins, rg.second - rg.first);
    }
  }
  // pass 0: the taxids of all records, so that every range numbers taxa identically (also database.kdb.counts); every
  // GPU reads those of its own group
  vector<vector<Slice>> slices(G);
  for (int g = 0; g < G; g++)
    for (size_t d = 0; d < n_db; d++)
      for (size_t c = plans[d].group[g]; c < plans[d].group[g + 1]; c++)
        slices[g].push_back(Slice{d, plans[d].ranges[c].first, plans[d].ranges[c].second});
  stage_slices(ctxs, kdbs, idxs, slices, false, false, db_counts);
  if (n_db == 1) cerr << "Database split into " << plans[0].ranges.size() << " chunks" << endl;
  if (G > 1) {
    string per;
    for (size_t d = 0; d < n_db; d++) {
      per += d ? ", " : "";
      for (int g = 0; g < G; g++) per += (g ? "/" : "") + std::to_string(plans[d].group[g + 1] - plans[d].group[g]);
    }
    fprintf(stderr, "classify: %s streamed over %d GPUs: ranges per GPU %s\n",
            n_db == 1 ? "database" : (std::to_string(n_db) + " databases").c_str(), G, per.c_str());
  }
  share_taxa(ctxs, db_counts);
  if (unit_rule)
    for (kuq_ctx *c : ctxs)
      if (kuq_mark_zero_hits(c, 1)) die(EX_SOFTWARE, kuq_last_error(c));
  // device memory of a round: the budget (and what the card has free, shared among its contexts) minus the two range
  // buffers, on the tightest context (stream_round_bytes)
  const uint64_t range_bytes = 2 * (max_rec * 12 + (max_bins + 1) * 8 + 4096);     // 12 B per record in HBM
  vector<uint64_t> free_b;
  for (kuq_ctx *c : ctxs) free_b.push_back(kuq_device_free_bytes(c));
  const uint64_t round_bytes = sm.round_bytes = stream_round_bytes(ctx_devices, free_b, hbm_budget, range_bytes);
  // An end of a sample in the middle of a round (a sheet run) finds the round's later batches in device memory, where
  // the end of a separate run finds the range buffers, which every round releases after its lookups.  So the later
  // batches may take the range buffers' bytes, plus what the budget keeps from every round on the tightest context:
  // none where the card's free memory limits the round.
  uint64_t unused = UINT64_MAX;
  for (size_t g = 0; g < ctx_devices.size(); g++) {
    uint64_t sharing = 0;
    for (int d : ctx_devices) sharing += d == ctx_devices[g];
    const uint64_t share = (free_b[g] > (2ull << 30) ? free_b[g] - (2ull << 30) : 0) / sharing;
    unused = std::min<uint64_t>(unused, share > hbm_budget ? share - hbm_budget : 0);
  }
  sm.tail_bytes = range_bytes + unused;
  // A batch of b bases takes b bytes on every GPU and 4 b more on its owner (batch_shared_bytes / batch_id_bytes), so G
  // batches, one per owner, take about (G + 4) b per GPU: batches of round / (G + 5) bases let a round give every GPU a
  // batch to resolve.  One GPU: round / 6.
  sm.batch_nt = std::max<uint64_t>(1, std::min<uint64_t>(96ull << 20, round_bytes / (G + 5)));
  uint64_t db_bytes = 0;                                           // what every round copies to the device
  for (size_t d = 0; d < n_db; d++) db_bytes += kdbs[d].size + idxs[d].size;
  if (round_bytes < db_bytes)
    fprintf(stderr, "classify: %llu MiB of device memory per round of reads next to the range buffers, while every round "
                    "copies the %llu MiB of the database(s) again: more device memory (KUQ_HBM_BUDGET) means fewer rounds\n",
            (unsigned long long)(round_bytes >> 20), (unsigned long long)(db_bytes >> 20));
  // Mappings registered as pinned memory (the range copies overlap the lookups only from pinned memory), in command-line
  // order while they take at most half of the host's physical memory together: the rest streams from pageable memory
  // rather than page-locking what the reads and the rest of the host need.
  {
    const uint64_t phys = (uint64_t)sysconf(_SC_PHYS_PAGES) * (uint64_t)sysconf(_SC_PAGESIZE);
    uint64_t locked = 0;
    for (size_t d = 0; d < n_db; d++)
      for (const Mapped *m : {&kdbs[d], &idxs[d]})
        if (locked + m->size <= phys / 2 && kuq_host_register(m->p, m->size) == KUQ_OK) {
          locked += m->size;
          sm.pinned.push_back(m->p);
        }
  }
  if (Timing) fprintf(stderr, "[timing] streamed: %zu database(s), %llu MiB per round\n", n_db, (unsigned long long)(round_bytes >> 20));
  int g0 = 0;
  while (g0 + 1 < G && slices[g0].empty()) g0++;
  return g0;
}

// The batches of the run's samples, sample after sample, each read by a BatchReader of its own (opened when the reading
// reaches the sample) and tagged with its sample; a sample without reads yields one batch without reads, so that its turn
// comes.  Reading runs ahead of the sample being written, so what it finds is kept with the sample and takes effect at
// the sample's turn: the merger's stop, the messages of a malformed record, an input that cannot be opened (nothing is
// read after that one).
struct SampleBatches {
  struct Found { string pair_error, log, fail_msg; int fail = 0; };
  const vector<Sample> &samples;
  BatchLimits lim;
  vector<Found> found;
  size_t si = 0;
  std::unique_ptr<BatchReader> br;
  bool any = false, stopped = false;
  SampleBatches(const vector<Sample> &s, const BatchLimits &l) : samples(s), lim(l), found(s.size()) {}
  bool next(Batch &b) {
    while (si < samples.size() && !stopped) {
      if (!br) {
        br.reset(new BatchReader(files_of(samples[si]), lim, Extract && !samples[si].extract.empty(), &found[si].pair_error, &found[si].log));
        any = false;
      }
      if (br->next(b)) { b.sample = si; any = true; return true; }
      found[si].fail = br->fail;
      found[si].fail_msg = br->fail_msg;
      stopped = br->fail != 0;
      br.reset();
      if (!any) { b.clear(); b.sample = si++; return true; }
      si++;
    }
    return false;
  }
};

// The rounds on G >= 1 GPUs, each streaming its group of every database's ranges over its own link.  A round holds the
// batches of one or more samples, in input order:
//   1. every GPU receives every batch of the round; each batch has one owner (contiguous blocks balanced by bases,
//      round_peak_bytes; with one GPU, GPU 0 owns every batch), which alone holds the batch's id buffer and zeroes it;
//   2. host barrier;
//   3. database by database, in command-line order, one host thread per GPU streams the GPU's group of the database's
//      ranges through its two range buffers and looks every batch up into the owner's id buffer (a peer pointer when the
//      owner is another GPU): the first database stores hits only, the later ones fill the windows still empty;
//   4. host barrier after each database: both slots of every GPU synced, the stream checked; after the last database
//      every GPU releases its range buffers (kuq_stream_close) and the next round opens the stream again;
//   5. the round's batches, in runs of one sample: a later sample's begin_sample at its first batch, the owners resolve the
//      run's batches, one in flight per owner, the results are written in input order and the batches freed on every
//      GPU, and the sample's end_sample after its last batch.
// The lookups write ids only and touch no per-taxon state (no counting in MODE_LOOKUP without shard counting), so a round
// looks up the batches of samples that have not begun; the resolves, which count, run between the sample's
// kuq_reset_counts and its end_sample.
// The barrier of step 4 is what makes KUQ_LOOKUP_FILL_EMPTY correct here: lookup_window_multi reads the owner's word with
// a plain load, which sees the words other GPUs stored over the peer link only because a host barrier and a kernel
// boundary separate the two databases' lookups.  The sharded layout orders its phases with device flags and no host
// barrier, and reads the word with a system-scope load (load_relaxed_sys).  Do not drop this barrier without switching
// to that load.  With one GPU it costs a host sync per database and round but no overlap: kuq_stream_load makes the
// next database's first copy wait on the device for every lookup queued before it anyway.
static void classify_streamed(Streamed &sm) {
  const vector<kuq_ctx *> &ctxs = sm.ctxs;
  const int G = (int)ctxs.size();
  const size_t n_db = sm.plans.size();
  const bool unit_rule = sm.unit_rule;
  const size_t S = Run.samples.size();
  SampleBatches input(Run.samples, batch_limits(sm.batch_nt, unit_rule, false));
  struct DevBatch { void *bases, *offs, *units; };
  vector<Batch> round;
  Batch pending;
  bool have_pending = false;
  size_t n_rounds = 0, begun = 1;                                  // begun: samples whose begin_sample ran
  begin_sample(0);                                                 // the first sample's time includes its first pass
  for (;;) {
    round.clear();
    vector<uint64_t> bases, reads;
    uint64_t tail = 0;                                             // the batches after the round's first end of a sample
    for (;;) {
      if (!have_pending) have_pending = input.next(pending);
      if (!have_pending) break;
      bases.push_back(pending.bases.size());
      reads.push_back(pending.reads.size());
      const bool past_end = !round.empty() && pending.sample != round.front().sample;
      const uint64_t held = past_end ? batch_shared_bytes(bases.back(), reads.back(), unit_rule) + batch_id_bytes(bases.back()) : 0;
      if (!round.empty() && (round_peak_bytes(bases, reads, unit_rule, G) > sm.round_bytes || tail + held > sm.tail_bytes)) {
        bases.pop_back();
        reads.pop_back();
        break;
      }
      tail += held;
      round.push_back(std::move(pending));
      have_pending = false;
    }
    if (round.empty()) break;
    n_rounds++;
    const size_t nb = round.size();
    vector<size_t> first;                                          // GPU g owns batches [first[g], first[g + 1])
    round_peak_bytes(bases, reads, unit_rule, G, &first);
    vector<int> owner(nb);
    for (int g = 0; g < G; g++) for (size_t bi = first[g]; bi < first[g + 1]; bi++) owner[bi] = g;
    // 1. (a pageable copy has left the source once it returns); a batch without reads stands for its sample's turn only
    vector<vector<DevBatch>> dev(G, vector<DevBatch>(nb, DevBatch{NULL, NULL, NULL}));
    vector<uint32_t *> ids(nb, NULL);
    for (size_t bi = 0; bi < nb; bi++) {
      const Batch &b = round[bi];
      if (b.reads.empty()) continue;
      vector<uint64_t> offs(b.offs);
      offs.push_back(offs.back()); offs.push_back(offs.back());
      for (int g = 0; g < G; g++) {
        kuq_ctx *c = ctxs[g];
        DevBatch &d = dev[g][bi];
        d.bases = kuq_device_alloc(c, b.bases.size() + 64);
        d.offs = kuq_device_alloc(c, (b.reads.size() + 4) * 8);
        d.units = unit_rule ? kuq_device_alloc(c, (b.reads.size() + 4) * 4) : NULL;
        if (!d.bases || !d.offs || (unit_rule && !d.units)) die(EX_OSERR, "device allocation for the read batches failed");
        if (kuq_device_memset(c, 0, (char *)d.bases + b.bases.size(), 'N', 64) ||
            kuq_copy_to_device(c, 0, d.bases, b.bases.data(), b.bases.size()) ||
            kuq_copy_to_device(c, 0, d.offs, offs.data(), offs.size() * 8) ||
            (unit_rule && kuq_copy_to_device(c, 0, d.units, b.units.data(), b.units.size() * 4)))
          die(EX_SOFTWARE, kuq_last_error(c));
      }
      kuq_ctx *o = ctxs[owner[bi]];
      ids[bi] = (uint32_t *)kuq_device_alloc(o, batch_id_bytes(b.bases.size()));
      if (!ids[bi]) die(EX_OSERR, "device allocation for the read batches failed");
      if (kuq_device_memset(o, 0, ids[bi], 0, batch_id_bytes(b.bases.size()))) die(EX_SOFTWARE, kuq_last_error(o));
    }
    // 2.
    for (kuq_ctx *c : ctxs) if (kuq_sync_slot(c, 0)) die(EX_SOFTWARE, kuq_last_error(c));
    uint64_t seqs = 0;
    for (const Batch &b : round) seqs += b.reads.size();
    vector<double> stream_s(G, 0.0);
    for (size_t db = 0; db < n_db; db++) {
      const Streamed::Plan &pl = sm.plans[db];
      if (pl.ranges.empty()) continue;                             // a database without records answers nothing
      const uint32_t only_hits = db == 0 ? 1 : KUQ_LOOKUP_FILL_EMPTY;
      // 3. and 4.: every GPU's part returns with its slots and copies synced; the join is the host barrier
      vector<int> ex(G, 0);
#pragma omp parallel for num_threads(G) schedule(static, 1)
      for (int g = 0; g < G; g++) {
        const double t0 = now_s();
        kuq_ctx *c = ctxs[g];
        const size_t lo = pl.group[g], hi = pl.group[g + 1];
        auto part = [&]() -> int {
          // every context opens the stream, an empty group too: the open numbers the taxa, which its resolves need
          const DbFile &f = pl.f;
          if (f.nt != sm.open_nt[g] || f.idx_type != sm.open_type[g]) {
            if ((sm.open_nt[g] && kuq_stream_check(c)) || kuq_stream_open(c, f.k, f.nt, f.idx_type, sm.max_rec, sm.max_bins))
              return EX_DATAERR;
            sm.open_nt[g] = f.nt;
            sm.open_type[g] = f.idx_type;
          }
          if (lo == hi) return 0;
          auto load = [&](uint32_t buf, size_t r) {
            const uint64_t blo = pl.ranges[r].first, bhi = pl.ranges[r].second;
            return kuq_stream_load(c, buf, f.records + f.offsets[blo] * f.pair_sz, f.offsets[bhi] - f.offsets[blo], f.offsets + blo,
                                   blo, bhi);
          };
          if (load(0, lo)) return EX_DATAERR;
          for (size_t r = lo; r < hi; r++) {
            if (kuq_stream_use(c, (uint32_t)((r - lo) & 1))) return EX_SOFTWARE;
            if (r + 1 < hi && load((uint32_t)((r + 1 - lo) & 1), r + 1)) return EX_DATAERR;
            for (size_t bi = 0; bi < nb; bi++) {
              const Batch &b = round[bi];
              if (b.reads.empty()) continue;
              if (kuq_lookup_device(c, (uint32_t)(bi & 1), (const char *)dev[g][bi].bases, (const uint64_t *)dev[g][bi].offs,
                                    (uint32_t)b.reads.size(), b.bases.size(), ids[bi], only_hits))
                return EX_SOFTWARE;
            }
          }
          return kuq_sync_slot(c, 0) || kuq_sync_slot(c, 1) || kuq_stream_check(c) ? EX_SOFTWARE : 0;
        };
        ex[g] = part();
        stream_s[g] += now_s() - t0;
      }
      for (int g = 0; g < G; g++) if (ex[g]) die(ex[g], kuq_last_error(ctxs[g]));
      for (size_t c = 0; c < pl.ranges.size(); c++) {
        if (n_db == 1) fprintf(stderr, "\r Processed %llu sequences (database chunk %zu of %zu)\n", (unsigned long long)seqs, c + 1, pl.ranges.size());
        else fprintf(stderr, "\r Processed %llu sequences (database %zu of %zu, chunk %zu of %zu)", (unsigned long long)seqs, db + 1, n_db,
                     c + 1, pl.ranges.size());
      }
    }
    for (int g = 0; g < G; g++) {
      if (kuq_stream_close(ctxs[g])) die(EX_SOFTWARE, kuq_last_error(ctxs[g]));
      sm.open_nt[g] = sm.open_type[g] = 0;
    }
    // 5. the owner's next batch of the run is queued before this one is written: the results stay in the slot's host
    // buffers until the slot's next collect
    const double t1 = now_s();
    for (size_t a = 0; a < nb;) {
      const size_t si = round[a].sample;
      size_t e = a;
      while (e < nb && round[e].sample == si) e++;
      if (si == begun) { begin_sample(si); begun++; }
      vector<size_t> next(G), end(G);
      for (int g = 0; g < G; g++) {
        next[g] = std::min(std::max(first[g], a), e);
        end[g] = std::max(std::min(first[g + 1], e), next[g]);
      }
      auto resolve_next = [&](int g) {
        while (next[g] < end[g] && round[next[g]].reads.empty()) next[g]++;
        if (next[g] == end[g]) return;
        const size_t bi = next[g]++;
        const Batch &b = round[bi];
        if (kuq_resolve_device(ctxs[g], 0, (const char *)dev[g][bi].bases, (const uint64_t *)dev[g][bi].offs, (uint32_t)b.reads.size(),
                               b.bases.size(), ids[bi], (const uint32_t *)dev[g][bi].units, 0))
          die(EX_SOFTWARE, kuq_last_error(ctxs[g]));
      };
      for (int g = 0; g < G; g++) resolve_next(g);
      for (size_t bi = a; bi < e; bi++) {
        Batch &b = round[bi];
        if (b.reads.empty()) continue;
        const int g = owner[bi];
        kuq_batch_result res;
        if (kuq_collect_device_batch(ctxs[g], 0, &res)) die(EX_SOFTWARE, kuq_last_error(ctxs[g]));
        resolve_next(g);
        write_reads(b, res, 0, b.reads.size());
        book_batch(b.reads.size(), b.bases.size(), res.n_classified);
      }
      for (size_t bi = a; bi < e; bi++) {
        for (int g = 0; g < G; g++)
          for (void *p : {dev[g][bi].bases, dev[g][bi].offs, dev[g][bi].units}) if (p) kuq_device_free(ctxs[g], p);
        if (ids[bi]) kuq_device_free(ctxs[owner[bi]], ids[bi]);
        string().swap(round[bi].bases);
        string().swap(round[bi].raw);
      }
      // the sample ends here unless its batches go on in the next round
      if (e < nb || !have_pending || pending.sample != si) {
        SampleBatches::Found &f = input.found[si];
        cerr << f.log;
        if (f.fail) die(f.fail, f.fail_msg);
        Pair_error = f.pair_error;
        if (si + 1 == S && n_db > 1) {
          string per;
          for (size_t d = 0; d < n_db; d++) per += (d ? "/" : "") + std::to_string(sm.plans[d].ranges.size());
          fprintf(stderr, "\nclassify: %zu databases streamed: %zu rounds, ranges per database %s\n", n_db, n_rounds, per.c_str());
        }
        end_sample(si);
      }
      a = e;
    }
    if (Timing) {
      string per;
      for (int g = 0; g < G; g++) {
        char s[64];
        snprintf(s, sizeof s, "%s%.3f s (%zu batches)", g ? ", " : "", stream_s[g], first[g + 1] - first[g]);
        per += s;
      }
      fprintf(stderr, "\n[timing] streamed round %zu: stream per GPU %s; resolve %.3f s\n", n_rounds, per.c_str(), now_s() - t1);
    }
  }
  if (Run.sheet) fprintf(stderr, "classify: %zu samples streamed in %zu rounds\n", S, n_rounds);
}

// ---- databases that fit the GPUs of the node together but not one of them: minimizer-range shards (SURVEY §8(e).2) --
// GPU g stages bin range g of every database (kuq_ranges.h, plan_shards).  Every GPU scans every batch and looks up the
// k-mers whose minimizer it holds; each hit is stored straight into the id buffer of the GPU that resolves the read (peer
// stores over NVLink); device flags order the phases (no host barrier between GPUs); every GPU resolves a contiguous
// share of the batch.  One process, so peer access instead of CUDA IPC.
//   One database: one lookup phase, and the GPU that finds a hit also does its sketch work; the sketches follow the
//   chunked rule, as for any database the reference could only run with -x.
//   Several databases: one lookup phase per run of databases with equal (nt, index type); a later
//   phase fills only the windows no earlier phase answered on any GPU.  The owners do all the sketch work in the resolve
//   half, with the work-unit ids of the per-work-unit rule (the reference's rule for -d a -d b), so shares hold whole
//   work units.
// shard_loop is what both share: batches, id buffers, flags, shares, phases, resolve and output.
static void shard_loop(const vector<kuq_ctx *> &ctxs, uint32_t n_phases, bool multi, const vector<pair<const char *, const char *>> &files) {
  const int G = (int)ctxs.size();
  const uint64_t R = n_phases;
  vector<Batch> batches;
  {
    // KUQ_SHARD_BATCH_READS closes a batch at the first unit boundary after that many reads (tests: a sharded run of a
    // small input in several batches)
    BatchLimits lim = batch_limits(96ull << 20, true, false);
    if (const char *v = getenv("KUQ_SHARD_BATCH_READS")) lim.batch_reads = std::min<size_t>(lim.batch_reads, std::max<size_t>(1, strtoull(v, NULL, 10)));
    BatchReader input(files, lim, Extract_now);
    for (Batch b; input.next(b);) batches.push_back(std::move(b));
    if (input.fail) die(input.fail, input.fail_msg);
  }
  uint64_t max_bases = 64, max_reads = 4;
  for (auto &b : batches) { max_bases = std::max<uint64_t>(max_bases, b.bases.size()); max_reads = std::max<uint64_t>(max_reads, b.reads.size()); }
  // per GPU and id-buffer parity: the batch, its offsets, the offsets (and unit ids) of the GPU's share, the id buffer
  struct Dev { void *bases[2], *offs[2], *share_offs[2], *units[2], *ids[2], *flags; };
  vector<Dev> dev(G);
  const uint64_t id_bytes = (max_bases + 64) * 4;
  for (int g = 0; g < G; g++) {
    Dev &d = dev[g];
    for (int k = 0; k < 2; k++) {
      d.bases[k] = kuq_device_alloc(ctxs[g], max_bases + 64);
      d.offs[k] = kuq_device_alloc(ctxs[g], (max_reads + 4) * 8);
      d.share_offs[k] = kuq_device_alloc(ctxs[g], (max_reads + 4) * 8);
      d.units[k] = multi ? kuq_device_alloc(ctxs[g], (max_reads + 4) * 4) : NULL;
      d.ids[k] = kuq_device_alloc(ctxs[g], id_bytes);
      if (!d.bases[k] || !d.offs[k] || !d.share_offs[k] || (multi && !d.units[k]) || !d.ids[k])
        die(EX_OSERR, "device allocation for the sharded batches failed");
      if (kuq_device_memset(ctxs[g], 0, d.ids[k], 0, id_bytes)) die(EX_SOFTWARE, kuq_last_error(ctxs[g]));
    }
    d.flags = kuq_device_alloc(ctxs[g], 256);            // [0:8) done counters, [16:24) ready counters
    if (!d.flags || kuq_device_memset(ctxs[g], 0, d.flags, 0, 256)) die(EX_OSERR, "device allocation failed");
    const uint64_t two[8] = {2, 2, 2, 2, 2, 2, 2, 2};     // both id buffers are clean for steps 0 and 1
    if (kuq_copy_to_device(ctxs[g], 0, (char *)d.flags + 128, two, 64) || kuq_sync_slot(ctxs[g], 0)) die(EX_SOFTWARE, kuq_last_error(ctxs[g]));
  }
  vector<uint32_t *> peer_ids(G);
  vector<uint64_t *> peer_done(G), peer_ready(G);
  uint64_t step = 0;
  for (auto &b : batches) {
    const size_t n = b.reads.size();
    const int par = (int)(step & 1);
    const vector<uint32_t> &units = b.units;
    // shares: contiguous; with work-unit ids a share starts where a unit starts (k_unit_decide sees every read of a unit
    // on one GPU), else anywhere (the chunked rule does not depend on units)
    vector<size_t> first(G + 1, 0);
    first[G] = n;
    for (int g = 1; g < G; g++) {
      size_t x = std::max(first[g - 1], std::min(n, (n * g / G) & ~(size_t)1));
      while (multi && x > 0 && x < n && units[x] == units[x - 1]) x++;
      first[g] = x;
    }
    vector<uint64_t> bounds(G + 1);
    for (int g = 0; g <= G; g++) bounds[g] = b.offs[first[g]];
    bounds[0] = 0;
    vector<uint64_t> offs(b.offs);
    offs.push_back(offs.back()); offs.push_back(offs.back());
    // the batch goes to every GPU (a pageable copy may wait for the stream: everything it can wait for is queued)
    for (int g = 0; g < G; g++) {
      const size_t share = first[g + 1] - first[g];
      if (kuq_copy_to_device(ctxs[g], 0, dev[g].bases[par], b.bases.data(), b.bases.size()) ||
          kuq_device_memset(ctxs[g], 0, (char *)dev[g].bases[par] + b.bases.size(), 'N', 64) ||
          kuq_copy_to_device(ctxs[g], 0, dev[g].offs[par], offs.data(), offs.size() * 8) ||
          kuq_copy_to_device(ctxs[g], 0, dev[g].share_offs[par], offs.data() + first[g], (share + 3) * 8) ||
          (multi && share && kuq_copy_to_device(ctxs[g], 0, dev[g].units[par], units.data() + first[g], share * 4)))
        die(EX_SOFTWARE, kuq_last_error(ctxs[g]));
    }
    for (int h = 0; h < G; h++) {
      peer_ids[h] = (uint32_t *)dev[h].ids[par];
      peer_done[h] = (uint64_t *)dev[h].flags;
      peer_ready[h] = (uint64_t *)((char *)dev[h].flags + 128);
    }
    // lookup phases with peer scatter, then the owners resolve — all stream ordered, flags between the GPUs.  Phase r
    // starts when the owners cleared their buffers (r = 0) or every GPU finished phase r - 1, and signals done
    // step * R + r + 1.
    for (uint32_t r = 0; r < n_phases; r++)
      for (int g = 0; g < G; g++) {
        const uint64_t *wait_on = r == 0 ? (const uint64_t *)((char *)dev[g].flags + 128) : (const uint64_t *)dev[g].flags;
        if (kuq_wait_flags(ctxs[g], 0, wait_on, (uint32_t)G, r == 0 ? step + 1 : step * R + r, 0) ||
            (multi ? kuq_lookup_device_peers_run(ctxs[g], 0, (const char *)dev[g].bases[par], (const uint64_t *)dev[g].offs[par],
                                                 (uint32_t)n, b.bases.size(), peer_ids.data(), bounds.data(), (uint32_t)G, r)
                   : kuq_lookup_device_peers(ctxs[g], 0, (const char *)dev[g].bases[par], (const uint64_t *)dev[g].offs[par],
                                             (uint32_t)n, b.bases.size(), peer_ids.data(), bounds.data(), (uint32_t)G)) ||
            kuq_signal_peers(ctxs[g], 0, peer_done.data(), (uint32_t)G, (uint32_t)g, step * R + r + 1))
          die(EX_SOFTWARE, kuq_last_error(ctxs[g]));
      }
    for (int g = 0; g < G; g++) {
      const size_t share = first[g + 1] - first[g];
      if (kuq_wait_flags(ctxs[g], 0, (const uint64_t *)dev[g].flags, (uint32_t)G, (step + 1) * R, 0)) die(EX_SOFTWARE, kuq_last_error(ctxs[g]));
      if (share && kuq_resolve_device(ctxs[g], 0, (const char *)dev[g].bases[par], (const uint64_t *)dev[g].share_offs[par],
                                      (uint32_t)share, b.bases.size(), (const uint32_t *)dev[g].ids[par],
                                      multi ? (const uint32_t *)dev[g].units[par] : NULL, 0))
        die(EX_SOFTWARE, kuq_last_error(ctxs[g]));
      if (kuq_device_memset(ctxs[g], 0, (char *)dev[g].ids[par] + bounds[g] * 4, 0, (bounds[g + 1] - bounds[g]) * 4) ||
          kuq_signal_peers(ctxs[g], 0, peer_ready.data(), (uint32_t)G, (uint32_t)g, step + 3))
        die(EX_SOFTWARE, kuq_last_error(ctxs[g]));
    }
    // results of the shares, in read order
    uint64_t classified = 0;
    for (int g = 0; g < G; g++) {
      const size_t share = first[g + 1] - first[g];
      if (!share) { if (kuq_sync_slot(ctxs[g], 0)) die(EX_SOFTWARE, kuq_last_error(ctxs[g])); continue; }
      kuq_batch_result res;
      if (kuq_collect_device_batch(ctxs[g], 0, &res)) die(EX_SOFTWARE, kuq_last_error(ctxs[g]));
      write_reads(b, res, first[g], first[g + 1]);
      classified += res.n_classified;
    }
    book_batch(n, b.bases.size(), classified);
    step++;
  }
  for (int g = 0; g < G; g++) {
    if (kuq_finish(ctxs[g])) die(EX_SOFTWARE, kuq_last_error(ctxs[g]));
    for (int k = 0; k < 2; k++)
      for (void *p : {dev[g].bases[k], dev[g].offs[k], dev[g].share_offs[k], dev[g].units[k], dev[g].ids[k]})
        if (p) kuq_device_free(ctxs[g], p);
    kuq_device_free(ctxs[g], dev[g].flags);
  }
}

// Staging, once per process: every GPU stages, in command-line order, the bins of its range of each database's run (a
// range of several databases may be empty).  One database is one run, with a non-empty range on every GPU, and the GPU
// that finds a hit counts it (kuq_set_shard_counting).  Returns the runs: shard_loop's lookup phases.
static uint32_t stage_shards(const vector<kuq_ctx *> &ctxs, const vector<Mapped> &kdbs, const vector<Mapped> &idxs,
                             const vector<DbFile> &files, vector<map<uint32_t, uint64_t>> &db_counts) {
  const int G = (int)ctxs.size();
  const size_t n_db = kdbs.size();
  vector<ShardDb> sd;
  for (const DbFile &f : files) sd.push_back(ShardDb{f.offsets, f.nt, f.idx_type});
  const vector<ShardRun> runs = plan_shards(sd, G);
  if (n_db == 1) {
    cerr << "Database sharded over " << G << " GPUs by minimizer range" << endl;
    for (int g = 0; g < G; g++)
      if (runs[0].cut[g + 1] <= runs[0].cut[g]) die(EX_DATAERR, "more GPUs than non-empty minimizer ranges: use fewer devices (KUQ_DEVICES)");
  } else {
    fprintf(stderr, "classify: %zu databases sharded over %d GPUs by minimizer range (%zu lookup phases)\n", n_db, G, runs.size());
  }
  vector<vector<Slice>> slices(G);
  for (int g = 0; g < G; g++)
    for (const ShardRun &run : runs)
      for (size_t d = run.first; d < run.end; d++) {
        uint64_t lo = run.cut[g], hi = run.cut[g + 1];
        if (lo == hi) lo = hi = files[d].n_bins;                     // an empty slice
        slices[g].push_back(Slice{d, lo, hi});
      }
  stage_slices(ctxs, kdbs, idxs, slices, true, false, db_counts);
  for (int g = 0; g < G; g++) {
    uint32_t n_runs = 0;
    if (n_db == 1 ? kuq_set_shard_counting(ctxs[g], 1) : kuq_db_runs(ctxs[g], &n_runs)) die(EX_SOFTWARE, kuq_last_error(ctxs[g]));
    if (n_db > 1 && n_runs != runs.size()) die(EX_SOFTWARE, "the library groups the databases into other lookup runs than the planner");
  }
  share_taxa(ctxs, db_counts);
  return (uint32_t)runs.size();
}

// What a staged database takes in HBM: 12 bytes per record whatever the file's record size (records of k <= 28 databases
// are widened on the way in), plus the index.  Every decision about what fits a card counts these bytes, not the file's.
static uint64_t hbm_bytes(const DbFile &f, const Mapped &idx) { return f.key_ct * 12 + idx.size; }

static uint32_t extract_flags() {
  return (Extract_subtree ? KUQ_EXTRACT_SUBTREE : 0) | (Extract_invert ? KUQ_EXTRACT_INVERT : 0) |
         (Extract_others ? KUQ_EXTRACT_OTHERS : 0) | (Only_classified_kraken_output ? KUQ_EXTRACT_CLASSIFIED_ONLY : 0);
}

// The checks of --extract that need the inputs or the taxonomy, before any device call: an extraction file that is an
// input or another output, FASTA mates (the script dies on -a -p at the first read it prints), and a cycle below the
// listed taxa (the script's get_children recursion never ends).  The taxonomy is read here for the last one.
static void check_extract(const vector<Sample> &samples, TaxDB &tax, bool &tax_read) {
  for (const Sample &s : samples) {
    if (s.extract.empty()) continue;
    set<string> in_keys;
    for (auto &f : s.inputs) {
      in_keys.insert(path_key(f.first));
      if (!f.second.empty()) in_keys.insert(path_key(f.second));
      if (f.second.empty()) continue;
      LineReader lr;
      if (lr.open(f.first.c_str()) && lr.peek() == '>')
        die(EX_USAGE, "--extract with --paired needs FASTQ mates: krakenuniq-extract-reads cannot print FASTA mates (" + f.first + ")");
      lr.close();
    }
    if (s.extract == "-") {
      if (Sample_sheet.empty() && (Kraken_output_file.empty() || Kraken_output_file == "-"))
        die(EX_USAGE, "--extract-out - : the Kraken output goes to standard output (give -o)");
      if (Classified_output_file == "-" || Unclassified_output_file == "-")
        die(EX_USAGE, "--extract-out - : -C or -U writes to standard output");
      continue;
    }
    const string key = path_key(s.extract);
    if (in_keys.count(key)) die(EX_USAGE, "--extract-out " + s.extract + " is one of the inputs");
    if (Sample_sheet.empty())
      for (const string *o : {&Kraken_output_file, &Report_output_file, &Classified_output_file, &Unclassified_output_file})
        if (!o->empty() && *o != "-" && *o != "off" && path_key(*o) == key) die(EX_USAGE, "--extract-out " + s.extract + " is another output");
  }
  if (!Extract_subtree) return;
  if (!tax_read) tax.read(TaxDB_file);                             // (check_scripts may have read it)
  tax_read = true;
  uint32_t n = 0;
  if (kuq_extract_taxa(Extract_taxa.data(), (uint32_t)Extract_taxa.size(), KUQ_EXTRACT_SUBTREE, tax.row_ids.data(),
                       tax.row_parents.data(), (uint32_t)tax.row_ids.size(), NULL, 0, &n))
    die(EX_USAGE, "--extract-subtree: the children of the listed taxa in " + TaxDB_file + " form a cycle");
}

// The checks of --mpa-report and --translate-out, before any database file is opened: -a, where the outputs go (not
// onto an input or another output, one writer of standard output), and the taxonomy's cycles that keep the scripts
// going forever: a cycle of the child lists reachable from 1 (mpa-report's recursion) or of F (translate's walk).  The
// taxonomy is read here.
static void check_scripts(const vector<Sample> &samples, TaxDB &tax, bool &tax_read) {
  bool translate = false;
  for (const Sample &s : samples) translate = translate || !s.translate.empty();
  if (!Mpa && !translate) return;
  if (TaxDB_file.empty()) die(EX_USAGE, "--mpa-report and --translate-out take the taxonomy from the taxDB: give it with -a");
  set<string> in_keys;
  if (!Sample_sheet.empty()) in_keys.insert(path_key(Sample_sheet));
  vector<pair<string, bool>> outs;                 // every output of the run; true: one of this feature's
  for (const Sample &s : samples) {
    for (auto &f : s.inputs) {
      in_keys.insert(path_key(f.first));
      if (!f.second.empty()) in_keys.insert(path_key(f.second));
    }
    if (Sample_sheet.empty()) {
      outs.emplace_back(Kraken_output_file.empty() ? "-" : Kraken_output_file == "-" ? "off" : Kraken_output_file, false);
      for (const string *o : {&Report_output_file, &Classified_output_file, &Unclassified_output_file}) outs.emplace_back(*o, false);
    } else {
      for (const string *o : {&s.kraken, &s.report, &s.classified, &s.unclassified}) outs.emplace_back(*o, false);
    }
    outs.emplace_back(s.extract, false);
    outs.emplace_back(s.translate, true);
  }
  if (Mpa) outs.emplace_back(Mpa_output_file, true);
  for (size_t i = 0; i < outs.size(); i++) {
    const string &o = outs[i].first;
    if (!outs[i].second || o.empty() || o == "off") continue;
    for (size_t j = 0; j < outs.size(); j++) {
      const string &q = outs[j].first;
      if (j == i || q.empty() || q == "off") continue;
      if (o == "-" && q == "-") die(EX_USAGE, "two outputs go to standard output (--mpa-report / --translate-out -)");
      if (o != "-" && q != "-" && path_key(o) == path_key(q)) die(EX_USAGE, o + " is written twice");
    }
    if (o != "-" && in_keys.count(path_key(o))) die(EX_USAGE, o + " is one of the inputs");
  }
  tax.keep_text = true;
  tax.read(TaxDB_file);
  tax_read = true;
  if (Mpa) {
    const uint32_t root = 1;
    uint32_t n = 0;
    if (kuq_extract_taxa(&root, 1, KUQ_EXTRACT_SUBTREE, tax.row_ids.data(), tax.row_parents.data(), (uint32_t)tax.row_ids.size(),
                         NULL, 0, &n))
      die(EX_USAGE, "--mpa-report: the children of taxon 1 in " + TaxDB_file + " form a cycle");
  }
  Script_tax.mpa_format = Translate_mpa;
  if (!Script_tax.build(tax, translate)) die(EX_USAGE, "--translate-out: the parents in " + TaxDB_file + " form a cycle");
}

int main(int argc, char **argv) {
  parse_command_line(argc, argv);
  if (Map_UIDs) die(EX_USAGE, "-I (UID mapping) is not supported by the GPU classify");
  if (DB_filenames.size() != Index_filenames.size()) die(EX_USAGE, "Must specify a index file for each database file");
  const size_t n_db = DB_filenames.size();
  if (n_db > 1 && Populate_memory_size > 0) die(EX_USAGE, "-x with several databases is not supported by the GPU classify");
  const bool sheet = !Sample_sheet.empty();
  vector<Sample> samples;
  if (sheet) {
    samples = read_sample_sheet(Sample_sheet);
  } else {
    Sample s;
    for (int i = optind; i < argc; i += Paired ? 2 : 1) s.inputs.emplace_back(argv[i], Paired ? argv[i + 1] : "");
    s.extract = Extract_output_file;
    s.translate = Translate_output_file;
    samples.push_back(s);
  }
  TaxDB tax;
  bool tax_read = false;
  check_scripts(samples, tax, tax_read);
  if (Extract) check_extract(samples, tax, tax_read);
  if (Populate_memory && Populate_memory_size == 0) cerr << "Loading database(s)... " << endl;
  vector<Mapped> kdbs(n_db), idxs(n_db);
  vector<DbFile> files(n_db);                                      // every database is checked before a device is touched
  for (size_t i = 0; i < n_db; i++) {
    cerr << " Database " << DB_filenames[i] << endl;
    kdbs[i].open(DB_filenames[i]);
    idxs[i].open(Index_filenames[i]);
    string err;
    if (parse_db(kdbs[i].p, kdbs[i].size, idxs[i].p, idxs[i].size, files[i], err)) die(EX_DATAERR, err);
  }
  for (size_t i = 1; i < n_db; i++) {                               // classify.cpp:203-210
    if (files[i].k != files[0].k) {
      fprintf(stderr, "Different k-mer sizes in databases 1 and %zu: %i vs %i!\n", i + 1, (int)files[0].k, (int)files[i].k);
      exit(1);
    }
  }
  if (!sheet && optind == argc) {                                  // `-M` without inputs: page-cache warm-up idiom
    if (Populate_memory && Populate_memory_size == 0) cerr << "\ncomplete." << endl;
    return 0;
  }
  if (TaxDB_file.empty()) { cerr << "TaxDB argument is required!" << endl; return 1; }

  // -x: the reference cuts the database into chunks of that many bytes (prepare_chunking).  HBM, not host RAM, is
  // what limits us: the database is split only when it does not fit the HBM budget (or KUQ_FORCE_CHUNKS=1 asks for
  // the reference's exact chunk size); either way -x selects the chunked HLL rule.
  uint64_t hbm_budget = 60ull << 30;          // of an 80 GB H100: room left for the sparse tier and the batch slots
  if (getenv("KUQ_HBM_BUDGET")) hbm_budget = strtoull(getenv("KUQ_HBM_BUDGET"), NULL, 10);
  uint64_t chunk_budget = 0;
  // The databases (one, or several together) larger than one card: sharded over the visible GPUs when they hold them
  // together (stage_shards, shard_loop), else streamed through the GPUs in ranges of at most 40 GB (two range
  // buffers + a round of reads have to fit, classify_streamed).  Several databases that fit the budget together are
  // resident.
  bool want_shards = false;
  uint64_t all_hbm = 0;
  for (size_t i = 0; i < n_db; i++) all_hbm += hbm_bytes(files[i], idxs[i]);
  if (all_hbm > hbm_budget || getenv("KUQ_FORCE_SHARDS")) {
    int n_vis = 0;
    if (const char *dl = getenv("KUQ_DEVICES")) { if (strcmp(dl, "all") == 0) n_vis = kuq_device_count(); else { n_vis = 1; for (const char *c = dl; *c; c++) n_vis += *c == ','; } }
    else if (!getenv("KUQ_DEVICE")) n_vis = kuq_device_count();
    want_shards = n_vis > 1 && (getenv("KUQ_FORCE_SHARDS") || all_hbm / n_vis + (16ull << 30) < hbm_budget);
  }
  if (all_hbm > hbm_budget && !want_shards) chunk_budget = std::min<uint64_t>(hbm_budget / 4, 40ull << 30);
  if (Populate_memory_size > 0 && getenv("KUQ_FORCE_CHUNKS")) { chunk_budget = Populate_memory_size; want_shards = false; }
  kuq_config cfg;
  kuq_config_default(&cfg);
  cfg.n_slots = 3;                             // classify b + 1 on the GPU, format b, gather b + 2 (process_file_parallel)
  // shards use slot 0; streamed runs (shards that fall back to streaming too) use slots 0 and 1
  if (want_shards || chunk_budget) cfg.n_slots = 2;
  cfg.max_bases_per_batch = 288ull << 20;      // one read may be a whole chromosome (the largest human one is 248 Mbp)
  cfg.work_unit_size = Work_unit_size;
  // -x (or a database that has to be split) → one global sketch per taxon (classify.cpp:719); else per work unit, which
  // is also the reference's rule for several databases (resident, streamed or sharded)
  cfg.hll_mode = (Populate_memory_size > 0 || ((chunk_budget || want_shards) && n_db == 1)) ? KUQ_HLL_CHUNKED : KUQ_HLL_PRELOAD;
#ifdef EXACT_COUNTING
  // classifyExact (classify.cpp:46-49): sets of k-mers instead of sketches.  Work units, chunks and devices make no
  // difference to a union of sets, so replicas and shards run as for classify and kuq_merge_into unites the sets.
  cfg.hll_mode = KUQ_HLL_EXACT;
  if (Quick_mode) die(EX_USAGE, "-q is not supported by the GPU classifyExact");
#endif
  if ((chunk_budget || want_shards) && !Populate_memory_size && n_db == 1)
    cerr << "classify: database larger than one GPU's HBM budget: " << (want_shards ? "sharding it over the GPUs" : "processing it in ranges")
         << (cfg.hll_mode == KUQ_HLL_EXACT ? "" : " (unique k-mer counts follow the -x rule)") << endl;
  if (getenv("KUQ_SPARSE_SLOTS")) cfg.sparse_set_slots = strtoull(getenv("KUQ_SPARSE_SLOTS"), NULL, 10);
  if (getenv("KUQ_DEVICE")) cfg.device = atoi(getenv("KUQ_DEVICE"));
  // devices: KUQ_DEVICES=0,2,3 (or "all"); default = every visible sm_90 GPU, whether the databases are replicated (they
  // fit a card), sharded (they fit the cards together) or streamed in ranges (each GPU streams its share of the ranges);
  // KUQ_DEVICE=n: that one device.
  vector<int> devices;
  {
    const char *dl = getenv("KUQ_DEVICES");
    if (dl && strcmp(dl, "all") != 0) {
      for (const char *q = dl; *q;) { devices.push_back(atoi(q)); while (*q && *q != ',') q++; if (*q) q++; }
    } else if (dl || !getenv("KUQ_DEVICE")) {
      for (int d = 0; d < kuq_device_count(); d++) devices.push_back(d);
    }
    if (devices.empty()) devices.assign(1, cfg.device);
    cfg.device = devices[0];
  }
  kuq_ctx *ctx = NULL;
  int rc = kuq_create(&cfg, &ctx);
  if (rc) die(EX_UNAVAILABLE, string("libkuq: ") + kuq_strerror(rc));
  All_ctx.assign(1, ctx);
  vector<int> ctx_devices(1, cfg.device);
  for (size_t g = 1; g < devices.size(); g++) {
    kuq_config c2 = cfg;
    c2.device = devices[g];
    kuq_ctx *cx = NULL;
    int r2 = kuq_create(&c2, &cx);
    if (r2) { fprintf(stderr, "classify: device %d not usable (%s): continuing without it\n", devices[g], kuq_strerror(r2)); continue; }
    All_ctx.push_back(cx);
    ctx_devices.push_back(devices[g]);
  }
  // shards on fewer than two contexts: streamed instead, over the contexts there are
  if (want_shards && All_ctx.size() < 2) { want_shards = false; chunk_budget = std::min<uint64_t>(hbm_budget / 4, 40ull << 30); }
  if (All_ctx.size() > 1 && !want_shards && !chunk_budget && n_db == 1)
    fprintf(stderr, "classify: %zu GPUs, database replicated, batches round-robin\n", All_ctx.size());
  if (n_db > 1 && !chunk_budget && !want_shards) fprintf(stderr, "classify: %zu databases resident on %zu GPU(s)\n", n_db, All_ctx.size());
  // -q: the preloaded path leaves a read at its -m'th hit; with -x every k-mer is counted (classify.cpp:943-944 / :701-738)
  for (kuq_ctx *c : All_ctx)
    if (Quick_mode && kuq_set_quick_mode(c, Minimum_hit_count, Populate_memory_size == 0)) die(EX_SOFTWARE, kuq_last_error(c));
  // records per taxid of each database (the .counts files)
  vector<map<uint32_t, uint64_t>> db_counts(n_db);
  if (!chunk_budget && !want_shards) {
    double T0__ = now_s();
    // the pinned staging sets of the ingest pipeline are allocated while the database travels to the GPUs
    std::thread prealloc([] {
      const size_t want = 3 * All_ctx.size();
      vector<Stage> tmp(want);
      for (auto &s : tmp) prepare_stage(s, 150ull << 20, 1u << 20);
      Prealloc_stages.swap(tmp);
    });
    // every device stages every database whole, in command-line order, from the same mapped files
    vector<Slice> whole;
    for (size_t d = 0; d < n_db; d++) whole.push_back(Slice{d, 0, 0});
    stage_slices(All_ctx, kdbs, idxs, vector<vector<Slice>>(All_ctx.size(), whole), true, true, db_counts);
    prealloc.join();
    TICK("stage_db");
  }
  if (Populate_memory && Populate_memory_size == 0) cerr << "\ncomplete." << endl;

  cerr << "Reading taxonomy index from " << TaxDB_file;
  if (!tax_read) tax.read(TaxDB_file);
  cerr << ". Done.\n";
  {
    vector<uint32_t> ids, parents;
    tax.parent_map(ids, parents);
    for (kuq_ctx *c : All_ctx)
      if (kuq_set_taxonomy(c, ids.data(), parents.data(), (uint32_t)ids.size())) die(EX_SOFTWARE, kuq_last_error(c));
    for (kuq_ctx *c : All_ctx)
      if (Filter && kuq_set_threshold(c, Threshold, tax.row_ids.data(), tax.row_parents.data(), (uint32_t)tax.row_ids.size()))
        die(EX_DATAERR, kuq_last_error(c));
    for (kuq_ctx *c : All_ctx)
      if (Extract && kuq_set_extract(c, Extract_taxa.data(), (uint32_t)Extract_taxa.size(), extract_flags(), tax.row_ids.data(),
                                     tax.row_parents.data(), (uint32_t)tax.row_ids.size()))
        die(EX_DATAERR, kuq_last_error(c));
  }
  // staging of the layouts that stage in pieces (the resident layouts staged above)
  Streamed streamed;
  uint32_t shard_runs = 0;
  int g0 = 0;                                                       // the first context that staged a slice
  if (want_shards) shard_runs = stage_shards(All_ctx, kdbs, idxs, files, db_counts);
  else if (chunk_budget) g0 = stage_streamed(streamed, All_ctx, ctx_devices, kdbs, idxs, files, chunk_budget, hbm_budget, db_counts);
  // the per-work-unit rule (resident without -x, and several databases in every layout); kuq_unit_table_rows finalizes
  // the context, so it comes after the taxonomy and the taxid universe
  if (want_shards || chunk_budget ? n_db > 1 : cfg.hll_mode == KUQ_HLL_PRELOAD) {
    uint32_t rows = 0;
    if (kuq_unit_table_rows(All_ctx[g0], &rows)) die(EX_SOFTWARE, kuq_last_error(All_ctx[g0]));
    if (rows) Max_units_per_batch = rows;
  }
#ifdef EXACT_COUNTING
  // classifyExact on several contexts: the counters join the first context, and the exact k-mer sets are spread over
  // all contexts by k-mer instead of united on one card, so no card has to hold the union.  The report's clades come
  // from the roll-up books summed over the parts.  A taxonomy with entries below taxon 0 keeps the union on the first
  // context: print_report counts those clades one by one, which needs every pair in one place.
  {
    auto z = tax.idx.find(0);
    Exact_union_needed = z != tax.idx.end() && !tax.e[z->second].children.empty();
    Exact_partitioned = All_ctx.size() > 1 && !Exact_union_needed;
  }
  // KUQ_EXACT_HOST_BUDGET=<bytes>: a set that outgrows the devices spills to host memory by k-mer part, up to that many
  // bytes of pairs over all contexts, and is counted part by part at the end of each sample (end_sample)
  // A taxonomy with entries below taxon 0 counts those clades one by one from the whole set on one GPU, which a spilled
  // set does not have: spilling stays off there, so a set that outgrows the card stops at its first failed growth.
  if (const char *e = getenv("KUQ_EXACT_HOST_BUDGET")) {
    const uint64_t budget = strtoull(e, NULL, 10);
    if (Exact_union_needed && budget)
      fprintf(stderr, "classifyExact: KUQ_EXACT_HOST_BUDGET is not used: this taxonomy has entries below taxon 0, whose clades "
                      "need the whole exact k-mer set on one GPU\n");
    for (kuq_ctx *c : All_ctx)
      if (!Exact_union_needed && kuq_set_exact_spill(c, budget)) die(EX_SOFTWARE, kuq_last_error(c));
  }
#endif
  Run.samples = samples;
  Run.sheet = sheet;
  Run.tax = &tax;
  Run.db_counts = db_counts;
  // the streamed layout shares its passes over the database(s) among the samples: it runs every sample's lifecycle
  if (chunk_budget) classify_streamed(streamed);
  for (size_t si = 0; si < Run.samples.size() && !chunk_budget; si++) {
    begin_sample(si);
    const vector<pair<const char *, const char *>> files = files_of(Run.samples[si]);
    if (want_shards) shard_loop(All_ctx, shard_runs, n_db > 1, files);
    else for (auto &in : files) process_file(ctx, in.first, in.second);
    end_sample(si);
  }
  Sample_label.clear();
  if (Mpa) {                                                        // one table for every sample of the run
    OutStream mo;
    mo.open(Mpa_output_file);
    mo.write(Script_tax.mpa_table(Mpa_counts, Mpa_ids, Mpa_show_zeros, Mpa_header_line, Mpa_intermediate));
    mo.close();
  }
  for (const void *p : streamed.pinned) kuq_host_unregister((void *)p);
  for (kuq_ctx *c : All_ctx) kuq_destroy(c);
  return Run.status;
}
