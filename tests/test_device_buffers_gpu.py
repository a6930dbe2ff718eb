"""Every CUDA resource libkuq takes is given back: device memory, pinned memory, streams and events.

A small interposer (compiled here, loaded with LD_PRELOAD into the subprocesses only) records each handle that
cudaMalloc, cudaMallocHost, cudaHostAlloc, cudaStreamCreate* and cudaEventCreate* return against its destroy call, and
at exit writes the handles still live and every free of a handle it never handed out.  libkuq.so links the CUDA runtime
shared, so its calls bind to the interposer's definitions.  Each layout of classify / classifyExact, db_sort and
set_lcas, and a ctypes script over the C ABI must end with neither: a leaked temporary, a leaked or doubly freed owner
shows up in one of the two lists.  The only handles allowed to outlive a run are the pinned batch stages that the
classify executable takes through kuq_host_alloc and keeps for the life of the process."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from krakenuniq_b200 import build
from tests import util
from tests.test_db_build_ranges_gpu import _budgets, _golden_style, _jdb, _lca_budget

pytestmark = pytest.mark.gpu
G = util.GOLDEN
M = os.path.join(util.ROOT, "tests", "golden", "multidb")

LEDGER_C = r"""
#define _GNU_SOURCE
#include <dlfcn.h>
#include <pthread.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/syscall.h>
#include <unistd.h>

enum { MEM, PINNED, STREAM, EVENT };
static const char *KIND[] = {"device", "pinned", "stream", "event"};
typedef struct { void *h; int kind; size_t bytes; char who[48]; } Entry;
static Entry *live;
static size_t n_live, cap_live, unknown_frees;
static char unknown[4096];
static FILE *trace;
static pthread_mutex_t mu = PTHREAD_MUTEX_INITIALIZER;

static void *real(const char *name) {
  void *f = dlsym(RTLD_NEXT, name);
  if (!f) {   /* libkuq was dlopen'ed locally (ctypes): look in the runtime it loaded */
    void *rt = dlopen("libcudart.so.12", RTLD_NOW | RTLD_NOLOAD);
    if (rt) f = dlsym(rt, name);
  }
  if (!f) { fprintf(stderr, "ledger: no %s\n", name); abort(); }
  return f;
}
static void note(const char *call, size_t bytes) {
  if (trace) fprintf(trace, "%ld %s %zu\n", (long)syscall(SYS_gettid), call, bytes);
}
static void add(void *h, int kind, size_t bytes, const char *call, void *ret) {
  if (!h) return;
  pthread_mutex_lock(&mu);
  note(call, bytes);
  if (n_live == cap_live) { cap_live = cap_live ? 2 * cap_live : 1024; live = realloc(live, cap_live * sizeof *live); }
  Entry *e = &live[n_live++];
  e->h = h; e->kind = kind; e->bytes = bytes;
  Dl_info di;
  snprintf(e->who, sizeof e->who, "%s", dladdr(ret, &di) && di.dli_sname ? di.dli_sname : "?");
  pthread_mutex_unlock(&mu);
}
static void drop(void *h, int kind, const char *call) {
  if (!h) return;
  pthread_mutex_lock(&mu);
  size_t i = 0;
  while (i < n_live && !(live[i].h == h && live[i].kind == kind)) i++;
  if (i == n_live) {
    unknown_frees++;
    size_t at = strlen(unknown);
    if (at + 64 < sizeof unknown) snprintf(unknown + at, sizeof unknown - at, "%s%s %p", at ? ", " : "", call, h);
    note(call, 0);
  } else {
    note(call, live[i].bytes);
    live[i] = live[--n_live];
  }
  pthread_mutex_unlock(&mu);
}

#define RET __builtin_return_address(0)
int cudaMalloc(void **p, size_t n) {
  int e = ((int (*)(void **, size_t))real("cudaMalloc"))(p, n);
  if (!e) add(*p, MEM, n, "cudaMalloc", RET);
  return e;
}
int cudaMallocHost(void **p, size_t n) {
  int e = ((int (*)(void **, size_t))real("cudaMallocHost"))(p, n);
  if (!e) add(*p, PINNED, n, "cudaMallocHost", RET);
  return e;
}
int cudaHostAlloc(void **p, size_t n, unsigned flags) {
  int e = ((int (*)(void **, size_t, unsigned))real("cudaHostAlloc"))(p, n, flags);
  if (!e) add(*p, PINNED, n, "cudaHostAlloc", RET);
  return e;
}
int cudaFree(void *p) { drop(p, MEM, "cudaFree"); return ((int (*)(void *))real("cudaFree"))(p); }
int cudaFreeHost(void *p) { drop(p, PINNED, "cudaFreeHost"); return ((int (*)(void *))real("cudaFreeHost"))(p); }
int cudaStreamCreate(void **s) {
  int e = ((int (*)(void **))real("cudaStreamCreate"))(s);
  if (!e) add(*s, STREAM, 0, "cudaStreamCreate", RET);
  return e;
}
int cudaStreamCreateWithFlags(void **s, unsigned f) {
  int e = ((int (*)(void **, unsigned))real("cudaStreamCreateWithFlags"))(s, f);
  if (!e) add(*s, STREAM, 0, "cudaStreamCreate", RET);
  return e;
}
int cudaStreamCreateWithPriority(void **s, unsigned f, int prio) {
  int e = ((int (*)(void **, unsigned, int))real("cudaStreamCreateWithPriority"))(s, f, prio);
  if (!e) add(*s, STREAM, 0, "cudaStreamCreate", RET);
  return e;
}
int cudaStreamDestroy(void *s) { drop(s, STREAM, "cudaStreamDestroy"); return ((int (*)(void *))real("cudaStreamDestroy"))(s); }
int cudaEventCreate(void **ev) {
  int e = ((int (*)(void **))real("cudaEventCreate"))(ev);
  if (!e) add(*ev, EVENT, 0, "cudaEventCreate", RET);
  return e;
}
int cudaEventCreateWithFlags(void **ev, unsigned f) {
  int e = ((int (*)(void **, unsigned))real("cudaEventCreateWithFlags"))(ev, f);
  if (!e) add(*ev, EVENT, 0, "cudaEventCreate", RET);
  return e;
}
int cudaEventDestroy(void *ev) { drop(ev, EVENT, "cudaEventDestroy"); return ((int (*)(void *))real("cudaEventDestroy"))(ev); }

__attribute__((constructor)) static void start(void) {
  const char *t = getenv("LEDGER_TRACE");
  if (t && *t) trace = fopen(t, "w");
}
__attribute__((destructor)) static void finish(void) {
  const char *path = getenv("LEDGER_OUT");
  FILE *f = path ? fopen(path, "w") : NULL;
  if (!f) return;
  pthread_mutex_lock(&mu);
  fprintf(f, "{\"unknown_frees\": %zu, \"unknown\": \"%s\", \"live\": [", unknown_frees, unknown);
  for (size_t i = 0; i < n_live; i++)
    fprintf(f, "%s{\"kind\": \"%s\", \"bytes\": %zu, \"by\": \"%s\"}", i ? ", " : "", KIND[live[i].kind], live[i].bytes, live[i].who);
  fprintf(f, "]}\n");
  fclose(f);
  if (trace) fclose(trace);
  pthread_mutex_unlock(&mu);
}
"""

# The C ABI paths the executables do not take: kuq_merge_into of sparse and exact sets (in rounds), the clade roll-up
# over sparse and dense clades, the exact roll-up in passes, the *_alloc exports freed by the caller, and
# kuq_stream_open twice.  No torch: its own CUDA allocations would pass through the interposer too.
SCRIPT = r"""
import sys
sys.path.insert(0, sys.argv[1])
import numpy as np
from krakenuniq_b200 import binding, synth

rng = np.random.default_rng(5)
tax = synth.make_taxonomy(6, 3, 2)
genomes = synth.random_genomes(rng, 6, 3000)
km, tx = synth.label_kmers(genomes, synth.species_ids(tax), tax, 31)
kdb, idx = synth.build_db_images(km, tx, 31, 8, 2)
bases, offs = synth.sample_reads(rng, genomes, 1024, 150, 0.01, 0.2, 0.2)
ids, parents = tax.parent_map()
half = len(offs) // 2


def ctx(mode):
    c = binding.Classifier(device=0, max_reads=1 << 12, max_bases=1 << 20, hll_mode=mode, sparse_set_slots=1024)
    c.stage_db(kdb, idx)
    c.set_taxonomy(ids, parents)
    return c


for mode in (binding.HLL_PRELOAD, binding.HLL_DENSE_ONLY, binding.HLL_EXACT):
    a, b = ctx(mode), ctx(mode)
    a.classify(bases, offs[:half + 1])
    b.classify(bases, offs[half:])
    a.finish()
    b.finish()
    a.merge_from(b)
    r, k, u = a.clade_counts_tree(ids)
    assert r.sum() > 0 and u.max() > 0
    if mode != binding.HLL_DENSE_ONLY:
        export = a.exact_export_partitioned_alloc if mode == binding.HLL_EXACT else a.sparse_export_partitioned_alloc
        p, counts = export(2)
        assert counts.sum() > 0
        a.device_free(p)
    a.close()
    b.close()

s = binding.Classifier(device=0, max_reads=1 << 12, max_bases=1 << 20, sparse_set_slots=1024)
s.set_db_taxid_universe(np.unique(tx))
s.set_taxonomy(ids, parents)
for _ in range(2):
    s.stream_open(31, 8, 2, len(km), 1 << 16)
s.close()
print("script ok")
"""


@pytest.fixture(scope="module")
def ledger(tmp_path_factory):
    d = tmp_path_factory.mktemp("ledger")
    (d / "ledger.c").write_text(LEDGER_C)
    so = d / "libledger.so"
    subprocess.run(["gcc", "-shared", "-fPIC", "-O1", "-o", str(so), str(d / "ledger.c"), "-ldl", "-lpthread"], check=True)
    return str(so)


def _run(ledger, tmp_path, cmd, env=None, cwd=None, tag="run"):
    out = tmp_path / f"{tag}.ledger.json"
    full_env = dict(os.environ, **(env or {}), LD_PRELOAD=ledger, LEDGER_OUT=str(out))
    r = subprocess.run(cmd, capture_output=True, text=True, env=full_env, cwd=cwd or tmp_path)
    assert r.returncode == 0, r.stderr[-3000:]
    book = json.loads(out.read_text())
    leaked = [h for h in book["live"] if h["by"] != "kuq_host_alloc"]
    assert not leaked and not book["unknown_frees"], (tag, leaked[:20], book["unknown"])
    return r


def _classify(tool="classify"):
    return os.path.join(os.path.dirname(build.build_classify()), tool)


def _db(path=G, name="database"):
    return ["-d", os.path.join(path, f"{name}.kdb"), "-i", os.path.join(path, f"{name}.idx")]


SMALL = {"KUQ_SPARSE_SLOTS": "4096", "KUQ_BATCH_READS": "200"}


@pytest.mark.parametrize("tag,tool,dbs,extra,env", [
    ("resident", "classify", [("", "database")], ["-M"], {}),
    ("replicas", "classify", [("", "database")], ["-M"], {"KUQ_DEVICES": "0,0"}),
    ("chunked", "classify", [("", "database")], ["-x", "40K"], {"KUQ_FORCE_CHUNKS": "1"}),
    ("two_databases", "classify", [("", "database"), (M, "db2")], ["-M", "-u", "20000"], {}),
    ("shards", "classify", [("", "database")], ["-M"], {"KUQ_DEVICES": "0,0", "KUQ_FORCE_SHARDS": "1"}),
    ("exact_partition", "classifyExact", [("", "database")], ["-M"], {"KUQ_DEVICES": "0,0", "KUQ_SPARSE_SLOTS": "1024"}),
])
def test_classify_layouts_release_everything(ledger, tmp_path, tag, tool, dbs, extra, env):
    cmd = [_classify(tool)] + sum((_db(p or G, n) for p, n in dbs), []) + ["-a", os.path.join(G, "taxDB"), "-t", "1"] + extra + \
        ["-r", str(tmp_path / "o.report"), "-o", str(tmp_path / "o.kraken"), os.path.join(G, "reads.fa")]
    r = _run(ledger, tmp_path, cmd, dict(SMALL, **env), tag=tag)
    assert "not usable" not in r.stderr


def test_threshold_extract_sample_sheet_releases_everything(ledger, tmp_path):
    sheet = tmp_path / "s.tsv"
    sheet.write_text("name\tinput\toutput\treport\textract_out\n"
                     f"a\t{os.path.join(G, 'reads.fa')}\ta.kraken\ta.report\ta.x\n"
                     f"b\t{os.path.join(G, 'reads_300.fq')}\tb.kraken\tb.report\tb.x\n")
    cmd = [_classify()] + _db() + ["-a", os.path.join(G, "taxDB"), "-M", "--threshold", "0.5", "--extract", "0",
                                   "--extract-invert", "--sample-sheet", str(sheet)]
    _run(ledger, tmp_path, cmd, SMALL)
    assert (tmp_path / "a.x").stat().st_size > 0 and (tmp_path / "b.x").stat().st_size > 0


def test_db_sort_and_set_lcas_release_everything(ledger, tmp_path):
    db_sort, set_lcas = build.build_dbtools()
    _jdb(31, 200000, 4).tofile(tmp_path / "database.jdb")
    sort = [db_sort, "-z", "-n", "8", "-d", "database.jdb", "-o", "database0.kdb", "-i", "database.idx"]
    _run(ledger, tmp_path, sort, tag="db_sort")
    budget = _budgets(np.fromfile(tmp_path / "database.idx", np.uint8), 12)["several"]
    r = _run(ledger, tmp_path, sort, {"KUQ_DB_SORT_BUDGET": str(budget)}, tag="db_sort_passes")
    assert "db_sort: 1 pass" not in r.stderr
    d = tmp_path / "lib"
    d.mkdir()
    _golden_style(d)
    lcas = [set_lcas, "-x", "-d", "database0.kdb", "-i", "database.idx", "-b", "taxDB", "-m", "seqid2taxid.map", "-c",
            "database.kdb.counts", "-F", "lib.fa"]
    budget = _lca_budget(d)
    _run(ledger, tmp_path, lcas, cwd=d, tag="set_lcas")
    r = _run(ledger, tmp_path, lcas, {"KUQ_SET_LCAS_BUDGET": str(budget)}, cwd=d, tag="set_lcas_ranges")
    assert "minimizer ranges" in r.stderr


def test_c_abi_releases_everything(ledger, tmp_path):
    """merges, clade roll-ups, caller-freed exports and a re-opened stream, without torch in the process"""
    script = tmp_path / "abi.py"
    script.write_text(SCRIPT)
    env = {"KUQ_EXACT_MERGE_SLOTS": "256", "KUQ_EXACT_ROLLUP_BUDGET": "20000"}
    r = _run(ledger, tmp_path, [sys.executable, "-s", str(script), util.ROOT], env)
    assert "script ok" in r.stdout
