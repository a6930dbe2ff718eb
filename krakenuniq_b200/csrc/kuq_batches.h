// Where classify's batches close and which work unit each read belongs to, for every ingest path and for the library's
// own unit ids (kuq_submit_batch without ids).  The batch boundaries are part of the output: the per-work-unit HLL rule
// is exact only when batches hold whole units (DESIGN.md §4).
//
// The rule, over the reads of one input file in order (process_file, src/classify.cpp:506-524):
//   - A read joins the open work unit; the unit closes once its bases reach the unit size (-u).
//   - Unit-aligned: the batch closes after a read that closes a unit once it holds batch_nt bases, batch_reads reads or
//     max_units units.  Inside one unit it closes after 150 MiB or 2^20 - 1 reads (a unit larger than a slot, huge -u:
//     it is then counted as two).
//   - Not aligned (the -x path, which reads sequence by sequence without work units, :566-791): the batch closes after
//     batch_nt bases or 2^20 - 1 reads.
//   - With a slot (slot_nt > 0), a read that would take the batch past slot_nt bases closes it before itself and starts
//     the next one.
//   - At the end of the input, aligned: a last work unit of total length 0 is dropped (:523-524).
//   - Work units do not span input files: a file that kept reads ends its last unit, and the next file starts a new one
//     (kuq_finish does the same for the library's unit ids).
#ifndef KUQ_BATCHES_H
#define KUQ_BATCHES_H
#include <stddef.h>
#include <stdint.h>

// The open work unit: reads join it until its bases reach the unit size (classify.cpp:514-520).  Units do not span
// input files: new_file() starts the next one.
struct WorkUnits {
  uint64_t nt = 0;      // bases of the open unit
  uint32_t id = 0;      // id of the open unit
  // a read of len bases joins the open unit; true when it closes it
  bool add(uint64_t len, uint64_t unit_size) {
    nt += len;
    if (nt < unit_size) return false;
    nt = 0;
    id++;
    return true;
  }
  void new_file() { nt = 0; id++; }
};

struct BatchLimits {
  uint64_t batch_nt = 96ull << 20;
  size_t batch_reads = (1u << 20) - 4096;
  size_t max_units = SIZE_MAX;
  uint64_t slot_nt = 0;                  // 0: no slot
  uint64_t unit_size = 500000;
  bool aligned = true;
};

struct BatchCutter {
  static constexpr uint64_t UNIT_SPLIT_NT = 150ull << 20;
  static constexpr size_t SPLIT_READS = (1u << 20) - 1;
  BatchLimits lim;
  WorkUnits units;
  uint64_t nt = 0;                       // bases of the open batch
  size_t reads = 0, closed_units = 0;    // reads and closed units of the open batch
  size_t tail = 0;                       // reads of the open batch after its last closed unit
  size_t file_reads = 0;                 // reads of the open input file
  explicit BatchCutter(const BatchLimits &l) : lim(l) {}

  struct Step {
    bool before, after;                  // the batch closes before / after this read
    uint32_t unit;                       // the read's work unit
  };
  Step next(uint64_t len) {
    Step s{false, false, units.id};
    if (lim.slot_nt && reads && nt + len > lim.slot_nt) { s.before = true; start(); }
    nt += len;
    reads++;
    tail++;
    file_reads++;
    const bool closed = units.add(len, lim.unit_size);
    if (!lim.aligned) {
      s.after = nt >= lim.batch_nt || reads >= SPLIT_READS;
    } else if (closed) {
      tail = 0;
      closed_units++;
      s.after = nt >= lim.batch_nt || reads >= lim.batch_reads || closed_units >= lim.max_units;
    } else {
      s.after = reads >= SPLIT_READS || nt >= UNIT_SPLIT_NT;
    }
    if (s.after) start();
    return s;
  }
  // at the end of the input: how many reads at the end of the open batch are dropped
  size_t drop() const { return lim.aligned && units.nt == 0 ? tail : 0; }
  // after drop(): the next input file starts a new batch, and a new unit when this file kept reads
  void next_file() {
    if (file_reads > drop()) units.new_file();
    units.nt = 0;
    file_reads = 0;
    start();
  }

 private:
  void start() { nt = 0; reads = closed_units = tail = 0; }
};

#endif
