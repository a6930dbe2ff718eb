"""kuq_batches.h (where classify's batches close, which work unit each read belongs to) compiled for the host and held
against the loops it replaced, restated here from the commit before it: process_file_parallel's cut, the serial
process_file, BatchReader::next, the unit ids of run_streamed / shard_loop, and the library's cut_units + kuq_finish.
Only read lengths are fed, so reads of hundreds of MiB cost nothing."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

MiB = 1 << 20
BATCH_NT = 96 * MiB
SLOT_NT = 280 * MiB
HDR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "krakenuniq_b200", "csrc", "kuq_batches.h")

SHIM = r'''
#include "%s"
extern "C" void cut(const uint64_t *len, const int32_t *file, size_t n, const uint64_t *lim, uint8_t *flags,
                    uint32_t *unit, uint64_t *drop) {
  BatchLimits l;
  l.batch_nt = lim[0]; l.batch_reads = lim[1]; l.max_units = lim[2]; l.slot_nt = lim[3]; l.unit_size = lim[4];
  l.aligned = lim[5] != 0;
  BatchCutter c(l);
  for (size_t i = 0; i < n; i++) {
    if (i && file[i] != file[i - 1]) { drop[file[i - 1]] = c.drop(); c.next_file(); }
    const BatchCutter::Step s = c.next(len[i]);
    flags[i] = (uint8_t)(s.before | s.after << 1);
    unit[i] = s.unit;
  }
  if (n) drop[file[n - 1]] = c.drop();
}
extern "C" void lib_units(const uint64_t *len, const int32_t *file, size_t n, uint64_t unit_size, uint32_t *unit) {
  WorkUnits u;
  for (size_t i = 0; i < n; i++) {
    if (i && file[i] != file[i - 1]) u.new_file();
    unit[i] = u.id;
    u.add(len[i], unit_size);
  }
}
'''


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    d = tmp_path_factory.mktemp("batches")
    (d / "b.cpp").write_text(SHIM % HDR)
    subprocess.run(["/usr/bin/g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-x", "c++", str(d / "b.cpp"), "-o", str(d / "b.so")],
                   check=True)
    return ctypes.CDLL(str(d / "b.so"))


def run_cutter(lib, files, batch_nt=BATCH_NT, batch_reads=MiB - 4096, max_units=2**64 - 1, slot_nt=0, unit_size=500000,
               aligned=True):
    """files: one list of read lengths per input file.  Returns (batches, units): batches as (file, begin, end) over the
    reads of all files, the dropped tails left out; units: the work unit of every kept read."""
    lens = np.array([x for f in files for x in f], np.uint64)
    file = np.array([k for k, f in enumerate(files) for _ in f], np.int32)
    n = len(lens)
    lim = np.array([batch_nt, batch_reads, max_units, slot_nt, unit_size, int(aligned)], np.uint64)
    flags = np.zeros(n, np.uint8)
    unit = np.zeros(n, np.uint32)
    drop = np.zeros(max(1, len(files)), np.uint64)
    p = ctypes.c_void_p
    lib.cut(p(lens.ctypes.data), p(file.ctypes.data), ctypes.c_size_t(n), p(lim.ctypes.data), p(flags.ctypes.data),
            p(unit.ctypes.data), p(drop.ctypes.data))
    batches, begin, i = [], 0, 0
    for k, f in enumerate(files):
        end = i + len(f)
        for i in range(i, end):
            if flags[i] & 1:
                batches.append((k, begin, i))
                begin = i
            if flags[i] & 2:
                batches.append((k, begin, i + 1))
                begin = i + 1
        i = end
        assert int(drop[k]) <= end - begin                  # only reads of the open batch are dropped
        if end - int(drop[k]) > begin:
            batches.append((k, begin, end - int(drop[k])))
        begin = end
    units = [int(unit[j]) for _, a, b in batches for j in range(a, b)]
    return batches, units


# ---- the loops of the commit before kuq_batches.h (classify_main.cpp / kuq_api.cu there) ---------------------------

def parent_parallel(lens, wus, batch_reads=None, max_units=float("inf")):
    """process_file_parallel's Cut loop, classify_main.cpp:1145-1176"""
    br = max(1, batch_reads) if batch_reads is not None else MiB - 4096
    batches, unit_nt, batch_nt, begin, unit_first, batch_units = [], 0, 0, 0, 0, 0
    for i, ln in enumerate(lens):
        if batch_nt + ln > SLOT_NT and i > begin:
            batches.append((begin, i))
            begin, batch_nt, batch_units = i, 0, 0
        unit_nt += ln
        batch_nt += ln
        close_unit = unit_nt >= wus
        if close_unit:
            unit_nt, unit_first, batch_units = 0, i + 1, batch_units + 1
        if ((close_unit and (batch_nt >= BATCH_NT or i + 1 - begin >= min(br, MiB - 4096) or batch_units >= max_units)) or
                (not close_unit and (i + 1 - begin >= MiB - 1 or batch_nt >= 150 * MiB))):
            batches.append((begin, i + 1))
            begin, batch_nt, batch_units = i + 1, 0, 0
            if not close_unit:
                unit_first = i + 1
    end = len(lens)
    if unit_nt == 0 and unit_first < len(lens):
        end = unit_first
    if end > begin:
        batches.append((begin, end))
    return batches


def parent_serial(lens, wus, max_units=float("inf")):
    """process_file's serial loop, classify_main.cpp:1347-1431"""
    batches, begin, nt, unit_nt, unit_first, batch_units = [], 0, 0, 0, 0, 0
    for i, ln in enumerate(lens):
        if nt + ln > SLOT_NT and i > begin:         # moved to the next batch, without the close test
            batches.append((begin, i))
            begin, nt, unit_first, batch_units = i, ln, 0, 0
            unit_nt += ln
            if unit_nt >= wus:
                unit_nt, unit_first, batch_units = 0, 1, batch_units + 1
            continue
        nt += ln
        unit_nt += ln
        reads = i + 1 - begin
        if unit_nt >= wus:
            unit_nt, unit_first = 0, reads
            batch_units += 1
            cut = nt >= BATCH_NT or reads >= MiB - 4096 or batch_units >= max_units
        else:
            cut = reads >= MiB - 1 or nt >= 150 * MiB
        if cut:
            batches.append((begin, i + 1))
            begin, nt, unit_first, batch_units = i + 1, 0, 0, 0
    end = len(lens)
    if unit_nt == 0 and unit_first < end - begin:
        end = begin + unit_first
    if end > begin:
        batches.append((begin, end))
    return batches


def parent_batch_reader(lens, wus, max_nt, aligned, max_units=float("inf")):
    """BatchReader::next over one file, classify_main.cpp:1445-1486"""
    batches, begin, nt, unit_nt, unit_first, batch_units = [], 0, 0, 0, 0, 0
    for i, ln in enumerate(lens):
        nt += ln
        reads = i + 1 - begin
        if not aligned:
            cut = nt >= max_nt or reads >= MiB - 1
        else:
            unit_nt += ln
            close_unit = unit_nt >= wus
            if close_unit:
                unit_nt, unit_first, batch_units = 0, reads, batch_units + 1
            cut = ((nt >= max_nt or reads >= MiB - 4096 or batch_units >= max_units) if close_unit else
                   (reads >= MiB - 1 or nt >= 150 * MiB))
        if cut:
            batches.append((begin, i + 1))
            begin, nt, unit_first, batch_units = i + 1, 0, 0, 0
    end = len(lens)
    if aligned and unit_nt == 0 and unit_first < end - begin:
        end = begin + unit_first
    if end > begin:
        batches.append((begin, end))
    return batches


def parent_unit_ids(batches, lens, wus):
    """run_streamed :1597-1647 and shard_loop :1760-1777: ids over the (file, begin, end) batches in order"""
    unit_next, unit_nt, unit_file, ids = 0, 0, -1, []
    for f, a, b in batches:
        if unit_file >= 0 and f != unit_file:
            unit_next, unit_nt = unit_next + 1, 0
        unit_file = f
        for i in range(a, b):
            ids.append(unit_next)
            unit_nt += lens[i]
            if unit_nt >= wus:
                unit_next, unit_nt = unit_next + 1, 0
    return ids


def parent_library_units(files, wus):
    """cut_units, kuq_api.cu:1172-1180, with kuq_finish (:2210-2216) after every file"""
    unit_next, unit_nt, ids = 0, 0, []
    for k, f in enumerate(files):
        if k:
            unit_next, unit_nt = unit_next + 1, 0
        for ln in f:
            ids.append(unit_next)
            unit_nt += ln
            if unit_nt >= wus:
                unit_next, unit_nt = unit_next + 1, 0
    return ids


def one_file(batches):
    return [(a, b) for _, a, b in batches]


def check_resident(lib, lens, wus, batch_reads=None, max_units=2**64 - 1, serial_too=True):
    """both ingest paths of the resident layout"""
    br = min(MiB - 4096, max(1, batch_reads)) if batch_reads is not None else MiB - 4096
    got, _ = run_cutter(lib, [lens], batch_reads=br, max_units=max_units, slot_nt=SLOT_NT, unit_size=wus)
    mu = max_units if max_units < 2**64 - 1 else float("inf")
    want = parent_parallel(lens, wus, batch_reads, mu)
    assert one_file(got) == want
    if serial_too:
        assert parent_serial(lens, wus, mu) == want
    return want


def check_reader(lib, files, wus, max_nt, aligned, max_units=2**64 - 1):
    """the streamed and sharded layouts: BatchReader per file, unit ids across the files"""
    got, units = run_cutter(lib, files, batch_nt=max_nt, max_units=max_units, unit_size=wus, aligned=aligned)
    mu = max_units if max_units < 2**64 - 1 else float("inf")
    want, at = [], 0
    for k, f in enumerate(files):
        want += [(k, at + a, at + b) for a, b in parent_batch_reader(f, wus, max_nt, aligned, mu)]
        at += len(f)
    assert got == want
    lens = [x for f in files for x in f]
    assert units == parent_unit_ids(want, lens, wus)
    return want


@pytest.mark.parametrize("aligned", [True, False])
@pytest.mark.parametrize("wus", [1, 100, 3000, 500000])
def test_random_lengths(lib, wus, aligned):
    rng = np.random.default_rng(wus)
    lens = rng.integers(0, 2001, 20000).tolist()
    for i in rng.integers(0, len(lens), 2000):
        lens[i] = 0
    lens += [0] * 7                                          # a tail of zero-length reads
    if aligned:
        for batch_reads, max_units in [(None, 2**64 - 1), (37, 2**64 - 1), (1, 2**64 - 1), (None, 5), (500, 3)]:
            check_resident(lib, lens, wus, batch_reads, max_units, serial_too=batch_reads is None)
    for max_nt, max_units in [(50000, 2**64 - 1), (7000, 4), (1, 2**64 - 1)]:
        check_reader(lib, [lens], wus, max_nt, aligned, max_units)


@pytest.mark.parametrize("wus", [1, 100, 500000])
def test_zero_length_reads(lib, wus):
    for lens in ([], [0], [0] * 50, [5, 0, 0], [0, 0, 7], [wus, 0, 0, 0], [wus - 1 if wus > 1 else 0, 0, 0]):
        check_resident(lib, lens, wus)
        for aligned in (True, False):
            check_reader(lib, [lens], wus, 96 * MiB, aligned)


def test_hundred_mib_read_closes_a_unit(lib):
    for lens in ([100 * MiB, 10, 20], [10, 100 * MiB, 0, 0], [50 * MiB, 100 * MiB, 30 * MiB, 0]):
        assert check_resident(lib, lens, 500000)[0][1] == lens.index(100 * MiB) + 1
        check_reader(lib, [lens], 500000, 96 * MiB, True)


@pytest.mark.parametrize("wus", [250 * MiB, 1 << 40])
def test_read_moved_past_the_slot(lib, wus):
    """100 MiB of an open unit, then a 200 MiB read that does not fit the slot next to it: the read starts the next
    batch and gets the close test there (with -u 250 MiB it closes a unit, with a huge -u it does not)"""
    lens = [100 * MiB, 200 * MiB, MiB, 0]
    want = check_resident(lib, lens, wus, serial_too=False)
    assert want[:2] == [(0, 1), (1, 2)]                     # the moved read is a batch of its own
    # the serial ingest of the commit before did not test the moved read: the next read joined its batch
    assert parent_serial(lens, wus)[1][1] > 2


def test_unit_longer_than_150_mib(lib):
    lens = [10 * MiB] * 40 + [0, 3]
    want = check_resident(lib, lens, 1 << 40)
    assert [b - a for a, b in want] == [15, 15, 12]
    check_reader(lib, [lens], 1 << 40, 96 * MiB, True)


def test_read_count_cut_inside_a_unit(lib):
    lens = [1] * (1 << 20)
    assert check_resident(lib, lens, 1 << 40) == [(0, MiB - 1), (MiB - 1, MiB)]
    check_reader(lib, [lens], 1 << 40, 96 * MiB, True)
    lens = [0] * ((1 << 20) + 5)                            # the cut keeps a unit of length 0, the tail after it goes
    assert check_resident(lib, lens, 100) == [(0, MiB - 1)]
    check_reader(lib, [lens], 100, 96 * MiB, True)


@pytest.mark.parametrize("wus", [1, 100, 3000])
def test_unit_ids_across_files(lib, wus):
    rng = np.random.default_rng(7)
    a = rng.integers(0, 300, 400).tolist()
    b = rng.integers(0, 300, 300).tolist() + [0, 0]
    files_list = [[a, b], [a + [0, 0], b], [a, [0, 0, 0], b], [[0, 0], a], [a, [], b], [[wus], [wus], [0]]]
    for files in files_list:
        for aligned in (True, False):
            check_reader(lib, files, wus, 5000, aligned, max_units=6)
        # the library's own unit ids: every file ends its last unit (kuq_finish)
        lens = np.array([x for f in files for x in f], np.uint64)
        file = np.array([k for k, f in enumerate(files) for _ in f], np.int32)
        unit = np.zeros(len(lens), np.uint32)
        p = ctypes.c_void_p
        lib.lib_units(p(lens.ctypes.data), p(file.ctypes.data), ctypes.c_size_t(len(lens)), ctypes.c_uint64(wus),
                      p(unit.ctypes.data))
        nonempty = [f for f in files if f]
        assert unit.tolist() == parent_library_units(nonempty, wus)
