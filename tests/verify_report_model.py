"""CPU restatement of --verifyreport: the damaged extents that a phase reports, from the expected
file content, the actual file bytes and the byte ranges the phase read.

Each read range (one block) gives one record per 512-byte file sector it touches: the differing
bytes of the sector inside the range and the first / last of them. A sector's count is kept per
part, a part being where the range starts in the sector (0 when it starts before it): records of
the same part (re-reads) count once with the largest count, parts of different ranges add up. An
extent is a maximal run of consecutive damaged sectors of one file; it spans its first to its last
differing byte. Lines are sorted by path, then offset."""
import collections

import numpy as np

from tests import verify_random_grain_model as vrg
from tests import verify_random_model as vrm

SECTOR = 512


def pattern_content(start, length, salt):
    """--verify: file byte x = byte (x % 8) of the little-endian u64 ((x & ~7) + salt)"""
    first = start & ~7
    words = (np.arange(first, start + length + 8, 8, dtype=np.uint64) + np.uint64(salt))
    raw = words.astype("<u8").tobytes()
    return raw[start - first:start - first + length]


def block_random_content(size, block, pct, seed, file_key):
    """--verifyrand per block: the file as the write's -b / -s cut it"""
    return vrm.file_random_content(size, block, pct, seed, file_key)


def grain_content(size, grain, pct, seed, file_key, dedupe_pct=0):
    """--verifyrandgrain (and --dedupepct)"""
    return vrg.file_content(size, grain, pct, seed, file_key, dedupe_pct)


def sector_records(expected, actual, ranges):
    """ranges: [(offset, length)] of one file -> [(sector, part, count, first, last)] of the
    damaged sectors, one per range and sector (first / last: file offsets)"""
    want = np.frombuffer(expected, dtype=np.uint8)
    got = np.frombuffer(actual, dtype=np.uint8)
    records = []
    for off, length in ranges:
        bad = off + np.flatnonzero(got[off:off + length] != want[off:off + length])
        for sector in np.unique(bad // SECTOR):
            in_sector = bad[bad // SECTOR == sector]
            part = max(off, int(sector) * SECTOR) - int(sector) * SECTOR
            records.append((int(sector), part, len(in_sector), int(in_sector[0]),
                            int(in_sector[-1])))
    return records


def merge(records_by_path):
    """{path: [(sector, part, count, first, last)]} -> [(path, offset, length, bytes)]"""
    lines = []
    for path in sorted(records_by_path):
        parts = collections.defaultdict(dict)  # sector -> part -> count
        bounds = {}                            # sector -> (first, last)
        for sector, part, count, first, last in records_by_path[path]:
            parts[sector][part] = max(parts[sector].get(part, 0), count)
            lo, hi = bounds.get(sector, (first, last))
            bounds[sector] = (min(lo, first), max(hi, last))
        extent = None
        for sector in sorted(parts):
            total = sum(parts[sector].values())
            if extent and sector == extent[1] + 1:
                extent = [extent[0], sector, extent[2], bounds[sector][1], extent[4] + total]
            else:
                if extent:
                    lines.append((path, extent[2], extent[3] - extent[2] + 1, extent[4]))
                extent = [sector, sector, bounds[sector][0], bounds[sector][1], total]
        if extent:
            lines.append((path, extent[2], extent[3] - extent[2] + 1, extent[4]))
    return lines


def extents(files, ranges_by_path):
    """files: {path: (expected bytes, actual bytes)}; ranges_by_path: {path: [(offset, length)]}
    -> the sorted extent lines [(path, offset, length, differing bytes)]"""
    return merge({path: sector_records(exp, act, ranges_by_path.get(path, []))
                  for path, (exp, act) in files.items()})


def runs_of_block(records):
    """the runs (consecutive damaged sectors) of one block's records, sorted by sector"""
    runs, run = [], None
    for rec in sorted(records):
        if run and rec[0] == run[-1][0] + 1:
            run.append(rec)
        else:
            run = [rec]
            runs.append(run)
    return runs


def truncate_runs(block_records, max_runs):
    """a worker's runs in submission order: the first max_runs are listed, the others are counted
    -> (listed records, number of runs left out, their differing bytes)"""
    listed, dropped_runs, dropped_bytes, num_runs = [], 0, 0, 0
    for records in block_records:
        for run in runs_of_block(records):
            if num_runs < max_runs:
                listed += run
            else:
                dropped_runs += 1
                dropped_bytes += sum(rec[2] for rec in run)
            num_runs += 1
    return listed, dropped_runs, dropped_bytes


def report_text(lines, dropped_runs=0, dropped_bytes=0):
    """the text of elb_mgr_verify_report for the lines"""
    text = "".join("%s\t%d\t%d\t%d\n" % line for line in lines)
    if dropped_runs:
        text += "# truncated: %d more extents, %d differing bytes not listed\n" % (dropped_runs,
                                                                                 dropped_bytes)
    return text
