"""GPU tests of the --checksums report across a checksum list: the report lists what its phase
computed, even after a list of another algorithm or chunk size is set for the next phases, and a
read that checks a CRC list and lists its chunks lists the values it checked."""
import os
import shutil

import numpy as np
import pytest

from tests import test_checksums_gpu as base  # noqa: F401  (sets the mock cuFile library first)
from elbencho_b200 import BenchPhase, WorkerConfig, WorkerManager  # noqa: E402
from tests.test_checksums_gpu import make_workdir  # noqa: E402

pytestmark = pytest.mark.gpu

MiB = 1 << 20
SIZE, SHIFT = 4 * MiB, 16
DIGITS = {"crc32": 8, "crc32c": 8, "crc64nvme": 16, "blake3": 64}


@pytest.fixture()
def workdir(cuda_device):
    path = make_workdir()
    yield path
    shutil.rmtree(path, ignore_errors=True)


def zero_list(path, algo):
    """a chunked list of SIZE bytes of path with all-zero values (it is set, never checked)"""
    return "# phase WRITE chunk %d %s\n" % (1 << SHIFT, algo) + "".join(
        "%s %d %d %s\n" % (path, off, 1 << SHIFT, "0" * DIGITS[algo])
        for off in range(0, SIZE, 1 << SHIFT))


@pytest.mark.parametrize("chunk_shift", [0, SHIFT])
@pytest.mark.parametrize("list_algo", ["blake3", "crc64nvme"])
def test_report_keeps_the_phase_algorithm_after_a_list(workdir, chunk_shift, list_algo):
    path = os.path.join(workdir, "f")
    cfg = WorkerConfig(paths=[path], file_size=SIZE, block_size=MiB, num_threads=2,
                       checksums=True, checksum_chunk_shift=chunk_shift,
                       block_variance_percent=100)
    with WorkerManager(cfg) as mgr:
        mgr.run_phase(BenchPhase.CREATEFILES)
        written = mgr.checksums_text()
        mgr.set_checksum_list(zero_list(path, list_algo))
        assert mgr.checksums_text() == written
    lines = written.splitlines()
    assert len(lines) == (SIZE >> SHIFT if chunk_shift else 1)
    assert all(len(line.rsplit(" ", 1)[1]) == DIGITS["crc32"] for line in lines)


def test_checked_and_listed_read_lists_the_checked_values(workdir):
    path = os.path.join(workdir, "f")
    with open(path, "wb") as f:
        f.write(np.random.default_rng(7).integers(0, 256, SIZE, dtype=np.uint8).tobytes())
    cfg = WorkerConfig(paths=[path], file_size=SIZE, block_size=MiB, num_threads=2,
                       checksums=True, checksum_chunk_shift=SHIFT, checksum_algo="crc32c")
    with WorkerManager(cfg) as mgr:
        mgr.run_phase(BenchPhase.READFILES)
        listed = mgr.checksums_text()
        mgr.set_checksum_list("# phase READ chunk %d crc32c\n" % (1 << SHIFT) + listed)
        mgr.run_phase(BenchPhase.READFILES)
        assert mgr.checksum_verify_counts() == (SIZE >> SHIFT, 1)
        assert mgr.checksums_text() == listed
