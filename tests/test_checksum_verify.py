"""CPU tests of --checksumchunk and --checksumverify: the list parser (good lists, the last chunked
section winning, blanks in paths, malformed lines and their line numbers), the command line and
config rejections, the help texts, dry runs, the elb_cfg field and the finish of partial chunks."""
import ctypes
import random
import zlib

import pytest

from elbencho_b200 import WorkerConfig, WorkerError, WorkerManager, _native, kernels
from tests import crc_model as model
from tests.test_cli import run_cli

KiB, MiB = 1 << 10, 1 << 20

CLI = ["-r", "-b", "256k", "-s", "4m", "--gpuids", "0"]


def write(path, text):
    path.write_text(text)
    return str(path)


GOOD = ("# phase WRITE chunk 65536\n"
        "/d/a 0 65536 0000abcd\n"
        "/d/a 65536 100 DEADBEEF\n")


def manager(tmp_path, **kwargs):
    args = dict(paths=[str(tmp_path / "f")], block_size=256 * KiB, file_size=MiB)
    args.update(kwargs)
    return WorkerManager(WorkerConfig(**args))


def dry_run(tmp_path, text, *extra):
    """the command line parses the list with the library's parser before anything runs"""
    lst = write(tmp_path / "list", text)
    return run_cli("--dryrun", *CLI, *extra, "--checksumverify", lst, str(tmp_path / "data"))


@pytest.mark.parametrize("text", [
    GOOD, "\n" + GOOD + "\n", "# phase READ chunk 4096\n/x y z 0 4096 00000000\n",
    "# phase WRITE chunk 4096\n/d/a b  c 4096 4096 00000001\n",  # (blanks in the path)
    "# phase WRITE\n/a 4096 4096 12345678\n" + GOOD + "# phase READ\n/a 4096 4096 -\n",
])
def test_good_lists_parse(tmp_path, text):
    res = dry_run(tmp_path, text)
    assert res.returncode == 0, res.stderr


def test_last_chunked_section_wins(tmp_path):
    text = ("# phase WRITE chunk 4096\n/a 0 4096 00000000\n"
            "# phase READ chunk 65536\n/a 0 65536 00000000\n"
            "# phase READ\n/a 1048576 1048576 12345678\n")
    # the 64 KiB section wins: a 96 KiB block is no multiple of it, of 4 KiB it would be
    res = dry_run(tmp_path, text, "-b", "96k")
    assert res.returncode == 1
    assert "multiple of the chunk size of the checksum list (65536)" in res.stderr, res.stderr
    res = dry_run(tmp_path, text.replace("chunk 65536\n/a 0 65536", "chunk 32768\n/a 0 32768"),
                  "-b", "96k")
    assert res.returncode == 0, res.stderr


@pytest.mark.parametrize("text,line_num,reason", [
    ("/a 0 65536 00000000\n", 1, 'a line before the first "# phase" header'),
    ("# phase WRITE chunk 65536\n/a 0 65536 0000000\n", 2, 'not "path offset length crc32"'),
    ("# phase WRITE chunk 65536\n/a 0 65536 0000000g\n", 2, 'not "path offset length crc32"'),
    ("# phase WRITE chunk 65536\n/a x 65536 00000000\n", 2, 'not "path offset length crc32"'),
    ("# phase WRITE chunk 65536\n0 65536 00000000\n", 2, 'not "path offset length crc32"'),
    ("# phase WRITE chunk 65536\n\n/a 100 65536 00000000\n", 3, "not a chunk of 65536 bytes"),
    ("# phase WRITE chunk 65536\n/a 0 65537 00000000\n", 2, "not a chunk of 65536 bytes"),
    ("# phase WRITE chunk 65536\n/a 0 0 00000000\n", 2, "not a chunk of 65536 bytes"),
    ("# phase WRITE chunk 65536\n/a 0 9 00000000\n/a 0 9 00000000\n", 3,
     "a second line for this path and offset"),
    ("# phase WRITE chunk 65535\n", 1, "the chunk size is not a power of two from 4K to 1G"),
    ("# phase WRITE chunk 2048\n", 1, "the chunk size is not a power of two from 4K to 1G"),
    ("# phase WRITE chunk\n", 1, "not a phase header"),
    ("# phase DELETE\n", 1, "not a phase header"),
    ("# phase READ chunk 4096 x\n", 1, "not a phase header"),
])
def test_malformed_lines_name_their_line(tmp_path, text, line_num, reason):
    res = dry_run(tmp_path, text)
    assert res.returncode == 1
    assert "Checksum list line %d: %s: " % (line_num, reason) in res.stderr, res.stderr


def test_list_without_chunked_section(tmp_path):
    res = dry_run(tmp_path, "# phase WRITE\n/a 4096 4096 12345678\n")
    assert res.returncode == 1
    assert "Checksum list has no section with a chunk size" in res.stderr, res.stderr


def test_set_checksum_list_argument_checks():
    lib = _native.load()
    assert lib.elb_mgr_set_checksum_list(None, b"", 0) == -1
    assert "NULL manager or text" in _native.last_error()


def test_cfg_field_fills_padding():
    assert ctypes.sizeof(_native.Cfg) == _native.load().elb_cfg_struct_size() == 360
    assert _native.Cfg.numDataSetThreads.offset == 32
    assert _native.Cfg.checksumChunkShift.offset == 36
    assert _native.Cfg.blockSize.offset == 40


@pytest.mark.parametrize("kwargs,message", [
    (dict(checksum_chunk_shift=11), "The checksum chunk shift (11) is not in [12, 30]."),
    (dict(checksum_chunk_shift=31), "The checksum chunk shift (31) is not in [12, 30]."),
    (dict(checksum_chunk_shift=16, block_size=96 * KiB),
     "The block size (98304) is not a multiple of the checksum chunk size (--checksumchunk) "
     "(65536)."),
    (dict(checksum_chunk_shift=16, use_random_offsets=True, use_random_unaligned=True),
     "Checksum chunks cannot be used together with unaligned random offsets (--norandalign)."),
])
def test_config_rejection(tmp_path, kwargs, message):
    with pytest.raises(WorkerError) as excinfo:
        manager(tmp_path, checksums=True, **kwargs)
    assert str(excinfo.value) == message


@pytest.mark.parametrize("length", [1, 100, 4095, 4096, 65535, 65536])
def test_finish_of_partial_chunks_is_zlib(length):
    data = random.Random(length).randbytes(length)
    assert kernels.crc32_finish(model.raw_crc(data), length) == zlib.crc32(data)


def test_crc32_chunks_argument_checks():
    lib = _native.load()
    raw = kernels.pack_block_descs([(0x1000, 16, 0, 0)])
    descs = ctypes.create_string_buffer(raw, len(raw))
    crcs = (ctypes.c_uint32 * 4)(0)
    assert lib.elb_crc32_chunks(descs, None, 1, 11, 1, crcs, None, None, None) == -1
    assert "chunk shift 11 is neither 64 nor in [12, 40]" in _native.last_error()
    assert lib.elb_crc32_chunks(descs, None, 1, 12, 0, crcs, None, None, None) == -1
    assert "slots per descriptor must be at least 1" in _native.last_error()
    assert lib.elb_crc32_chunks(descs, None, 1, 64, 1, crcs, None, None, None) == -1
    assert "NULL descriptor, shift or CRC array" in _native.last_error()
    assert lib.elb_crc32_chunks(descs, None, 1, 12, 1, crcs, crcs, None, None) == -1
    assert "host CRCs and device ticket go together" in _native.last_error()
    raw = kernels.pack_block_descs([(0x1000, 8192, 4095, 0)])
    descs = ctypes.create_string_buffer(raw, len(raw))
    assert lib.elb_crc32_chunks(descs, None, 1, 12, 2, crcs, None, None, None) == -1
    assert "descriptor 0 spans 3 chunks, more than 2 slots" in _native.last_error()
    assert lib.elb_crc32_chunks(None, None, 0, 12, 1, None, None, None, None) == 0


# ------------------------------------------------------------------------------------------------
# command line
# ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("extra,message", [
    (["--norandalign", "--rand"], 'Option "--checksumverify" cannot be used together with '
     '"--norandalign"'),
    (["--rwmixpct", "20"], 'Option "--checksumverify" cannot be used together with "--rwmixpct"'),
    (["--rwmixthr", "1", "-t", "2"],
     'Option "--checksumverify" cannot be used together with "--rwmixthr"'),
    (["--hosts", "localhost:1"], 'Option "--checksumverify" cannot be used together with '
     '"--hosts"'),
    (["--verify", "1", "--verifyreport", "/tmp/elb_vr"],
     'Option "--checksumverify" cannot be used together with "--verifyreport"'),
    (["--checksumchunk", "4k", "--checksums", "/tmp/elb_sums"],
     'Option "--checksumchunk" (4096) differs from the chunk size of the checksum list (65536)'),
])
def test_verify_validation_messages(tmp_path, extra, message):
    lst = write(tmp_path / "list", GOOD)
    res = run_cli(*CLI, *extra, "--checksumverify", lst, str(tmp_path / "x"))
    assert res.returncode == 1
    assert message in res.stderr, res.stderr


def test_block_size_must_be_a_multiple_of_the_list_chunk(tmp_path):
    lst = write(tmp_path / "list", GOOD)
    res = run_cli("-r", "-b", "96k", "-s", "4m", "--gpuids", "0", "--checksumverify", lst,
                  str(tmp_path / "x"))
    assert res.returncode == 1
    assert ("The block size (98304) must be a multiple of the chunk size of the checksum list "
            "(65536)") in res.stderr, res.stderr


def test_same_path_as_checksums_rejected(tmp_path):
    lst = write(tmp_path / "list", GOOD)
    res = run_cli(*CLI, "--checksums", lst, "--checksumverify", lst, str(tmp_path / "x"))
    assert res.returncode == 1
    assert 'Options "--checksumverify" and "--checksums" cannot name the same file' in res.stderr


def test_malformed_list_rejected_with_line(tmp_path):
    lst = write(tmp_path / "list", GOOD + "/d/a 131072 65536 xyz\n")
    res = run_cli(*CLI, "--checksumverify", lst, str(tmp_path / "x"))
    assert res.returncode == 1
    assert "Checksum list line 4: not \"path offset length crc32\"" in res.stderr, res.stderr


def test_missing_list_rejected(tmp_path):
    res = run_cli(*CLI, "--checksumverify", str(tmp_path / "none"), str(tmp_path / "x"))
    assert res.returncode == 1
    assert "Unable to read checksum list" in res.stderr, res.stderr


@pytest.mark.parametrize("extra,message", [
    ([], 'Option "--checksumchunk" requires "--checksums" or "--checksumverify"'),
    (["--checksums", "/tmp/elb_sums", "-b", "96k"],
     'The block size (98304) must be a multiple of "--checksumchunk" (65536)'),
    (["--checksums", "/tmp/elb_sums", "--norandalign"],
     'Option "--checksumchunk" cannot be used together with "--norandalign"'),
    (["--checksums", "/tmp/elb_sums", "--rand"],
     'Option "--checksums" cannot be used together with "--rand"'),
    (["--checksums", "/tmp/elb_sums", "--infloop", "--timelimit", "1"],
     'Option "--checksums" cannot be used together with "--infloop"'),
])
def test_chunk_validation_messages(tmp_path, extra, message):
    res = run_cli(*CLI, "--checksumchunk", "64k", *extra, str(tmp_path / "x"))
    assert res.returncode == 1
    assert message in res.stderr, res.stderr


@pytest.mark.parametrize("size", ["2k", "48k", "2g"])
def test_chunk_size_range(tmp_path, size):
    res = run_cli(*CLI, "--checksums", str(tmp_path / "s"), "--checksumchunk", size,
                  str(tmp_path / "x"))
    assert res.returncode == 1
    assert 'Option "--checksumchunk" must be a power of two from 4K to 1G' in res.stderr


@pytest.mark.parametrize("args", [
    ["--checksums", "SUMS", "--checksumchunk", "64k"],
    ["--checksumverify", "LIST"],
    ["--checksumverify", "LIST", "--checksumchunk", "64k", "--rand", "--randamount", "2m"],
    ["--checksumverify", "LIST", "--infloop", "--timelimit", "1", "--verify", "3"],
    ["--checksumverify", "LIST", "--checksums", "SUMS", "-b", "1m"],
])
def test_accepted_combinations(tmp_path, args):
    lst = write(tmp_path / "list", GOOD)
    args = [a.replace("SUMS", str(tmp_path / "sums")).replace("LIST", lst) for a in args]
    res = run_cli("--dryrun", *CLI, *args, str(tmp_path / "data"))
    assert res.returncode == 0, res.stderr


def test_help_lists_the_options():
    res = run_cli("--help-all")
    assert res.returncode == 0
    text = " ".join(res.stdout.split())
    assert "--checksumchunk" in text and "--checksumverify" in text
    assert "# phase WRITE|READ chunk <K>" in text
    assert ("Cannot be used with --norandalign, --rwmixpct, --rwmixthr, --hosts or "
            "--verifyreport.") in text
