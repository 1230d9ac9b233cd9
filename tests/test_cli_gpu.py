"""GPU tests of the command line front end and of distributed mode, the way the reference's only
test suite does it (tools/test-examples.sh): black-box runs of the binary, multi-file write with
--verify then read back with a different block size, and two --service instances on localhost
ports driven by a master (:291-353)."""
import json
import os
import shutil
import socket
import subprocess
import tempfile
import time

import pytest

from elbencho_b200.build import CLI_PATH
from tests import oracle_lib

pytestmark = pytest.mark.gpu

MiB = 1 << 20


@pytest.fixture()
def workdir(cuda_device):
    base = "/dev/shm" if os.path.isdir("/dev/shm") else None
    path = tempfile.mkdtemp(prefix="elb_cli_", dir=base)
    yield path
    shutil.rmtree(path, ignore_errors=True)


def run_cli(*args, timeout=300):
    return subprocess.run([CLI_PATH] + list(args), capture_output=True, text=True, timeout=timeout)


def table_value(stdout, phase, result_type, column=-1):
    """value of a result row below the given phase name"""
    in_phase = False
    for line in stdout.splitlines():
        if line.startswith(phase + " "):
            in_phase = True
        elif line and not line.startswith(" ") and in_phase:
            in_phase = False
        if in_phase and result_type in line and ":" in line:
            return line.split(":", 1)[1].split()[column]
    raise AssertionError("row %r of phase %r not found in:\n%s" % (result_type, phase, stdout))


def test_file_write_read_verify_with_result_files(workdir):
    path = os.path.join(workdir, "file.bin")
    csv, jsn, txt = (os.path.join(workdir, n) for n in ("res.csv", "res.json", "res.txt"))
    res = run_cli("-w", "-r", "-t", "2", "-b", "1m", "-s", "16m", "--verify", "1", "--gpuids", "0",
                  "--lat", "--latpercent", "--cpu", "--allelapsed", "--nolive", "--csvfile", csv,
                  "--jsonfile", jsn, "--resfile", txt, "--label", "run1", path)
    assert res.returncode == 0, res.stderr + res.stdout
    assert res.stdout.startswith("OPERATION   RESULT TYPE")
    assert table_value(res.stdout, "WRITE", "Total MiB") == "16"
    assert table_value(res.stdout, "READ", "Total MiB") == "16"
    assert int(table_value(res.stdout, "READ", "IOPS")) > 0
    assert "IO latency" in res.stdout and "IO lat % us" in res.stdout
    assert "Time ms each" in res.stdout
    with open(path, "rb") as f:
        assert f.read() == oracle_lib.fill_pattern(16 * MiB, 0, 1)
    # read back with a different block size (tools/test-examples.sh:226,243)
    res2 = run_cli("-r", "-t", "3", "-b", "128k", "-s", "16m", "--verify", "1", "--gpuids", "0",
                   "--nolive", "--csvfile", csv, path)
    assert res2.returncode == 0, res2.stderr
    assert table_value(res2.stdout, "READ", "Total MiB") == "16"
    lines = open(csv).read().splitlines()
    assert len(lines) == 4 and lines[0].startswith("ISO date,label,path type")  # labels once
    rows = [dict(zip(lines[0].split(","), line.split(","))) for line in lines[1:]]
    assert [r["operation"] for r in rows] == ["WRITE", "READ", "READ"]
    assert rows[0]["label"] == "run1" and rows[0]["MiB [last]"] == "16" and rows[2]["threads"] == "3"
    docs = [json.loads(line) for line in open(jsn).read().splitlines()]
    assert [d["phase_type"] for d in docs] == ["WRITE", "READ"]
    assert docs[1]["last_done"]["bytes"] == str(16 * MiB)
    assert "WRITE" in open(txt).read()
    # corrupt one byte: the CLI ends with the reference's message and exit code 1
    with open(path, "r+b") as f:
        f.seek(5 * MiB + 3)
        f.write(b"\x00" if oracle_lib.fill_pattern(1, 5 * MiB + 3, 1) != b"\x00" else b"\x01")
    res3 = run_cli("-r", "-b", "1m", "-s", "16m", "--verify", "1", "--gpuids", "0", "--nolive", path)
    assert res3.returncode == 1
    assert "ERROR: Data verification failed. Offset: %d; Expected value:" % (5 * MiB + 3) in res3.stderr


def test_dir_mode_full_cycle_and_rwmix(workdir):
    res = run_cli("-d", "-w", "--stat", "-r", "-F", "-D", "-t", "2", "-n", "2", "-N", "3", "-s",
                  "64k", "-b", "64k", "--verify", "1", "--gpuids", "0", "--nolive", "--dirstats",
                  workdir)
    assert res.returncode == 0, res.stderr
    for phase in ("MKDIRS", "WRITE", "STAT", "READ", "RMFILES", "RMDIRS"):
        assert phase in res.stdout
    assert table_value(res.stdout, "MKDIRS", "Dirs total") == "4"
    assert table_value(res.stdout, "WRITE", "Files total") == "12"
    assert table_value(res.stdout, "WRITE", "Dirs total") == "4"
    assert "IOPS" not in res.stdout.split("WRITE")[1].split("---")[0]  # block == file size
    assert os.listdir(workdir) == []
    path = os.path.join(workdir, "mix.bin")
    assert run_cli("-w", "-s", "8m", "--gpuids", "0", "--nolive", path).returncode == 0
    res = run_cli("-w", "-s", "8m", "-b", "64k", "--rwmixpct", "25", "--gpuids", "0", "--nolive",
                  path)
    assert res.returncode == 0, res.stderr
    assert "RWMIX25" in res.stdout and "IOPS read" in res.stdout and "MiB/s total" in res.stdout
    # 128 blocks, reads where (0 + n) % 100 < 25: blocks 0-24 and 100-124 (integer MiB division)
    assert table_value(res.stdout, "RWMIX25", "MiB write") == str((78 * 65536) >> 20)
    assert table_value(res.stdout, "RWMIX25", "MiB read") == str((50 * 65536) >> 20)


def free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def wait_for_port(port):
    for _ in range(200):
        try:
            with socket.create_connection(("127.0.0.1", port), timeout=1):
                return
        except OSError:
            time.sleep(0.05)
    raise AssertionError("service did not start on port %d" % port)


def test_distributed_mode_two_services_on_localhost(workdir):
    """tools/test-examples.sh:291-353: two services on localhost ports, master with
    --hosts localhost:[p1-p2] -t 4 -d -n 8 -w -r -N 16 -s 4k -F -D --verify 1, then --quit"""
    ports = sorted([free_port(), free_port()])
    services = [subprocess.Popen([CLI_PATH, "--service", "--foreground", "--port", str(p)],
                                 stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
                for p in ports]
    hosts = ",".join("127.0.0.1:%d" % p for p in ports)
    try:
        for p in ports:
            wait_for_port(p)
        csv = os.path.join(workdir, "dist.csv")
        res = run_cli("--hosts", hosts, "-t", "4", "-d", "-n", "8", "-w", "-r", "-N", "16", "-s",
                      "4k", "-F", "-D", "--verify", "1", "--gpuids", "0", "--nolive", "--lat",
                      "--csvfile", csv, workdir)
        assert res.returncode == 0, res.stderr + res.stdout
        # 2 services x 4 threads x 8 dirs x 16 files
        assert table_value(res.stdout, "MKDIRS", "Dirs total") == "64"
        assert table_value(res.stdout, "WRITE", "Files total") == "1024"
        assert table_value(res.stdout, "READ", "Files total") == "1024"
        assert table_value(res.stdout, "READ", "Total MiB") == "4"
        assert table_value(res.stdout, "RMFILES", "Files total") == "1024"
        assert "Files latency" in res.stdout
        rows = open(csv).read().splitlines()
        header = rows[0].split(",")
        first = dict(zip(header, rows[1].split(",")))
        assert first["hosts"] == "2" and first["threads"] == "4" and first["shared paths"] == "1"
        assert sorted(os.listdir(workdir)) == ["dist.csv"]  # -F -D removed everything else

        # shared file across the two services: ranks 0-3 on service 0, 4-7 on service 1
        path = os.path.join(workdir, "shared.bin")
        res = run_cli("--hosts", hosts, "-t", "4", "-w", "-r", "-b", "64k", "-s", "9m", "--verify",
                      "5", "--gpuids", "0", "--nolive", path)
        assert res.returncode == 0, res.stderr + res.stdout
        assert table_value(res.stdout, "WRITE", "Total MiB") == "9"
        with open(path, "rb") as f:
            assert f.read() == oracle_lib.fill_pattern(9 * MiB, 0, 5)
        # a verify error on a service reaches the master with the reference's text
        with open(path, "r+b") as f:
            f.seek(8 * MiB)
            f.write(b"\xAB")
        res = run_cli("--hosts", hosts, "-t", "4", "-r", "-b", "64k", "-s", "9m", "--verify", "5",
                      "--gpuids", "0", "--nolive", path)
        assert res.returncode == 1
        assert "Data verification failed. Offset: %d;" % (8 * MiB) in res.stderr
        # the services survive and serve the next run
        res = run_cli("--hosts", hosts, "-t", "2", "-w", "-b", "64k", "-s", "1m", "--gpuids", "0",
                      "--nolive", path)
        assert res.returncode == 0, res.stderr
        assert run_cli("--hosts", hosts, "--quit").returncode == 0
        for svc in services:
            svc.wait(timeout=30)
            assert svc.returncode == 0
    finally:
        for svc in services:
            if svc.poll() is None:
                svc.kill()


def test_travelling_options_through_a_service_match_a_local_run(workdir):
    """options that travel to a service, off their defaults: a run through one local service
    writes the bytes of a local run, counts the same entries and bytes and verifies cleanly"""
    common = ["-t", "2", "-b", "64k", "-s", "8m", "--gpuids", "0", "--nolive"]
    verify = ["--verifyrand", "7", "--verifyrandgrain", "64k", "--dedupepct", "20",
              "--blockvarpct", "37"]
    runs = [  # (command, file name, bytes); the read reads the file of the verified write
        (["-w", "--blockvarpct", "37", "--blockvarseed", "5", "--iodepth", "4", "--trunc",
          "--staging", "kernel", "--batchblocks", "3", "--numbatches", "2", "--nogpunuma"],
         "plain", 8 * MiB),
        (["-w"] + verify, "verified", 8 * MiB),
        (["-r", "--rand", "--norandalign", "--randseed", "9", "--randamount", "3m"] + verify,
         "verified", 3 * MiB)]
    port = free_port()
    service = subprocess.Popen([CLI_PATH, "--service", "--foreground", "--port", str(port)],
                               stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    try:
        wait_for_port(port)
        for idx, (command, name, num_bytes) in enumerate(runs):
            totals = []
            for where, hosts in (("local", []), ("svc", ["--hosts", "127.0.0.1:%d" % port])):
                json_path = os.path.join(workdir, "%s_%d.json" % (where, idx))
                res = run_cli(*hosts, *common, *command, "--jsonfile", json_path,
                              os.path.join(workdir, where + "_" + name))
                assert res.returncode == 0, res.stdout + res.stderr
                with open(json_path) as f:
                    totals.append(json.loads(f.read())["last_done"])
            assert totals[0]["bytes"] == totals[1]["bytes"] == str(num_bytes)
            assert totals[0].get("entries") == totals[1].get("entries")
            with open(os.path.join(workdir, "local_" + name), "rb") as local, \
                    open(os.path.join(workdir, "svc_" + name), "rb") as remote:
                assert local.read() == remote.read()
        assert run_cli("--hosts", "127.0.0.1:%d" % port, "--quit").returncode == 0
        service.wait(timeout=30)
    finally:
        if service.poll() is None:
            service.kill()


def test_rate_limit_infloop_livecsv_and_start_time(workdir):
    """run control options of the reference: --limitwrite (RateLimiter.h), --infloop +
    --timelimit (LocalWorker.cpp:196-364), --livecsv (Statistics.cpp:2944-3113), --start"""
    path = os.path.join(workdir, "ctl.bin")
    # 2 threads x 8 MiB at 4 MiB/s per thread: the second half of each share has to wait one second
    t0 = time.time()
    res = run_cli("-w", "-t", "2", "-b", "1M", "-s", "16M", "--gpuids", "0", "--limitwrite", "4M",
                  "--nolive", path)
    elapsed = time.time() - t0
    assert res.returncode == 0, res.stdout + res.stderr
    assert elapsed >= 1.0
    assert int(table_value(res.stdout, "WRITE", "Total MiB")) == 16
    assert int(table_value(res.stdout, "WRITE", "Throughput MiB/s")) <= 16

    # infinite loop over a small file, stopped by the time limit: more bytes than the file holds
    live_csv = os.path.join(workdir, "live.csv")
    res = run_cli("-r", "-t", "2", "-b", "1M", "-s", "16M", "--gpuids", "0", "--infloop",
                  "--timelimit", "2", "--liveint", "200", "--livecsv", live_csv, path, timeout=120)
    assert res.returncode == 0, res.stdout + res.stderr
    assert int(table_value(res.stdout, "READ", "Total MiB")) > 16
    with open(live_csv) as f:
        lines = f.read().splitlines()
    assert lines[0].startswith("ISO Date,Label,Phase,RuntimeMS,Rank,MixType,Done%,DoneBytes,MiB/s,")
    assert len(lines[0].split(",")) == 18  # 17 columns + trailing comma
    rows = [line.split(",") for line in lines[1:]]
    assert len(rows) >= 3
    assert all(row[2] == "READ" and row[4] == "Total" and len(row) == 18 for row in rows)
    done_bytes = [int(row[7]) for row in rows]
    assert done_bytes == sorted(done_bytes) and done_bytes[-1] > 0
    assert all(int(row[14]) == 2 for row in rows[:2])  # both threads active

    # --livecsvex adds one line per worker (rank in column 5, no per-second values)
    live_csv_ex = os.path.join(workdir, "live_ex.csv")
    res = run_cli("-r", "-t", "2", "-b", "1M", "-s", "16M", "--gpuids", "0", "--infloop",
                  "--timelimit", "1", "--liveint", "200", "--livecsv", live_csv_ex, "--livecsvex",
                  path, timeout=120)
    assert res.returncode == 0, res.stdout + res.stderr
    with open(live_csv_ex) as f:
        rows = [line.split(",") for line in f.read().splitlines()[1:]]
    ranks = [row[4] for row in rows[:3]]
    assert ranks == ["Total", "0", "1"], ranks
    assert all(len(row) == 18 for row in rows)
    assert rows[1][8] == "" and rows[1][9] == ""  # no MiB/s and IOPS per worker
    # (the per-worker values are read a moment after the totals)
    assert abs(int(rows[0][7]) - int(rows[1][7]) - int(rows[2][7])) <= 256 * MiB

    # a start time in the past is an error (Coordinator.cpp:151-152), one 2 s ahead is waited for
    res = run_cli("-r", "-b", "1M", "-s", "16M", "--gpuids", "0", "--start", "1000", path)
    assert res.returncode == 1 and "Defined start time has already passed" in res.stderr
    start = int(time.time()) + 2
    res = run_cli("-r", "-b", "1M", "-s", "16M", "--gpuids", "0", "--nolive", "--start",
                  str(start), path)
    assert res.returncode == 0, res.stdout + res.stderr
    assert time.time() >= start


def test_gpu_per_service_assignment(workdir):
    """--gpuperservice: service i gets GPU gpuids[i % n] (ProgArgs.cpp:3852-3859)"""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    ports = [free_port(), free_port()]
    services = [subprocess.Popen([CLI_PATH, "--service", "--foreground", "--port", str(p)],
                                 stdout=subprocess.PIPE, stderr=subprocess.PIPE) for p in ports]
    try:
        path = os.path.join(workdir, "gps.bin")
        hosts = ",".join("127.0.0.1:%d" % p for p in ports)
        res = run_cli("-w", "-r", "-t", "2", "-b", "1M", "-s", "32M", "--verify", "1", "--gpuids",
                      "0,1", "--gpuperservice", "--hosts", hosts, "--svcwait", "20", path)
        assert res.returncode == 0, res.stdout + res.stderr
        assert int(table_value(res.stdout, "READ", "Total MiB")) == 32
    finally:
        run_cli("--quit", "--hosts", hosts)
        for svc in services:
            try:
                svc.wait(timeout=20)
            except subprocess.TimeoutExpired:
                svc.kill()


def test_time_limit_ends_the_run_after_the_current_phase(workdir):
    """an expired --timelimit is no error: the phase's results are printed, later phases are not
    started (Coordinator.cpp:111-116, 234-241); same through services, which apply the limit
    themselves"""
    path = os.path.join(workdir, "tl.bin")
    res = run_cli("-w", "-r", "-t", "2", "-b", "1M", "-s", "16M", "--gpuids", "0", "--infloop",
                  "--timelimit", "1", "--nolive", path, timeout=120)
    assert res.returncode == 0, res.stdout + res.stderr
    assert "Terminating due to phase time limit." in res.stdout
    assert int(table_value(res.stdout, "WRITE", "Total MiB")) > 16
    assert "\nREAD " not in res.stdout

    ports = [free_port(), free_port()]
    hosts = ",".join("127.0.0.1:%d" % p for p in ports)
    services = [subprocess.Popen([CLI_PATH, "--service", "--foreground", "--port", str(p)],
                                 stdout=subprocess.PIPE, stderr=subprocess.PIPE) for p in ports]
    try:
        res = run_cli("-w", "-r", "-t", "2", "-b", "1M", "-s", "16M", "--gpuids", "0", "--infloop",
                      "--timelimit", "1", "--nolive", "--hosts", hosts, "--svcwait", "30", path,
                      timeout=120)
        assert res.returncode == 0, res.stdout + res.stderr
        assert "Terminating due to phase time limit." in res.stdout
        assert int(table_value(res.stdout, "WRITE", "Total MiB")) > 16
        assert "\nREAD " not in res.stdout
    finally:
        run_cli("--quit", "--hosts", hosts)
        for svc in services:
            try:
                svc.wait(timeout=20)
            except subprocess.TimeoutExpired:
                svc.kill()


def test_file_size_is_detected_when_not_given(workdir):
    """no -s for an existing file: the file's own size is used; a larger -s than the file holds is
    an error in a read-only run; an empty new file without -s too (ProgArgs.cpp:2071-2104)"""
    path = os.path.join(workdir, "auto.bin")
    res = run_cli("-w", "-t", "2", "-b", "1M", "-s", "24M", "--verify", "1", "--gpuids", "0",
                  "--nolive", path)
    assert res.returncode == 0, res.stdout + res.stderr
    res = run_cli("-r", "-t", "2", "-b", "1M", "--verify", "1", "--gpuids", "0", "--nolive", path)
    assert res.returncode == 0, res.stdout + res.stderr
    assert int(table_value(res.stdout, "READ", "Total MiB")) == 24
    res = run_cli("-r", "-t", "2", "-b", "4K", "--rand", "--iodepth", "8", "--verify", "1",
                  "--gpuids", "0", "--nolive", path)
    assert res.returncode == 0, res.stdout + res.stderr
    assert int(table_value(res.stdout, "READ", "Total MiB")) == 24  # randamount = file size
    res = run_cli("-r", "-b", "1M", "-s", "32M", "--gpuids", "0", "--nolive", path)
    assert res.returncode == 1
    assert "Given size to use is larger than detected size." in res.stderr
    assert "Detected size: %d; Given size: %d" % (24 * MiB, 32 * MiB) in res.stderr
    res = run_cli("-r", "-b", "1M", "--gpuids", "0", "--nolive", os.path.join(workdir, "new.bin"))
    assert res.returncode == 1
    assert "File size must not be 0 when benchmark path is a file." in res.stderr
