"""One phase sequence and one results writer for local and distributed runs: what a distributed run
shares with a local one (--phasedelay between phases, the errors and the skip line of the results
file), checked against fake services, and the phase-start date of the CSV and JSON results of a
local run on the GPU."""
import json
import os
import re
import time

import pytest

from tests.test_master_fake_services import MiB, FakeService, run_master

ISO_DATE_MILLIS = re.compile(r"\d{4}-\d\d-\d\dT\d\d:\d\d:\d\d\.\d{3}[+-]\d{4}")


class TimedService(FakeService):
    """a fake service that also records when each request arrived"""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.arrivals = []  # (path, time)

    def dispatch(self, method, path, query, body):
        self.arrivals.append((path, time.time()))
        return super().dispatch(method, path, query, body)


def test_distributed_run_sleeps_phasedelay_between_phases(tmp_path):
    svc = TimedService(8 * MiB, [1000]).start()
    try:
        res = run_master("-w", "-r", "-t", "1", "-b", "1M", "-s", "8M", "--gpuids", "0", "--hosts",
                         "127.0.0.1:%d" % svc.port, "--nolive", "--svcupint", "50",
                         "--phasedelay", "1", str(tmp_path / "f"))
        assert res.returncode == 0, res.stdout + res.stderr
    finally:
        svc.stop()
    starts = [t for path, t in svc.arrivals if path == "/startphase"]
    results = [t for path, t in svc.arrivals if path == "/benchresult"]
    assert len(starts) == 2 and len(results) == 2
    assert starts[1] - results[0] >= 1.0


def test_distributed_run_reports_a_results_file_it_cannot_open(tmp_path):
    svc = FakeService(8 * MiB, [1000]).start()
    res_path = tmp_path / "no_such_dir" / "r.txt"
    try:
        res = run_master("-w", "-t", "1", "-b", "1M", "-s", "8M", "--gpuids", "0", "--hosts",
                         "127.0.0.1:%d" % svc.port, "--nolive", "--svcupint", "50",
                         "--resfile", str(res_path), str(tmp_path / "f"))
    finally:
        svc.stop()
    assert res.returncode == 0, res.stdout + res.stderr
    assert "ERROR: Opening results file failed: %s" % res_path in res.stderr
    assert "WRITE" in res.stdout


def test_distributed_run_without_worker_results_says_so_in_the_results_file(tmp_path):
    svc = FakeService(8 * MiB, []).start()
    res_path = tmp_path / "r.txt"
    try:
        res = run_master("-w", "-t", "1", "-b", "1M", "-s", "8M", "--gpuids", "0", "--hosts",
                         "127.0.0.1:%d" % svc.port, "--nolive", "--svcupint", "50",
                         "--resfile", str(res_path), str(tmp_path / "f"))
    finally:
        svc.stop()
    assert res.returncode == 0, res.stdout + res.stderr
    assert "Skipping stats print due to unavailable worker results." in res.stdout
    assert res_path.read_text() == "Skipping stats print due to unavailable worker results.\n\n"


@pytest.mark.gpu
def test_local_results_share_the_phase_start_date_with_millis(cuda_device, tmp_path):
    from tests.test_cli_gpu import run_cli
    base = "/dev/shm" if os.path.isdir("/dev/shm") else str(tmp_path)
    path = os.path.join(base, "elb_phase_reporting_%d.bin" % os.getpid())
    csv, jsn = tmp_path / "r.csv", tmp_path / "r.json"
    try:
        res = run_cli("-w", "-r", "-t", "1", "-b", "1m", "-s", "8m", "--gpuids", "0", "--nolive",
                      "--csvfile", str(csv), "--jsonfile", str(jsn), path)
        assert res.returncode == 0, res.stderr + res.stdout
    finally:
        if os.path.exists(path):
            os.unlink(path)
    lines = csv.read_text().splitlines()
    assert len(lines) == 3 and lines[0].startswith("ISO date,")
    csv_dates = [line.split(",")[0] for line in lines[1:]]
    json_dates = [json.loads(line)["iso_start_date"] for line in jsn.read_text().splitlines()]
    assert csv_dates == json_dates
    for date in csv_dates:
        assert ISO_DATE_MILLIS.fullmatch(date), date
