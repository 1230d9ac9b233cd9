"""The options that travel from a master to its services in the /preparephase tree (CPU only): the
trees that the master sends, against goldens, and the keys that a real --service reads, each with
its type. The service reads every key before it rejects an empty "gpuids" and before it touches
a GPU."""
import http.client
import json
import subprocess
import time

from elbencho_b200.build import CLI_PATH
from tests import option_wire_golden as wire
from tests.test_master_fake_services import free_port, run_master

# keys of reference modes and options that this build does not have: sent with fixed values
FIXED_KEYS = {"benchmode", "cufiledriveropen", "cuhostbufreg", "hdfs", "madv", "mmap", "netbench",
              "netbenchservers", "numservers", "opslog", "opsloglock", "recvbuf", "respsize",
              "sendbuf"}

# the number and true/false keys that a service reads; the others (no0usecerr, the fixed keys
# other than mmap, hdfs and netbench) are for reference services only
READ_KEYS = {
    "b200_batchblocks", "b200_blockvarseed", "b200_dedupepct", "b200_nogpunuma",
    "b200_nowritegate", "b200_numbatches", "b200_randseed", "b200_timelimit", "b200_verifyrand",
    "b200_verifyrandgrain", "b200_writegate", "backward", "block", "blockvarpct", "cufile",
    "datasetthreads", "deldirs", "delfiles", "direct", "dirs", "dirsharing", "dropcache", "fadv",
    "files", "flock", "gdsbufreg", "hdfs", "infloop", "iodepth", "limitread", "limitwrite",
    "mkdirs", "mmap", "netbench", "nodelerr", "nodiocheck", "nofdsharing", "norandalign",
    "preallocfile", "rand", "randamount", "rankoffset", "read", "readinline", "rwmixpct",
    "rwmixthr", "rwmixthrpct", "sharesize", "size", "stat", "statinline", "strided", "sync",
    "threads", "treerand", "treeroundup", "trunc", "trunctosize", "verify", "verifydirect",
    "write"}


def load_golden():
    with open(wire.GOLDEN) as f:
        return json.load(f)


def test_master_sends_the_golden_trees():
    golden = load_golden()
    assert [wire.capture(CLI_PATH, line) for line in wire.FULL_LINES] == golden["full"]
    assert wire.capture(CLI_PATH, wire.REQUIRED_LINE) == golden["required"]
    # every key but the fixed ones has another value in one of the full lines
    required = golden["required"]
    unmoved = {key for key, value in required.items()
               if all(tree[key] == value for tree in golden["full"])}
    assert unmoved == FIXED_KEYS | {key for key in required if key.startswith("s3")}


def test_service_reads_exactly_the_travelling_keys(tmp_path):
    tree = dict(load_golden()["required"], gpuids="")
    tree["path"] = tree["path"].replace(wire.DIR, str(tmp_path))
    port = free_port()
    svc = subprocess.Popen([CLI_PATH, "--service", "--foreground", "--port", str(port)],
                           stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    try:
        for _ in range(100):
            try:
                conn = http.client.HTTPConnection("127.0.0.1", port, timeout=5)
                conn.request("GET", "/protocolversion")
                assert conn.getresponse().read() == b"3.1.1"
                break
            except OSError:
                time.sleep(0.1)

        def prepare(sent):
            conn.request("POST", "/preparephase?ProtocolVersion=3.1.1&PwHash=", json.dumps(sent))
            response = conn.getresponse()
            body = response.read().decode()
            assert response.status == 400
            return body

        assert '"--gpuids"' in prepare(tree)
        checked = set()
        for key, value in tree.items():
            if key == "gpuids" or not (value.isdigit() or value in ("true", "false")):
                continue
            body = prepare(dict(tree, **{key: "x"}))
            if key in READ_KEYS:
                assert "conversion of data to type failed (%s=x)" % key in body, body
            else:
                assert '"--gpuids"' in body, (key, body)
            checked.add(key)
        assert READ_KEYS <= checked
        for key in ("block", "size", "path"):
            body = prepare({k: v for k, v in tree.items() if k != key})
            assert "No such node (%s)" % key in body, body
        conn.close()
    finally:
        run_master("--quit", "--hosts", "127.0.0.1:%d" % port)
        try:
            svc.wait(timeout=20)
        except subprocess.TimeoutExpired:
            svc.kill()
