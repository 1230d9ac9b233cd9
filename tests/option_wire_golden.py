"""The /preparephase trees that a master sends to its services for the command lines below, stored
as tests/golden/option_wire.json and checked by tests/test_option_wire.py. The golden pins the keys
and values on the wire; capture it again only on purpose, with the binary whose wire it should pin:

    python -m tests.option_wire_golden [path/to/elbencho-b200]
"""
import json
import os
import subprocess
import sys
import tempfile

from elbencho_b200.build import CLI_PATH
from tests.test_master_fake_services import FakeService

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "option_wire.json")
DIR = "<dir>"  # the benchmark directory, which holds tree.txt for --treefile
TREE_FILE = "d d1\nf 1048576 d1/a\n"

# Between them, these lines give every option that travels a value other than the one it has in
# REQUIRED_LINE. One line cannot do it: --verify excludes --verifyrand, --rwmixpct and random
# writes, --rwmixpct excludes --rwmixthr, --verifyrand excludes --treefile, and --iodepth excludes
# --verifydirect and --readinline. The lines with --rwmixpct or --rwmixthr only read, because the
# fake service has no results of a mixed write phase.
FULL_LINES = [
    ["-d", "-w", "-r", "--stat", "-F", "-D", "--sync", "--dropcache", "-t", "3", "-n", "2", "-N",
     "5", "-s", "256k", "-b", "64k", "--verify", "9", "--verifydirect", "--direct", "--dirsharing",
     "--trunc", "--trunctosize", "--preallocfile", "--nodelerr", "--backward", "--strided",
     "--cufile", "--gdsbufreg", "--nofdsharing", "--label", "wire golden", "--statinline",
     "--nodiocheck", "--infloop", "--timelimit", "30", "--limitread", "7M", "--limitwrite", "5M",
     "--rankoffset", "4", "--flock", "range", "--fadv", "seq,dontneed", "--blockvaralgo",
     "balanced", "--no0usecerr", "--writegate", "--nogpunuma", "--gpuids", "0,1", DIR],
    ["-r", "-t", "2", "-s", "1M", "-b", "4k", "--iodepth", "4", "--rand", "--randamount",
     "512k", "--norandalign", "--randalgo", "fast", "--randseed", "11", "--blockvarpct", "37",
     "--blockvarseed", "5", "--rwmixpct", "20", "--batchblocks", "3", "--numbatches", "2",
     "--nowritegate", "--staging", "kernel", "--gpuids", "0", DIR + "/f"],
    ["-r", "-t", "2", "-s", "1M", "-b", "64k", "--verifyrand", "7", "--verifyrandgrain",
     "64k", "--dedupepct", "20", "--readinline", "--rwmixthr", "1", "--rwmixthrpct", "30",
     "--gpuids", "0", DIR + "/f"],
    ["-w", "--treefile", DIR + "/tree.txt", "--treerand", "--treeroundup", "4k", "--sharesize",
     "2M", "--gpuids", "0", DIR],
]
REQUIRED_LINE = ["-w", "-b", "1M", "-s", "1M", "--gpuids", "0", DIR + "/f"]


def capture(cli_path, args):
    """the tree that the master sends to one fake service for args, with DIR for the temporary
    benchmark directory"""
    with tempfile.TemporaryDirectory() as tmp:
        with open(os.path.join(tmp, "tree.txt"), "w") as f:
            f.write(TREE_FILE)
        svc = FakeService(1 << 20, [1000]).start()
        try:
            res = subprocess.run([cli_path] + [arg.replace(DIR, tmp) for arg in args] +
                                 ["--hosts", "127.0.0.1:%d" % svc.port, "--nolive", "--svcupint",
                                  "50"], capture_output=True, text=True, timeout=120)
        finally:
            svc.stop()
        assert res.returncode == 0, res.stdout + res.stderr
        assert len(svc.prepare_trees) == 1
        return {key: value.replace(tmp, DIR) for key, value in svc.prepare_trees[0].items()}


def main():
    cli_path = sys.argv[1] if len(sys.argv) > 1 else CLI_PATH
    golden = {"full": [capture(cli_path, line) for line in FULL_LINES],
              "required": capture(cli_path, REQUIRED_LINE)}
    with open(GOLDEN, "w") as f:
        json.dump(golden, f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote", GOLDEN)


if __name__ == "__main__":
    main()
