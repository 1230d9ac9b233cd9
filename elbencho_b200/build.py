"""Build of the native library (nvcc, sm_90a only) and of the test oracle.

The product is ONE shared library with a plain C ABI (include/elbencho_b200.h):
``elbencho_b200/libelbencho_b200.so``. It is built in-tree so that it travels to the GPU box with
the repo snapshot.
"""
import os
import shutil
import subprocess

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
REPO_ROOT = os.path.dirname(PKG_DIR)
CSRC_DIR = os.path.join(PKG_DIR, "csrc")
INCLUDE_DIR = os.path.join(REPO_ROOT, "include")
LIB_PATH = os.path.join(PKG_DIR, "libelbencho_b200.so")

SOURCES = [
    "elb_kernels.cu",
    "elb_capi_kernels.cu",
    "elb_dedupe.cu",
    "elb_compress.cu",
    "elb_reduce.cu",
    "elb_cdc.cu",
    "elb_config.cpp",
    "elb_cufile.cpp",
    "elb_worker.cpp",
    "elb_manager.cpp",
    "elb_statsreduce.cu",
    "elb_cli.cpp",
    "elb_stats.cpp",
    "elb_coordinator.cpp",
    "elb_service.cpp",
]

CLI_PATH = os.path.join(PKG_DIR, "elbencho-b200")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC,-Wall,-Wno-unused-function",
    "-shared", "-cudart", "static",
]


def find_nvcc():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        raise RuntimeError("nvcc not found (needed to build libelbencho_b200.so)")
    return nvcc


def _newest_mtime(paths):
    return max(os.path.getmtime(p) for p in paths)


def native_sources():
    deps = [os.path.join(CSRC_DIR, f) for f in os.listdir(CSRC_DIR)]
    deps.append(os.path.join(INCLUDE_DIR, "elbencho_b200.h"))
    return deps


def needs_rebuild():
    if not os.path.exists(LIB_PATH):
        return True
    return _newest_mtime(native_sources()) > os.path.getmtime(LIB_PATH)


def build_native(force=False, verbose=False):
    """Compile every CUDA/C++ source of the product for sm_90a into LIB_PATH."""
    if not force and not needs_rebuild():
        return LIB_PATH
    cmd = [find_nvcc()] + NVCC_FLAGS + ["-I", INCLUDE_DIR, "-I", CSRC_DIR, "-o", LIB_PATH]
    cmd += [os.path.join(CSRC_DIR, s) for s in SOURCES]
    cmd += ["-lpthread", "-ldl"]
    if verbose:
        print(" ".join(cmd))
    subprocess.run(cmd, check=True, cwd=CSRC_DIR)
    # the command line executable: a main() that calls elb_cli_main of the library next to it
    cli_cmd = ["g++", "-O2", "-std=c++17", "-I", INCLUDE_DIR, "-o", CLI_PATH,
               os.path.join(CSRC_DIR, "elb_main.cpp"), "-L", PKG_DIR, "-lelbencho_b200",
               "-Wl,-rpath,$ORIGIN"]
    if verbose:
        print(" ".join(cli_cmd))
    subprocess.run(cli_cmd, check=True)
    return LIB_PATH


def build_oracle(verbose=False):
    """Build the CPU oracle and the cuFile stand-in (test infrastructure)."""
    oracle_dir = os.path.join(REPO_ROOT, "oracle")
    subprocess.run(["make", "-C", oracle_dir] + ([] if verbose else ["-s"]), check=True)
    # stand-in for libcufile used by the GDS-path tests (test infrastructure as well)
    mock_dir = os.path.join(REPO_ROOT, "tests", "mock_cufile")
    subprocess.run(["make", "-C", mock_dir] + ([] if verbose else ["-s"]), check=True)
    return os.path.join(oracle_dir, "libelb_oracle.so")


if __name__ == "__main__":
    print(build_native(force=True, verbose=True))
    print(build_oracle(verbose=True))
