"""CPU tests of the kernel-level C ABI's argument checks: every fill / verify entry point of the
binding table, each rejection it makes with its exact error text and in its order, and the early
returns that launch nothing. None of these calls reaches CUDA, so they run without a GPU."""
import re

import pytest

from elbencho_b200 import _native

P = 0x1000  # a non-NULL pointer; no call below dereferences it
N = None
SALT, SEED, KEY, DELTA = 0x5A17, 0xBEEF, 3, 1 << 20

PCT_101 = "Block variance percent must be in range 0..100. Given: 101"
ALGO_1 = "Unknown random fill algorithm: 1"
SHIFT = "Random verify grain shift must be in range 12..30. Given: %d"


class Args:
    """the arguments of one call: valid content and NULL data pointers by default"""

    def __init__(self, ptr=N, len=0, out=N, descs=N, n=0, results=N, pct=50, algo=0, shift=12):
        self.ptr, self.len, self.out = ptr, len, out
        self.descs, self.n, self.results = descs, n, results
        self.pct, self.algo, self.shift = pct, algo, shift


# entry point -> its argument list (include/elbencho_b200.h)
FORMS = {
    "elb_fill_pattern": lambda a: (a.ptr, a.len, 0, SALT, N),
    "elb_verify_pattern": lambda a: (a.ptr, a.len, 0, SALT, a.out, N),
    "elb_fill_random": lambda a: (a.ptr, a.len, a.pct, SEED, KEY, a.algo, N),
    "elb_verify_random": lambda a: (a.ptr, a.len, a.pct, SEED, KEY, a.algo, a.out, N),
    "elb_fill_random_grain": lambda a: (a.ptr, a.len, 0, a.shift, a.pct, SEED, KEY, N),
    "elb_verify_random_grain": lambda a: (a.ptr, a.len, 0, a.shift, a.pct, SEED, KEY, a.out, N),
    "elb_fill_pattern_batch": lambda a: (a.descs, a.n, SALT, N, N),
    "elb_verify_pattern_batch": lambda a: (a.descs, a.n, SALT, a.results, N, N),
    "elb_fill_random_batch": lambda a: (a.descs, a.n, a.pct, SEED, a.algo, N, N),
    "elb_fill_pattern_batch_sized": lambda a: (a.descs, a.n, SALT, N, 0, 0, N),
    "elb_verify_pattern_batch_sized": lambda a: (a.descs, a.n, SALT, a.results, N, 0, 0, N),
    "elb_fill_random_batch_sized": lambda a: (a.descs, a.n, a.pct, SEED, a.algo, N, 0, 0, N),
    "elb_verify_random_batch_sized":
        lambda a: (a.descs, a.n, a.pct, SEED, a.algo, a.results, N, 0, 0, N),
    "elb_fill_random_grain_batch_sized":
        lambda a: (a.descs, a.n, a.shift, a.pct, SEED, N, 0, 0, N),
    "elb_verify_random_grain_batch_sized":
        lambda a: (a.descs, a.n, a.shift, a.pct, SEED, a.results, N, 0, 0, N),
    "elb_fill_pattern_staged": lambda a: (a.descs, a.n, SALT, DELTA, N, 0, 0, N),
    "elb_fill_random_staged": lambda a: (a.descs, a.n, a.pct, SEED, a.algo, DELTA, N, 0, 0, N),
    "elb_fill_random_grain_staged":
        lambda a: (a.descs, a.n, a.shift, a.pct, SEED, DELTA, N, 0, 0, N),
    "elb_verify_pattern_staged":
        lambda a: (a.descs, a.n, SALT, DELTA, a.results, N, N, N, 0, 0, N),
    "elb_verify_random_staged":
        lambda a: (a.descs, a.n, a.pct, SEED, a.algo, DELTA, a.results, N, N, N, 0, 0, N),
    "elb_verify_random_grain_staged":
        lambda a: (a.descs, a.n, a.shift, a.pct, SEED, DELTA, a.results, N, N, N, 0, 0, N),
}

# every fill / verify entry point the binding declares (an entry point FORMS lacks fails below)
ENTRY_POINTS = sorted(n for n in _native.SIGNATURES
                      if re.match(r"elb_(fill|verify)_(pattern|random)", n))
SINGLE = [n for n in ENTRY_POINTS if not re.search(r"_(batch|staged)", n)]
BATCH = [n for n in ENTRY_POINTS if n not in SINGLE]
FILLS = [n for n in ENTRY_POINTS if n.startswith("elb_fill_")]


def kind(name):
    return "grain" if "_random_grain" in name else "random" if "_random" in name else "pattern"


def prefix(name):
    """the error prefix: the _batch_sized forms report as _batch"""
    return re.sub(r"_sized$", "", name)


def call(native, name, args):
    """calls the entry point and returns its result; no call may launch a kernel"""
    before = native.elb_num_kernel_launches()
    res = getattr(native, name)(*FORMS[name](args))
    assert native.elb_num_kernel_launches() == before
    return res


def assert_rejected(native, name, args, text):
    assert call(native, name, args) == -1
    assert _native.last_error() == text


def test_table_has_every_entry_point():
    assert len(ENTRY_POINTS) == 21
    assert sorted(FORMS) == ENTRY_POINTS


def content_cases():
    """(name, overrides, error): the content checks in their order, grain shift, pct, randAlgo"""
    for name in ENTRY_POINTS:
        if kind(name) == "random":
            yield name, dict(pct=101), PCT_101
            yield name, dict(algo=1), ALGO_1
            yield name, dict(pct=101, algo=1), PCT_101
        if kind(name) == "grain":
            yield name, dict(pct=101), PCT_101
            yield name, dict(shift=11), SHIFT % 11
            yield name, dict(shift=31), SHIFT % 31
            yield name, dict(shift=31, pct=101), SHIFT % 31


@pytest.mark.parametrize("size", [0, 1])
@pytest.mark.parametrize("name,overrides,text", list(content_cases()))
def test_content_argument_rejected_first(native, name, overrides, text, size):
    """reported before anything else, also with nothing to do (len 0, numDescs 0) and with NULL
    pointers"""
    args = Args(len=16 * size, n=size, **overrides)
    assert_rejected(native, name, args, text)


@pytest.mark.parametrize("name", [n for n in SINGLE if n in FILLS])
def test_single_fill_null_device_pointer(native, name):
    assert_rejected(native, name, Args(len=16), name + ": NULL device pointer")


@pytest.mark.parametrize("name", [n for n in SINGLE if n not in FILLS])
def test_single_verify_null_pointers(native, name):
    assert_rejected(native, name, Args(len=16, out=P), name + ": NULL device pointer")
    # the result pointer is checked first, before the length
    assert_rejected(native, name, Args(len=16), name + ": NULL result pointer")
    assert_rejected(native, name, Args(len=0), name + ": NULL result pointer")


@pytest.mark.parametrize("name", BATCH)
def test_batch_null_arrays(native, name):
    if name in FILLS:
        assert_rejected(native, name, Args(n=1), prefix(name) + ": NULL descriptor array")
        assert_rejected(native, name, Args(n=7, results=P),
                        prefix(name) + ": NULL descriptor array")
    else:
        text = prefix(name) + ": NULL descriptor or result array"
        assert_rejected(native, name, Args(n=1, results=P), text)
        assert_rejected(native, name, Args(n=1, descs=P), text)
        assert_rejected(native, name, Args(n=7), text)


@pytest.mark.parametrize("name", [n for n in ENTRY_POINTS if n in FILLS or n in BATCH])
def test_nothing_to_do_returns_0_without_launch(native, name):
    """fills of len 0 (pattern fill before its NULL pointer check) and every form with numDescs 0"""
    assert call(native, name, Args()) == 0
    assert call(native, name, Args(pct=100, shift=30)) == 0


def test_stage_copy_and_results_init(native):
    before = native.elb_num_kernel_launches()
    assert native.elb_stage_copy(N, 0, 1, DELTA, 0, 0, N) == 0
    assert native.elb_stage_copy(N, 1, 1, DELTA, 0, 0, N) == -1
    assert _native.last_error() == "stage_copy: descriptor array and host delta are required"
    assert native.elb_stage_copy(P, 1, 0, 0, 0, 0, N) == -1
    assert _native.last_error() == "stage_copy: descriptor array and host delta are required"
    assert native.elb_verify_results_init(N, 0, N) == 0
    assert native.elb_verify_results_init(N, 1, N) == -1
    assert _native.last_error() == "elb_verify_results_init: NULL result array"
    assert native.elb_num_kernel_launches() == before
