"""The worker, the manager, the stats reduce and the cuFile binding put nothing on the legacy
default stream (DESIGN.md §3): the library shares the primary context with the application, and
PyTorch's default stream is the legacy stream, so a copy, memset or launch queued there waits for
whatever the caller left on it, while the batch kernels on their non-blocking streams do not.
tests/test_default_stream_gpu.py shows what that breaks; this scan is the only guard for the
set-up calls, whose order no GPU test can pin down."""
import os
import re

import pytest

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "elbencho_b200",
                    "csrc")
SOURCES = ["elb_worker.cpp", "elb_manager.cpp", "elb_statsreduce.cu", "elb_cufile.cpp"]

# calls that take a stream -> position of the stream argument (the runtime's C++ declarations
# default an omitted stream to 0, so a short argument list is the legacy stream as well)
STREAM_CALLS = {
    "cudaMemcpyAsync": 4,
    "cudaMemsetAsync": 3,
    "cudaMemcpy2DAsync": 7,
    "cudaMemcpyToSymbolAsync": 5,
    "cudaMemcpyFromSymbolAsync": 5,
    "cudaEventRecord": 1,
    "cudaEventRecordWithFlags": 1,
    "cudaGraphLaunch": 1,
    "cudaStreamSynchronize": 0,
    "cudaStreamQuery": 0,
    "cudaStreamWaitEvent": 0,
    "cudaStreamBeginCapture": 0,
    "cudaStreamEndCapture": 0,
    "cudaLaunchKernel": 5,
}
LEGACY_STREAMS = {"0", "NULL", "nullptr", "cudaStreamLegacy", "(cudaStream_t)0",
                  "(cudaStream_t)NULL"}


def strip_comments_and_strings(text):
    """C/C++ source with comments and string / character literals blanked out (newlines kept, so
    that line numbers stay right)"""
    out = []
    i, n = 0, len(text)
    while i < n:
        c = text[i]
        if text.startswith("//", i):
            j = text.find("\n", i)
            i = n if j < 0 else j
        elif text.startswith("/*", i):
            j = text.find("*/", i + 2)
            j = n if j < 0 else j + 2
            out.append("\n" * text.count("\n", i, j))
            i = j
        elif c in "\"'":
            j = i + 1
            while j < n and text[j] != c:
                j += 2 if text[j] == "\\" else 1
            out.append(c + c)
            i = j + 1
        else:
            out.append(c)
            i += 1
    return "".join(out)


def split_top(text):
    """"a, f(b, c), d[1]" -> ["a", "f(b, c)", "d[1]"]; "" -> []"""
    args, depth, cur = [], 0, ""
    for c in text:
        depth += (c in "([{") - (c in ")]}")
        if c == "," and not depth:
            args.append(cur.strip())
            cur = ""
        else:
            cur += c
    return args + [cur.strip()] if (args or cur.strip()) else []


def call_args(text, open_pos):
    """text[open_pos] == "(": the top-level arguments of that call"""
    depth = 0
    for i in range(open_pos, len(text)):
        depth += (text[i] == "(") - (text[i] == ")")
        if not depth:
            return split_top(text[open_pos + 1:i])
    raise ValueError("unbalanced call at offset %d" % open_pos)


def legacy_stream_uses(source):
    """-> list of (line number, what) for every use of the legacy default stream in source"""
    text = strip_comments_and_strings(source)
    found = []

    def line_of(pos):
        return text.count("\n", 0, pos) + 1

    for m in re.finditer(r"\b(cudaMem(?:cpy|set)\w*)\s*\(", text):
        if not m.group(1).endswith("Async"):
            found.append((line_of(m.start()), m.group(1) + " (synchronous: legacy stream)"))
    for m in re.finditer(r"\bcudaDeviceSynchronize\s*\(", text):
        found.append((line_of(m.start()), "cudaDeviceSynchronize"))
    for m in re.finditer(r"\b(cuda\w+)\s*\(", text):
        name = m.group(1)
        if name not in STREAM_CALLS:
            if name.endswith("Async"):
                found.append((line_of(m.start()), name + " (stream position unknown to this test)"))
            continue
        args = call_args(text, m.end() - 1)
        pos = STREAM_CALLS[name]
        if len(args) <= pos:
            found.append((line_of(m.start()), name + " without a stream"))
        elif args[pos].replace(" ", "") in LEGACY_STREAMS:
            found.append((line_of(m.start()), name + " on stream " + args[pos]))
    for m in re.finditer(r"<<<", text):
        config = split_top(text[m.end():text.find(">>>", m.end())])
        if len(config) < 4:
            found.append((line_of(m.start()), "kernel launch without a stream"))
        elif config[3].replace(" ", "") in LEGACY_STREAMS:
            found.append((line_of(m.start()), "kernel launch on stream " + config[3]))
    return sorted(found)


@pytest.mark.parametrize("name", SOURCES)
def test_source_uses_no_legacy_default_stream(name):
    with open(os.path.join(CSRC, name)) as f:
        source = f.read()
    assert legacy_stream_uses(source) == [], name


@pytest.mark.parametrize("snippet", [
    "cudaMemset(p, 0, n);",
    "cudaMemcpy(dst, src, n, cudaMemcpyDeviceToHost);",
    "ok = ok && (cudaMemcpy2D(d, 1, s, 1, 1, 1, k) == cudaSuccess);",
    "cudaMemcpyToSymbol(sym, src, n);",
    "cudaMemcpyAsync(dst, src, n, kind);",
    "cudaMemcpyAsync(dst, src, n, kind, 0);",
    "cudaMemsetAsync(p, 0, sizeof(uint64_t) * (n + 1), NULL);",
    "cudaMemsetAsync(p, 0, f(a, b));",
    "cudaMemcpyAsync(dst, src, n, kind, cudaStreamLegacy);",
    "cudaMemPrefetchAsync(p, n, dev, s);",
    "cudaEventRecord(ev);",
    "cudaEventRecord(ev, 0);",
    "cudaStreamSynchronize(0);",
    "cudaGraphLaunch(exec, nullptr);",
    "k<<<grid, block>>>(args);",
    "k<<<grid, block, 0>>>(args);",
    "k<<<grid, block, 0, 0>>>(args);",
    "cudaDeviceSynchronize();",
])
def test_scan_finds_legacy_stream_uses(snippet):
    """the scan above is only a guard if it sees every form of a legacy stream use"""
    assert len(legacy_stream_uses("void f()\n{\n\t" + snippet + "\n}\n")) == 1, snippet


@pytest.mark.parametrize("snippet", [
    "cudaMemcpyAsync(dst, src, n, kind, batch.stream);",
    "cudaMemsetAsync(p, 0, sizeof(uint64_t) * (n + 1), gpus[0].stream);",
    "cudaEventRecord(batch.gpuDoneEvent, batch.stream);",
    "cudaStreamSynchronize(auxStream);",
    "k<<<(n + 255) / 256, 256, 0, stream>>>(args);",
    "// cudaMemcpy(dst, src, n, kind) in a comment",
    "/* cudaMemset(p, 0, n);\n   cudaDeviceSynchronize(); */",
    'throw Error("cudaMemcpy(x) failed");',
    "cudaMemcpyKind kind = cudaMemcpyHostToDevice;",
])
def test_scan_accepts_explicit_streams_comments_and_strings(snippet):
    assert legacy_stream_uses("void f()\n{\n\t" + snippet + "\n}\n") == [], snippet
