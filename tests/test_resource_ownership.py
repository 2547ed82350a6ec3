"""CPU: device memory, pinned host memory, events and streams in conflux_b200/csrc are owned.  Only the owning types of
common.cuh allocate or release them, so every buffer, event and stream is freed by the destructor of the scope or the
object that holds it, on every return path.  The one exception is cflx_host_alloc / cflx_host_free: that memory belongs
to the caller."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "conflux_b200", "csrc")
RAW = re.compile(r"\b(cudaMalloc|cudaMallocHost|cudaHostAlloc|cudaFree|cudaFreeHost|cudaEventDestroy|cudaStreamDestroy)\b")
CALLER_OWNED = ("cflx_host_alloc", "cflx_host_free")


def _strip_comments(text):
    text = re.sub(r"/\*.*?\*/", lambda m: "\n" * m.group(0).count("\n"), text, flags=re.S)
    return re.sub(r"//[^\n]*", "", text)


def _without_function(text, name):
    """text with the body of the function `name` blanked (lines kept, so reported line numbers stay right)"""
    m = re.search(r"\b%s\s*\([^)]*\)\s*\{" % name, text)
    if not m:
        return text
    depth, i = 1, m.end()
    while depth:
        depth += {"{": 1, "}": -1}.get(text[i], 0)
        i += 1
    return text[:m.start()] + re.sub(r"[^\n]", " ", text[m.start():i]) + text[i:]


def raw_sites(csrc=CSRC):
    sites = []
    for name in sorted(os.listdir(csrc)):
        if not name.endswith((".cu", ".cuh", ".h", ".inc")) or name == "common.cuh":
            continue
        text = _strip_comments(open(os.path.join(csrc, name)).read())
        for fn in CALLER_OWNED:
            text = _without_function(text, fn)
        for m in RAW.finditer(text):
            sites.append(f"{name}:{text.count(chr(10), 0, m.start()) + 1}: {m.group(1)}")
    return sites


def test_only_owning_types_allocate_and_release():
    sites = raw_sites()
    assert not sites, f"{len(sites)} raw allocation / release calls outside common.cuh:\n" + "\n".join(sites)

