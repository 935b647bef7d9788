"""CPU: libkbo's device memory has one owner.  DevBuf (kbo_internal.cuh) frees its allocation when its holder is destroyed,
so no other source allocates or frees device memory itself and no object keeps a hand-written list of buffers to free."""
import glob
import os
import re

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "kubeflow_b200", "csrc")


def _sources():
    paths = sorted(glob.glob(os.path.join(CSRC, "*.cu")) + glob.glob(os.path.join(CSRC, "*.cuh")))
    assert len(paths) >= 10
    return {os.path.basename(p): open(p).read() for p in paths}


def test_device_memory_is_allocated_and_freed_only_by_devbuf():
    hits = {name: sorted(set(re.findall(r"\bcuda(?:Malloc|Free)\b", txt))) for name, txt in _sources().items()}
    assert hits["kbo_internal.cuh"], "kbo_internal.cuh no longer holds DevBuf's cudaMalloc / cudaFree"
    outside = {name: calls for name, calls in hits.items() if calls and name != "kbo_internal.cuh"}
    assert not outside, f"device memory managed outside DevBuf: {outside}"


def test_no_hand_kept_free_lists():
    # `DevBuf* bufs[] = {...}` arrays, and loops over a braced list of buffers (`for (DevBuf* b : {&x, &y})`)
    pat = re.compile(r"DevBuf\s*\*\s*\w+\s*(?:\[\s*\]|:\s*\{)")
    lists = {name: len(pat.findall(txt)) for name, txt in _sources().items()}
    assert not any(lists.values()), f"DevBuf* free lists: { {k: v for k, v in lists.items() if v} }"
