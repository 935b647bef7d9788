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


# `DevBuf* bufs[] = {...}` arrays, and loops over a braced list of buffers (`for (DevBuf* b : {&x, &y})`), with or without
# the element type (`DevBuf<double>* bufs[]`)
FREE_LIST = re.compile(r"DevBuf\s*(?:<[^<>;]*(?:<[^<>;]*>[^<>;]*)*>)?\s*\*\s*\w+\s*(?:\[\s*\]|:\s*\{)")


def test_free_list_pattern_matches_typed_and_untyped_lists():
    for sample in ("DevBuf* bufs[] = {&a, &b};", "DevBuf<double>* bufs[] = {&a, &b};", "DevBuf < unsigned char > *bufs[] = {&a};",
                   "for (DevBuf* b : {&x, &y})", "for (DevBuf<int>* b : {&x, &y})", "DevBuf<std::pair<int, int>>* bufs[] = {&a};"):
        assert FREE_LIST.search(sample), sample
    for sample in ("DevBuf<double> a, b;", "DevBuf<double>& b", "template <class T> static int kbo_reserve(kbo_handle* h, DevBuf<T>& b, size_t n)"):
        assert not FREE_LIST.search(sample), sample


def test_no_hand_kept_free_lists():
    lists = {name: len(FREE_LIST.findall(txt)) for name, txt in _sources().items()}
    assert not any(lists.values()), f"DevBuf* free lists: { {k: v for k, v in lists.items() if v} }"
