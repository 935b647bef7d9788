"""CPU: every libkbo device buffer states its element type once, in its declaration (DevBuf<T>, kbo_internal.cuh).  Call sites
use the typed pointer as it is, and reservations and uploads count elements, so a buffer cannot be sized in one unit and read
in another without the compiler seeing it."""
import glob
import os
import re

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "kubeflow_b200", "csrc")


def _sources():
    paths = sorted(glob.glob(os.path.join(CSRC, "*.cu")) + glob.glob(os.path.join(CSRC, "*.cuh")))
    assert len(paths) >= 10
    return {os.path.basename(p): open(p).read() for p in paths}


def _lines(txt, pat):
    return [f"{i + 1}: {line.strip()}" for i, line in enumerate(txt.splitlines()) if pat.search(line)]


def _call_args(txt, fn):
    """The argument lists of every call of fn in txt, split at top-level commas."""
    out = []
    for m in re.finditer(rf"\b{fn}\s*\(", txt):
        depth, start, args = 0, m.end(), []
        for j in range(m.end() - 1, len(txt)):
            c = txt[j]
            if c in "([{":
                depth += 1
            elif c in ")]}":
                depth -= 1
                if depth == 0:
                    args.append(txt[start:j].strip())
                    break
            elif c == "," and depth == 1:
                args.append(txt[start:j].strip())
                start = j + 1
        out.append(args)
    return out


# (double*)c->B.p, (const int*)f->cols.p, (char*)e->dev.p, (float*)(h->mun.p) ...
CAST = re.compile(r"\(\s*(?:const\s+)?[A-Za-z_][\w:]*(?:\s+[A-Za-z_]\w*)*\s*\*+\s*\)\s*\(?\s*[A-Za-z_]\w*(?:(?:->|\.)\w+|\[[^\]]*\])*\.p\b")


def test_cast_pattern_matches_buffer_casts():
    for sample in ("(double*)c->B.p", "(const double*)c->B.p + D", "(int*)f->cols.p", "(const unsigned char*)f->blob.p",
                   "(char*)e->dev.p + offsetof(EnDev, err)", "(float*)(h->mun.p)", "(const __half*)h->rk_sched[i].dev.p", "(void*)X.p"):
        assert CAST.search(sample), sample
    for sample in ("c->B.p + D", "kbo_view<float>(h->mun)", "(size_t)n * D", "(unsigned)((n + 255) / 256)"):
        assert not CAST.search(sample), sample


def test_no_casts_of_buffer_pointers():
    # kbo_internal.cuh is where a byte buffer is viewed as another type; reqparse.cu's .p are host byte spans, not buffers
    hits = {name: _lines(txt, CAST) for name, txt in _sources().items() if name not in ("kbo_internal.cuh", "reqparse.cu")}
    hits = {k: v for k, v in hits.items() if v}
    assert not hits, f"casts of a DevBuf's .p (declare the buffer with its element type instead): {hits}"


def test_reservations_and_uploads_count_elements():
    # kbo_internal.cuh defines both and is the one place that turns elements into bytes
    bad = {}
    for name, txt in _sources().items():
        if name == "kbo_internal.cuh":
            continue
        for fn, k in (("kbo_reserve", 2), ("kbo_upload", 3)):
            for args in _call_args(txt, fn):
                size = args[k]
                if "sizeof(" in size or re.match(r"(?:\(\s*size_t\s*\)\s*)?(?:2|4|8|16)\s*\*", size):
                    bad.setdefault(name, []).append(f"{fn}({', '.join(args)})")
    assert not bad, f"reservation sizes given in bytes rather than elements: {bad}"


def test_every_devbuf_has_an_element_type():
    # a DevBuf named as a type (field, local, parameter or pointer) without <T>
    pat = re.compile(r"\bDevBuf\b(?!\s*<)(?!\s*\()")
    hits = {}
    for name, txt in _sources().items():
        # inside its own definition the template names itself without arguments
        txt = re.sub(r"struct DevBuf \{.*?\n\};", "", txt, flags=re.S)
        for i, line in enumerate(txt.splitlines()):
            if pat.search(line.split("//")[0]):
                hits.setdefault(name, []).append(line.strip())
    assert not hits, f"DevBuf without an element type: {hits}"
