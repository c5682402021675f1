"""Static checks on the CUDA sources for the properties the stream tests (test_streams_gpu.py) rely on, including in code those
tests do not reach: every kernel launch names the caller's stream, no call takes the synchronous stream-less form of a copy,
a fill or a device synchronise, and no index struct has a member that a const (read-only) path could write."""
import glob
import os
import re

import pytest

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "cuvs_b200", "csrc")


def _sources():
    paths = sorted(glob.glob(os.path.join(CSRC, "*.cu")) + glob.glob(os.path.join(CSRC, "*.cuh")) +
                   glob.glob(os.path.join(CSRC, "*.hpp")))
    assert paths, "no CUDA sources found under cuvs_b200/csrc"
    return paths


def _strip_comments(text):
    """Blank out comments and string literals, keeping newlines so line numbers survive."""
    out = re.sub(r"//[^\n]*|/\*.*?\*/|\"(?:\\.|[^\"\\\n])*\"",
                 lambda m: re.sub(r"[^\n]", " ", m.group(0)), text, flags=re.S)
    return out


def _code(path):
    with open(path) as f:
        return _strip_comments(f.read())


def _drop_templates(s):
    """Remove template argument lists (`name<...>`) so their commas do not split arguments; innermost first."""
    prev = None
    while prev != s:
        prev = s
        s = re.sub(r"(\w)\s*<[^<>;(){}]*>", r"\1", s)
    return s


def launch_args(config):
    """Top-level arguments of a launch configuration (the text between <<< and >>>)."""
    s = _drop_templates(config)
    args, depth, cur = [], 0, []
    for ch in s:
        if ch in "([{":
            depth += 1
        elif ch in ")]}":
            depth -= 1
        if ch == "," and depth == 0:
            args.append("".join(cur).strip())
            cur = []
        else:
            cur.append(ch)
    args.append("".join(cur).strip())
    return [a for a in args if a]


def launches(text):
    """(line, config) of every <<<...>>> launch, including launches written across several lines."""
    out = []
    for m in re.finditer(r"<<<(.*?)>>>", text, flags=re.S):
        out.append((text.count("\n", 0, m.start()) + 1, m.group(1)))
    return out


def test_launch_parser():
    assert launch_args("blocks_for(n, 256), 256, 0, s") == ["blocks_for(n, 256)", "256", "0", "s"]
    assert len(launch_args("std::min<int64_t>(1024, (n + 127) / 128), 128, 0, res->stream")) == 4
    assert len(launch_args("dim3(a, b), 128, smem,\n   s")) == 4
    assert len(launch_args("static_cast<unsigned>(grid), kThreads, std::max<size_t>(a, b)")) == 3
    assert len(launch_args("g, 128")) == 2
    text = "k<<<dim3(x,\n y), 64>>>(a);\nk2<<<std::min<int>(1, 2), 32, 0,\n s>>>(b);"
    found = launches(text)
    assert [ln for ln, _ in found] == [1, 3]
    assert [len(launch_args(c)) for _, c in found] == [2, 4]


def test_every_launch_names_a_stream():
    bad, n = [], 0
    for p in _sources():
        for line, config in launches(_code(p)):
            n += 1
            args = launch_args(config)
            if len(args) != 4:
                bad.append("%s:%d: <<<%s>>>" % (os.path.basename(p), line, " ".join(config.split())))
    assert n > 100, "found only %d launches: the launch pattern no longer matches the sources" % n
    assert not bad, "kernel launches without a stream argument:\n" + "\n".join(bad)


@pytest.mark.parametrize("pattern", [r"\bcudaMemcpy\s*\(", r"\bcudaMemcpy2D\s*\(", r"\bcudaMemset\s*\(", r"\bcudaMemset2D\s*\(",
                                     r"\bcudaDeviceSynchronize\b"])
def test_no_streamless_copy_fill_or_device_sync(pattern):
    bad = []
    for p in _sources():
        text = _code(p)
        for m in re.finditer(pattern, text):
            bad.append("%s:%d" % (os.path.basename(p), text.count("\n", 0, m.start()) + 1))
    assert not bad, "stream-less %s at:\n%s" % (pattern, "\n".join(bad))


def test_no_mutable_members():
    """A `mutable` member lets a path that takes an index as const (search, getters, serialisation) change it, which breaks
    concurrent readers of one index (DESIGN.md "Streams and concurrent callers")."""
    bad = []
    for p in _sources():
        text = _code(p)
        for m in re.finditer(r"\bmutable\b", text):
            before = text[max(0, m.start() - 200):m.start()].rstrip()
            if before.endswith(")"):  # a mutable lambda: `[...](...) mutable {`
                continue
            bad.append("%s:%d" % (os.path.basename(p), text.count("\n", 0, m.start()) + 1))
    assert not bad, "mutable members at:\n" + "\n".join(bad)
