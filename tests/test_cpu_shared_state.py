"""Process-wide state in the library sources.  State has one owner: the calling thread (the error slot), the context (launch record, stage
timer, flag epoch), the device (PerDevice in mf_kernels.h: SM count, occupancies, kernel attributes) or, guarded, the process.  So every
variable declared `static` -- at namespace scope, in a class or inside a function -- is const / constexpr, thread_local, a std::mutex, a
std::once_flag or a PerDevice<...>; the exceptions are the GEMM launcher's tensor-map cache and its driver entry point, both guarded by
g_gemmLock.  A static whose initialiser asks the runtime or the driver (cuda* / cu*) about a device is a PerDevice, since a process may drive
several devices.  The only __device__ globals are the stage clock of the -DMF_TRACK_TIMING build."""
from __future__ import annotations

import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "maskfusion_b200", "csrc")
GUARDED = {"g_mapCache", "g_encode"}                 # under g_gemmLock (mf_cnn.cu)
TIMING_GLOBALS = {"g_trackTiming", "g_trackTimingN"}  # -DMF_TRACK_TIMING only (mf_track.cu)
SYNC_TYPES = ("std::mutex", "std::once_flag")
CUDA_CALL = re.compile(r"\bcu(?:da)?[A-Z]\w*\s*\(")
CLOSE = {"(": ")", "[": "]", "{": "}"}


def _strip(text: str) -> str:
    """comments, string and character literals and preprocessor lines blanked; newlines kept, so offsets keep their line numbers"""
    out, i, n = [], 0, len(text)
    bol = True
    while i < n:
        c = text[i]
        if bol and c == "#" or (bol and c in " \t" and text[i:].lstrip(" \t").startswith("#")):
            while i < n and text[i] != "\n":               # the directive and its continuation lines
                if text[i] == "\\" and i + 1 < n and text[i + 1] == "\n":
                    out.append(" \n"); i += 2
                    continue
                out.append(" "); i += 1
            continue
        bol = False
        if text.startswith("//", i):
            while i < n and text[i] != "\n":
                out.append(" "); i += 1
        elif text.startswith("/*", i):
            j = text.index("*/", i + 2) + 2
            out.append(re.sub(r"[^\n]", " ", text[i:j])); i = j
        elif c in "\"'":
            j = i + 1
            while text[j] != c:
                j += 2 if text[j] == "\\" else 1
            out.append(c + " " * (j - i - 1) + c); i = j + 1
        else:
            out.append(c); i += 1
            bol = c == "\n"
    return "".join(out)


def _match(text: str, i: int) -> int:
    """index after the bracket that closes the one at text[i]"""
    stack = []
    for j in range(i, len(text)):
        if text[j] in CLOSE:
            stack.append(CLOSE[text[j]])
        elif stack and text[j] == stack[-1]:
            stack.pop()
            if not stack:
                return j + 1
    raise ValueError("unbalanced bracket at %d" % i)


def _statement_end(text: str, i: int) -> int:
    """index of the ';' that ends the declaration starting at i (brackets skipped)"""
    while text[i] != ";":
        i = _match(text, i) if text[i] in CLOSE else i + 1
    return i


PARAM = re.compile(r"^\s*(?:[\w:<>]+[\s\*&]+)+[\*&\s]*\w+\s*(?:\[[^\]]*\])?\s*$")


def _is_function(text: str, open_paren: int) -> bool:
    """the declarator's first '(' starts a parameter list: a body follows, or a ';' after a list of `type name` parameters"""
    close = _match(text, open_paren)
    rest = re.match(r"\s*(?:(?:const|noexcept|override)\b\s*)*(.)", text[close:], re.S)
    if rest and rest.group(1) == "{":
        return True
    params = text[open_paren + 1:close - 1].strip()
    return rest is not None and rest.group(1) == ";" and (params in ("", "void") or all(PARAM.match(p) for p in params.split(",")))


def _declarations(text: str, keyword: str):
    """(offset, head, rest) of every variable declared with `keyword`: head is the text up to the first declarator's name included, rest the
    initialiser and any further declarators up to the ';'"""
    for m in re.finditer(r"\b%s\b" % keyword, text):
        stop, angle = m.end(), 0
        while angle or text[stop] not in ";=({[,":          # the end of the first declarator's name; template arguments skipped
            angle += {"<": 1, ">": -1}.get(text[stop], 0)
            stop += 1
        if text[stop] == "(" and _is_function(text, stop):
            continue
        yield m.start(), text[m.end():stop], text[stop:_statement_end(text, stop)]


def _names(head: str, rest: str):
    first = re.findall(r"\w+", head)[-1]
    more, depth, part = [], 0, ""
    for c in rest:                                       # top-level commas separate further declarators
        depth += c in "([{"
        depth -= c in ")]}"
        if c == "," and depth == 0:
            more.append(part); part = ""
        else:
            part += c
    more.append(part)
    return [first] + [re.match(r"\s*[\*&\s]*(\w+)", p).group(1) for p in more[1:] if re.match(r"\s*[\*&\s]*(\w+)", p)]


def _allowed(head: str, name: str) -> bool:
    t = head[:head.rfind(name)] if name in head else head
    if name in GUARDED or "thread_local" in t or "constexpr" in t or t.strip().startswith("PerDevice<"):
        return True
    if any(re.search(r"(?:^|\s)%s\b" % re.escape(s), t) for s in SYNC_TYPES):
        return True
    if "*" in t:                                          # the pointer itself must be const, not only what it points to
        return bool(re.search(r"\*\s*const\b[^\*]*$", t))
    return bool(re.search(r"\bconst\b", t))


def _line(text: str, off: int) -> int:
    return text.count("\n", 0, off) + 1


def _scan():
    bad = []
    for f in sorted(os.listdir(CSRC)):
        text = _strip(open(os.path.join(CSRC, f)).read())
        for off, head, rest in _declarations(text, "static"):
            names = _names(head, rest)
            where = "%s:%d: static %s" % (f, _line(text, off), ", ".join(names))
            if not all(_allowed(head, n) for n in names):
                bad.append(where + " is shared mutable state (make it const, thread_local, a std::mutex / std::once_flag or a PerDevice)")
            elif CUDA_CALL.search(rest) and not head.strip().startswith("PerDevice<"):
                bad.append(where + " is computed from the device first met (%s...): make it a PerDevice" % CUDA_CALL.search(rest).group(0))
        for off, head, rest in _declarations(text, "__device__"):
            name = re.findall(r"\w+", head)[-1]
            if name not in TIMING_GLOBALS:
                bad.append("%s:%d: __device__ global %s" % (f, _line(text, off), name))
    return bad


def test_no_unguarded_process_wide_state():
    bad = _scan()
    assert not bad, "process-wide state without an owner:\n" + "\n".join(bad)


def test_the_scan_sees_what_it_checks():
    """the parser finds the declarations it is meant to judge: the allowed statics, PerDevice users and the two timing globals"""
    seen, per_device = set(), 0
    for f in sorted(os.listdir(CSRC)):
        text = _strip(open(os.path.join(CSRC, f)).read())
        for _, head, rest in _declarations(text, "static"):
            seen.update(_names(head, rest))
            per_device += head.strip().startswith("PerDevice<")
        for _, head, _ in _declarations(text, "__device__"):
            seen.add(re.findall(r"\w+", head)[-1])
    assert {"g_err", "g_gemmLock", "g_mapCache", "g_encode", "HANDLE_NAME", "sig"} | TIMING_GLOBALS <= seen, seen
    assert per_device >= 4, per_device
    assert not {"identity", "pickOwner", "mf_finalise", "grid2", "ok"} & seen      # functions are not variables
