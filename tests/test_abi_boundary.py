"""Every C entry point returns a psfm_status and never throws: its body runs inside psfm::guard (csrc/psfm_common.cuh),
the one place of the library that catches, and a host exception such as an out-of-memory std::bad_alloc becomes
PSFM_ERR_HOST with a message instead of terminating the process."""
import glob
import os
import re
import subprocess
import sys

from particlesfm_b200 import _abi, _lib

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "particle-sfm_b200", "csrc")

# entry points whose bodies call nothing that can throw
NOTHROW = {"psfm_last_error", "psfm_abi_version", "psfm_device_count", "psfm_launch_count", "psfm_dist_world_size",
           "psfm_dist_rank", "psfm_seg_max_window", "psfm_track_npy_data", "psfm_dist_finalize",
           "psfm_ba_global_options", "psfm_ba_default_refine_options"}


def _nothrow(name):
    return name in NOTHROW or name.endswith(("_default_options", "_destroy"))


def _strip(src):
    """src with its comments blanked and its string and character literals emptied"""
    def empty(m):
        t = m.group(0)
        return 2 * t[0] if t[0] in "\"'" else " "
    return re.sub(r'//[^\n]*|/\*.*?\*/|"(?:\\.|[^"\\\n])*"|\'(?:\\.|[^\'\\\n])*\'', empty, src, flags=re.S)


def _entry_points():
    """(file, name, body) of every extern "C" function defined in csrc/*.cu, comments and literals stripped."""
    found = []
    for path in sorted(glob.glob(os.path.join(CSRC, "*.cu"))):
        src = _strip(open(path).read())
        for m in re.finditer(r'extern\s+""\s+[^;{(]*?\b(psfm_\w+)\s*\(', src):
            depth = 1
            j = m.end()
            while depth:                                  # the parameter list's closing parenthesis
                depth += {"(": 1, ")": -1}.get(src[j], 0)
                j += 1
            k = j
            while src[k].isspace():
                k += 1
            if src[k] != "{":                             # a declaration
                continue
            depth, e = 1, k + 1
            while depth:
                depth += {"{": 1, "}": -1}.get(src[e], 0)
                e += 1
            found.append((os.path.basename(path), m.group(1), src[k + 1:e - 1]))
    return found


def _top_level(text):
    """text without the contents of its nested braces"""
    out, depth = [], 0
    for ch in text:
        if ch == "{":
            depth += 1
        elif ch == "}":
            depth -= 1
        elif depth == 0:
            out.append(ch)
    return "".join(out)


def test_only_the_guard_catches():
    offenders = []
    for path in sorted(glob.glob(os.path.join(CSRC, "*"))):
        name = os.path.basename(path)
        if name in ("psfm_common.cuh", "bindings.cc") or not name.endswith((".cu", ".cuh", ".h")):
            continue                                      # bindings.cc is the pybind11 module, not the C ABI
        if re.search(r"\bcatch\s*\(", _strip(open(path).read())):
            offenders.append(name)
    assert offenders == []


def test_every_entry_point_is_one_guard():
    entries = _entry_points()
    assert len(entries) > 100, "the parser found too few extern \"C\" definitions"
    bad = []
    for fname, name, body in entries:
        if _nothrow(name):
            continue
        m = re.search(r"\breturn\s+(?:psfm::)?guard\(", body)
        # straight-line set-up may precede the guard (the hooks' state); every exit is the guard's return
        prefix, rest = (body[:m.start()], body[m.start():]) if m else (body, "")
        if not m or re.search(r"\b(return|if|for|while|do|switch|try|throw|goto)\b", _top_level(prefix)) \
                or not _top_level(rest).rstrip().endswith(");") or _top_level(rest).count(";") != 1:
            bad.append("%s: %s" % (fname, name))
    assert bad == []


def test_every_guard_names_its_entry_point():
    bad = []
    for path in sorted(glob.glob(os.path.join(CSRC, "*.cu"))):
        src = re.sub(r"//[^\n]*", "", open(path).read())
        for m in re.finditer(r'extern "C" [^;{(]*?\b(psfm_\w+)\s*\(', src):
            name = m.group(1)
            nxt = src.find('extern "C"', m.end())
            chunk = src[m.end():nxt if nxt > 0 else len(src)]
            g = re.search(r'\breturn\s+(?:psfm::)?guard\((entry|"\w+")', chunk)
            if not g:
                continue
            arg = g.group(1)
            if arg == "entry":
                d = re.search(r'const char\* entry = "(\w+)";', chunk[:g.start()])
                arg = '"%s"' % d.group(1) if d else None
            if arg != '"%s"' % name:
                bad.append(name)
    assert bad == []


def test_nothrow_list_is_current():
    entries = _entry_points()
    names = {name for _, name, _ in entries}
    unguarded = {name for _, name, body in entries if not re.search(r"\bguard\(", body)}
    assert NOTHROW <= names
    assert unguarded == {n for n in names if _nothrow(n)}


# A child that loads only the library: a 1 GiB output buffer is mapped but never touched, the address space is capped
# 256 MB above the child's size, and psfm_seg_shuffle's 1 GiB host vector cannot be allocated.
_CHILD = r"""
import ctypes as C, mmap, os, resource, sys
L = C.CDLL(sys.argv[1])
L.psfm_last_error.restype = C.c_char_p
K = 1 << 28
buf = mmap.mmap(-1, 4 * K)
addr = C.addressof(C.c_char.from_buffer(buf))
size = int(open("/proc/self/statm").read().split()[0]) * os.sysconf("SC_PAGE_SIZE")
resource.setrlimit(resource.RLIMIT_AS, (size + (256 << 20), resource.getrlimit(resource.RLIMIT_AS)[1]))
rc = L.psfm_seg_shuffle(C.c_int32(K), C.c_void_p(addr))
print(rc, L.psfm_last_error().decode())
"""


def test_host_out_of_memory_is_a_status():
    r = subprocess.run([sys.executable, "-c", _CHILD, _lib.LIB_PATH], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, (r.returncode, r.stderr)
    assert r.stdout.strip() == "%d psfm_seg_shuffle: out of host memory" % _abi.PSFM_ERR_HOST
