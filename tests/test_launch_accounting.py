"""Every kernel launch in the library's host code goes through launch() in bftq.cu, which checks the launch and counts it in
bftq_stats: a `<<<` anywhere else is a launch that is neither checked nor counted.  bftq_measure_int_peak is the one
exception (a check per launch would sit inside its timed window); it adds its launches to the counter itself."""
import glob
import os
import re

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "bftkv_b200", "csrc")


def _sources():
    files = [os.path.join(CSRC, "bftq.cu"), os.path.join(CSRC, "pgp_digest.cuh")] + sorted(glob.glob(os.path.join(CSRC, "*.inc")))
    assert len(files) >= 7, files
    return files


def _code(path):
    """The file with comments, string and character literals blanked (line numbers kept)."""
    src = open(path).read()
    pat = r'//[^\n]*|/\*.*?\*/|"(?:\\.|[^"\\\n])*"|\'(?:\\.|[^\'\\\n])+\''
    return re.sub(pat, lambda m: '""' if m.group(0)[0] == '"' else "\n" * m.group(0).count("\n"), src, flags=re.S)


def _bodies(src):
    """(name, start, end) of every top-level function body; namespace and extern "C" blocks are looked through."""
    out, depth, head_at, open_at, head = [], 0, 0, 0, ""
    for m in re.finditer(r"[{};]", src):
        c, i = m.group(0), m.start()
        if depth == 0:
            if c == "{":
                head = src[head_at:i]
                if re.search(r'(\bnamespace\b[\w\s:]*|\bextern\s*"")\s*$', head):
                    head_at = i + 1                          # transparent block: its members are top level
                    continue
                depth, open_at = 1, i
            else:                                            # ';' or the '}' closing a transparent block
                head_at = i + 1
        elif c == "{":
            depth += 1
        elif c == "}":
            depth -= 1
            if depth == 0:
                names = [n for n in re.findall(r"(\w+)\s*\(", head) if not n.startswith("__")]
                out.append((names[0] if names else head.strip(), open_at, i))
                head_at = i + 1
    return out


def _enclosing(bodies, pos):
    return next((name for name, a, b in bodies if a < pos < b), None)


def _where(token_re):
    """(file, enclosing function) of every match of token_re in the library's host code."""
    hits = []
    for path in _sources():
        src = _code(path)
        bodies = _bodies(src)
        hits += [(os.path.basename(path), _enclosing(bodies, m.start())) for m in re.finditer(token_re, src)]
    return sorted(hits)


def test_kernels_launch_only_through_the_helper():
    assert _where(r"<<<") == [("bftq.cu", "bftq_measure_int_peak")] * 2 + [("bftq.cu", "launch")]


def test_launches_are_counted_only_by_the_helper():
    assert _where(r"stats\.launches\s*(\+=|\+\+|=)") == [("bftq.cu", "bftq_measure_int_peak"), ("bftq.cu", "launch")]
