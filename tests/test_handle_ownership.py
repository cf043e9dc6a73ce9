"""Every device buffer, stream and event of a handle has one owner: dhqr_api.cu allocates, frees, creates streams and destroys
streams and events only inside its owner types, so dhqr_destroy has nothing left to free by hand and no free can be forgotten."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "distributedhouseholderqr.jl_b200", "csrc", "dhqr_api.cu")
OWNERS = ("DevBuf", "Owned", "Stream", "Event")
CALLS = re.compile(r"\bcuda(?:Malloc\w*|Free\w*|StreamCreate\w*|StreamDestroy|EventDestroy)\b")


def _code():
    """The source with comments and string literals blanked out (same length, so offsets stay valid)."""
    src = open(SRC).read()
    blank = lambda m: re.sub(r"[^\n]", " ", m.group(0))
    return re.sub(r'//[^\n]*|/\*.*?\*/|"(?:\\.|[^"\\\n])*"', blank, src, flags=re.S)


def _body(code, head):
    """[start, end) of the definition that starts at `head` (a regex), from its first character to its closing brace."""
    m = re.search(head, code)
    assert m, f"no definition matches {head!r}"
    depth, i = 0, code.index("{", m.start())
    while True:
        depth += {"{": 1, "}": -1}.get(code[i], 0)
        i += 1
        if depth == 0:
            return m.start(), i


def test_resources_are_acquired_and_released_only_by_their_owners():
    code = _code()
    spans = [_body(code, r"\bstruct\s+%s\b[^;{]*\{" % name) for name in OWNERS]
    stray = []
    for m in CALLS.finditer(code):
        if not any(a <= m.start() < b for a, b in spans):
            stray.append(f"line {code.count(chr(10), 0, m.start()) + 1}: {m.group(0)}")
    assert not stray, "outside the owner types: " + ", ".join(stray)


def test_destroy_frees_nothing_by_hand():
    code = _code()
    a, b = _body(code, r"\bint\s+dhqr_destroy\s*\(")
    body = code[a:b]
    assert not CALLS.findall(body), CALLS.findall(body)
    assert "delete c;" in body
