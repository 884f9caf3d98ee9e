"""Every device allocation of the library has one owner type, DevArray (nucliadb_b200/csrc/api.cu), which frees what it holds when it
is destroyed.  A segment member or a temporary that is a raw owning pointer would need a hand-written free on every path, error
paths included; so cudaMalloc* / cudaFree* may appear in the sources only inside DevArray's definition."""
import os
import re

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "nucliadb_b200", "csrc")
CALL = re.compile(r"\bcuda(?:Malloc|Free)\w*")


def _code(path):
    """The source without its comments (line numbers kept)."""
    with open(path) as f:
        text = f.read()
    text = re.sub(r"/\*.*?\*/", lambda m: "\n" * m.group(0).count("\n"), text, flags=re.S)
    return re.sub(r"//[^\n]*", "", text)


def _owner_span(text):
    """[begin, end] character offsets of `struct DevArray { ... }`, or None."""
    m = re.search(r"\bstruct DevArray\s*\{", text)
    if not m:
        return None
    depth = 0
    for i in range(m.end() - 1, len(text)):
        depth += {"{": 1, "}": -1}.get(text[i], 0)
        if depth == 0:
            return m.start(), i
    raise AssertionError("unbalanced braces in DevArray")


def test_device_memory_is_allocated_and_freed_only_by_its_owner_type():
    owners, stray = 0, []
    for name in sorted(os.listdir(CSRC)):
        if not name.endswith((".cu", ".cuh", ".hpp", ".h", ".cpp")):
            continue
        text = _code(os.path.join(CSRC, name))
        span = _owner_span(text)
        owners += span is not None
        for m in CALL.finditer(text):
            if span is None or not span[0] <= m.start() <= span[1]:
                stray.append(f"{name}:{text.count(chr(10), 0, m.start()) + 1}: {m.group(0)}")
    assert not stray, "device memory allocated or freed outside DevArray:\n" + "\n".join(stray)
    assert owners == 1, f"DevArray is defined {owners} times"
