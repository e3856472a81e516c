"""Every CUDA resource an engine holds has one owner in islplace.cu: DevMem, HostMem or Handle (streams, events, peer mappings).  Only
those types allocate or release, so deleting an engine frees everything it holds and no entry point can leak or double-free a
buffer, stream, event or IPC mapping.  These checks read the source; they need no GPU."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "instaslice_b200", "csrc", "islplace.cu")

CALLS = ("cudaMalloc", "cudaHostAlloc", "cudaFree", "cudaFreeHost", "cudaIpcCloseMemHandle", "cudaStreamDestroy", "cudaEventDestroy")
# pinned memory allocated for and owned by the caller (the ABI's pinned-buffer helpers), not by an engine
CALLER_OWNED = ("isl_host_alloc", "isl_host_free")


def _code():
    text = open(SRC).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return re.sub(r"//[^\n]*", "", text)


def _split(code):
    """(the owner types, everything else): the owners run from `enum class Growth` to the engine struct."""
    start, end = code.find("enum class Growth"), code.index("struct isl_engine {")
    if start < 0:
        return "", code
    return code[start:end], code[:start] + code[end:]


def _body(code, name):
    """The brace-delimited body of the function definition `name(...) {`."""
    m = re.search(r"\b%s\([^;{]*\)\s*\{" % re.escape(name), code)
    assert m, name
    depth, i = 0, m.end() - 1
    while True:
        depth += {"{": 1, "}": -1}.get(code[i], 0)
        i += 1
        if depth == 0:
            return code[m.start():i]


def _uses(code, call):
    return len(re.findall(r"\b%s\s*\(" % call, code)) + len(re.findall(r"[<,]\s*%s\s*>" % call, code))


def test_only_the_owner_types_allocate_and_release():
    owners, rest = _split(_code())
    for name in CALLER_OWNED:
        rest = rest.replace(_body(rest, name), "")
    for call in CALLS:
        assert _uses(rest, call) == 0, f"{call} outside the owner types"
        assert _uses(owners, call) > 0, call


def test_streams_are_declared_before_the_memory_they_outlive():
    """Members are destroyed in reverse order: the stream and event owners come first, so every buffer is freed before them."""
    code = _code()
    struct = code[code.index("struct isl_engine {"):]
    members = re.findall(r"^\s*(DevMem|HostMem|PeerMap|Stream|Event)\b", struct[:struct.index("\n};")], flags=re.M)
    n_streams = sum(m in ("Stream", "Event") for m in members)
    assert n_streams >= 2 and all(m in ("Stream", "Event") for m in members[:n_streams]), members


def test_destroy_and_failed_create_free_through_the_members():
    code = _code()
    destroy, create = _body(code, "isl_destroy"), _body(code, "isl_create")
    assert "delete e;" in destroy and "isl_destroy" not in create and "delete e;" in create
    assert destroy.index("DeviceGuard") < destroy.index("delete e;")       # the engine's device is current while its members release
