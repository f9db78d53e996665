"""Every device allocation of the library has one owner: cudaMalloc and cudaFree are called only inside DeviceBuffer
(csrc/common.cuh), whose destructor frees what the model and front-end handles hold."""
import glob
import os
import re

from helpers import ROOT

CSRC = os.path.join(ROOT, "attention-lvcsr_b200", "csrc")
CALL = re.compile(r"\bcuda(Malloc|Free)\s*(?:<[^<>;(){}]*>\s*)?\(")     # cudaMalloc(...) and cudaMalloc<T>(...)


def _code(path):
    """The file's text with comments and string / character literals blanked (line breaks kept)."""
    text = open(path).read()
    token = re.compile(r'//[^\n]*|/\*.*?\*/|"(?:\\.|[^"\\\n])*"|\'(?:\\.|[^\'\\\n])*\'', re.S)
    return token.sub(lambda t: re.sub(r"[^\n]", " ", t.group(0)), text)


def _class_span(code, name):
    """[start, end) of the body of `class name` in code, braces matched."""
    head = re.search(r"\bclass\s+%s\b[^;{]*\{" % name, code)
    assert head, "no class %s" % name
    depth, i = 1, head.end()
    while depth:
        depth += {"{": 1, "}": -1}.get(code[i], 0)
        i += 1
    return head.start(), i


def test_cuda_malloc_and_free_only_inside_the_owner_type():
    sources = sorted(glob.glob(os.path.join(CSRC, "*.cu")) + glob.glob(os.path.join(CSRC, "*.cuh")) +
                     glob.glob(os.path.join(CSRC, "*.h")))
    assert len(sources) > 10
    owner = os.path.join(CSRC, "common.cuh")
    span = _class_span(_code(owner), "DeviceBuffer")
    outside, inside = [], {"Malloc": 0, "Free": 0}
    for path in sources:
        code = _code(path)
        for call in CALL.finditer(code):
            if path == owner and span[0] <= call.start() < span[1]:
                inside[call.group(1)] += 1
            else:
                line = code.count("\n", 0, call.start()) + 1
                outside.append("%s:%d: cuda%s(" % (os.path.basename(path), line, call.group(1)))
    assert not outside, "device memory allocated or freed outside DeviceBuffer:\n" + "\n".join(outside)
    assert inside == {"Malloc": 1, "Free": 1}, inside
