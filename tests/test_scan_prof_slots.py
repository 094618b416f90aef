"""The clock64 slots of the instrumented prefilter scan (the TS_PROF_* enum of csrc/tensor_scan.cu, read through
cdb_debug_scan_profile) and the copy of that list in tools/bench_prefilter_resident.py, which sizes its buffer from it and
names the per-tile breakdown DESIGN.md section 5c quotes: same slots, same order."""
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def enum_slots():
    with open(os.path.join(ROOT, "cosdata_b200", "csrc", "tensor_scan.cu")) as f:
        src = re.sub(r"//[^\n]*", "", f.read())
    body = re.search(r"enum : int \{([^}]*)\}", src).group(1)
    names = [s.strip() for s in body.split(",") if s.strip()]
    assert names[-1] == "TS_PROF_SLOTS", names
    return names[:-1]


def test_tool_slots_match_the_enum():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    try:
        import bench_prefilter_resident as tool
    finally:
        sys.path.pop(0)
    assert ["TS_PROF_" + s.upper() for s in tool.SLOTS] == enum_slots()


def test_every_s8_epilogue_slot_is_summed():
    # the s8 kernel's epilogue total is the sum of its parts, and every part is published
    with open(os.path.join(ROOT, "cosdata_b200", "csrc", "tensor_scan.cu")) as f:
        src = f.read()
    parts = [s for s in enum_slots() if s.startswith("TS_PROF_EPI_")]
    m = re.search(r"atomicAdd\(a\.prof \+ TS_PROF_EPILOGUE, (p_thr[^)]*)\);", src)
    assert m, "the s8 kernel's TS_PROF_EPILOGUE sum not found"
    assert len(m.group(1).split("+")) == len(parts), (m.group(1), parts)
    for s in parts:
        assert re.search(r"atomicAdd\(a\.prof \+ %s, p_\w+\);" % s, src), s
