"""The ESDF integrator's device state has one owner, EsdfState in nvb_api.cu, and its counter words and statistics are read
by name: no hand-packed offsets into the counters block, no statistics slot by number, the phase-max size and the
neighbour table's fill byte written once. No compute calls: this reads the CUDA sources and runs without a GPU."""
import glob
import os
import re

from test_device_memory_owners import owner_spans, strip_comments

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "isaac_ros_nvblox_b200", "csrc")

# NvbMapper members that EsdfState replaced
MOVED = ("work", "upd_list", "clr_list", "cleared_list", "ring_a", "ring_b", "stamp_a", "stamp_b", "seed_upd", "seed_clr",
         "psum", "nbr", "nbr27", "cand_stamp", "cand_a", "cand_b", "shadow", "xslab", "xrec", "xseg", "xseg_grid", "xcounts",
         "clr_bits", "stats", "phase_max", "barrier", "colset", "cols", "dead_cleared_xyz", "esdf_persistent",
         "esdf_reserved_sms", "esdf_split_min_k", "ges_switch", "prune_default", "prune_ok", "update_seq", "esdf_ints")
# the offsets of the hand-packed counters block
OFFSETS = ("kWorkCount", "kUpdCount", "kClrCount", "kClrAabb", "kClearedCount", "kRingCount", "kRingId", "kTodoCount",
           "kFrameCount", "kError", "kClearedSeq", "kTailState", "kDeadCount", "kDeadClearedCount", "kGesCounts",
           "kTodoFsCount", "kFsWorkCount", "kColsCount", "kColorWorkCount", "kXTail", "kTodoMeshCount", "kNumInts")


def _sources():
    paths = sorted(glob.glob(os.path.join(CSRC, "*.cu")) + glob.glob(os.path.join(CSRC, "*.cuh")))
    assert any(p.endswith("nvb_api.cu") for p in paths)
    return {os.path.basename(p): strip_comments(open(p).read()) for p in paths}


def _lines(text, pattern):
    return [text.count("\n", 0, m.start()) + 1 for m in re.finditer(pattern, text)]


def test_no_counter_offsets():
    word = r"\b(?:esdf_ints|%s)\b" % "|".join(OFFSETS)
    found = ["%s:%d" % (name, line) for name, text in _sources().items() for line in _lines(text, word)]
    assert not found, "counter words by offset instead of DeviceCounters fields:\n" + "\n".join(found)


def test_statistics_by_name():
    slot = r"\bstats(?:\.get\(\))?\s*(?:\[\s*\d|\+\s*\d)"
    found = ["%s:%d" % (name, line) for name, text in _sources().items()
             if name.startswith("nvb_esdf") and name.endswith(".cu") or name == "nvb_api.cu" for line in _lines(text, slot)]
    assert not found, "ESDF statistics slots by number instead of EsdfStat:\n" + "\n".join(found)


def test_phase_max_size_written_once():
    found = [(name, text.splitlines()[line - 1].strip()) for name, text in _sources().items()
             for line in _lines(text, r"\b4000\b")]
    assert found == [("nvb_internal.cuh", "constexpr int kPhaseMaxEntries = 4000;")]


def test_mapper_holds_no_esdf_state():
    text = _sources()["nvb_api.cu"]
    (start, end), = owner_spans(text, (r"\bstruct\s+NvbMapper\b",))
    body = text[start:end]
    declared = [name for name in MOVED if re.search(r"\b%s\b" % name, body)]
    assert not declared, "NvbMapper declares ESDF state that EsdfState owns: %s" % declared


def test_esdf_state_grows_only_in_its_members():
    text = _sources()["nvb_api.cu"]
    spans = owner_spans(text, (r"\bclass\s+EsdfState\b", r"\bEsdfState::\w+\s*\("))
    assert len(spans) > 5
    grow = r"\b(?:%s)_?\s*\.\s*grow\s*\(" % "|".join(MOVED)
    stray = [text.count("\n", 0, m.start()) + 1 for m in re.finditer(grow, text)
             if not any(a <= m.start() < b for a, b in spans)]
    assert not stray, "ESDF state grown outside EsdfState at nvb_api.cu lines %s" % stray


def test_neighbour_fill_byte_written_once():
    # the host's memset byte; the kernel's 0xFEFEFEFE word in nvb_esdf.cu is a device write
    assert len(_lines(_sources()["nvb_api.cu"], r"\b0x[fF][eE]\b")) == 1
