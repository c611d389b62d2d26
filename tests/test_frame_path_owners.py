"""The depth-frame path's host state has one owner per job in nvb_api.cu: ViewCompaction (the view bitset and the ticketed
compaction), ViewpointCache, HostInputRing (the staging of host inputs), LastView and FrameList. The ticketed compaction is
launched in one place, so the view path and nvb_blocks_union cannot disagree about the ticket counter, and the pinned host
words are read by name. No compute calls: this reads the CUDA source and runs without a GPU."""
import os
import re

from test_device_memory_owners import owner_spans, strip_comments

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
API = os.path.join(ROOT, "isaac_ros_nvblox_b200", "csrc", "nvb_api.cu")

# NvbMapper members that the owners replaced
MOVED = ("bits", "tile_state", "ticket", "ticket_base", "epoch", "vc_n", "vc_T", "vc_cam", "vc_grid", "vc_cells", "vc_bits",
         "depth_stage", "mask_stage", "stage_copied", "stage_consumed", "stage_used", "frame_seq", "last_depth", "last_rows",
         "last_cols", "last_T_L_C", "last_cam", "has_last_view", "h_list", "h_ints", "last_frame_n")
COMPACTION = (r"\bclass\s+ViewCompaction\b", r"\bViewCompaction::\w+\s*\(")
# a write of the ticket base or the epoch: an assignment or compound assignment (not ==), or an increment or decrement
WRITE = r"\b(?:ticket_base|epoch)_?\b\s*(?:[-+*/|&^]?=(?!=)|\+\+|--)|(?:\+\+|--)\s*(?:\w+(?:->|\.))*(?:ticket_base|epoch)_?\b"


def _api():
    return strip_comments(open(API).read())


def _line(text, pos):
    return text.count("\n", 0, pos) + 1


def _outside(text, pattern, spans):
    return [_line(text, m.start()) for m in re.finditer(pattern, text) if not any(a <= m.start() < b for a, b in spans)]


def test_mapper_holds_no_frame_path_state():
    text = _api()
    (start, end), = owner_spans(text, (r"\bstruct\s+NvbMapper\b",))
    body = text[start:end]
    declared = [name for name in MOVED if re.search(r"\b%s\b" % name, body)]
    assert not declared, "NvbMapper declares frame-path state that its owners hold: %s" % declared


def test_compaction_is_launched_once_inside_its_owner():
    text = _api()
    spans = owner_spans(text, COMPACTION)
    assert spans, "no ViewCompaction in nvb_api.cu"
    calls = [m.start() for m in re.finditer(r"\blaunchCompactAllocate\s*\(", text)]
    assert len(calls) == 1, "launchCompactAllocate( called at nvb_api.cu lines %s" % [_line(text, c) for c in calls]
    assert any(a <= calls[0] < b for a, b in spans), "launchCompactAllocate( outside ViewCompaction"


def test_ticket_base_and_epoch_are_written_only_by_their_owner():
    text = _api()
    spans = owner_spans(text, COMPACTION)
    assert spans, "no ViewCompaction in nvb_api.cu"
    stray = _outside(text, WRITE, spans)
    assert not stray, "ticket base or epoch written outside ViewCompaction at nvb_api.cu lines %s" % stray


def test_pinned_host_words_by_name():
    text = _api()
    pinned = set(re.findall(r"std::unique_ptr<[^;]*?\bPinnedFree>\s+(\w+)\s*;", text))
    assert "h_count_ring_" in pinned
    # an index or offset that is a number or a named constant (kSomething) picks a word by position
    by_number = r"\b(?:%s)\b(?:\.get\(\))?\s*(?:\[\s*(?:\d|k[A-Z])|\+\s*(?:\d|k[A-Z]))" % "|".join(sorted(pinned))
    found = [_line(text, m.start()) for m in re.finditer(by_number, text)]
    assert not found, "pinned host words addressed by number at nvb_api.cu lines %s" % found


def test_write_pattern_matches_the_hand_written_forms():
    for s in ("m->ticket_base += 3;", "ca.epoch = ++m->epoch;", "epoch_++;", "ticket_base_ = 0;"):
        assert re.search(WRITE, s), s
    for s in ("a.ticket_base == b", "x = ticket_base_;", "f(epoch)"):
        assert not re.search(WRITE, s), s
