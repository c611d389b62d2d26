"""The state of the features added after the layers has one owner per job in nvb_api.cu: MeshArena (the mesh arena),
SlotOrder (the block-index sort of a layer's slots), GroundPlaneEstimator, DynamicsOutputs, MaskerOutputs and BlockUnion.
Doubling growth is written once, in DeviceArray, and the union's state words are read by name. No compute calls: this reads
the CUDA sources and runs without a GPU."""
import os
import re

from test_device_memory_owners import owner_spans, strip_comments

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "isaac_ros_nvblox_b200", "csrc")

# owner -> the NvbMapper members it replaced
MOVED = {
    "MeshArena": ("mesh_v", "mesh_n", "mesh_t", "mesh_c", "mesh_alt_v", "mesh_alt_n", "mesh_alt_t", "mesh_alt_c", "mesh_state",
                  "mesh_counts", "mesh_offsets", "mesh_xyz_dev"),
    "GroundPlaneEstimator": ("gp_keys", "gp_slots", "gp_counts", "gp_sort_temp", "gp_totals", "gp_crossings", "gp_candidates",
                             "gp_fit_points", "gp_states", "gp_costs", "gp_planes", "gp_result", "gp_valid", "gp_num_crossings",
                             "gp_num_candidates", "gp_found", "gp_plane"),
    "DynamicsOutputs": ("dyn_depth", "dyn_mask", "dyn_clean", "dyn_overlay", "dyn_points", "dyn_counts", "dyn_totals",
                        "dyn_rows", "dyn_cols", "cc_labels", "cc_sizes"),
    "MaskerOutputs": ("msk_min_depth", "msk_background", "msk_foreground", "msk_overlay", "msk_rows", "msk_cols",
                      "msk_has_overlay"),
    "BlockUnion": ("union_list", "union_list_count", "union_bits", "union_state"),
}
OWNERS = ("MeshArena", "SlotOrder", "GroundPlaneEstimator", "DynamicsOutputs", "MaskerOutputs", "BlockUnion")


def _read(name):
    return strip_comments(open(os.path.join(CSRC, name)).read())


def _line(text, pos):
    return text.count("\n", 0, pos) + 1


def _spans(text, owner):
    return owner_spans(text, (r"\b(?:class|struct)\s+%s\b" % owner, r"\b%s::\w+\s*\(" % owner))


def test_mapper_holds_no_feature_state():
    text = _read("nvb_api.cu")
    (start, end), = owner_spans(text, (r"\bstruct\s+NvbMapper\b",))
    body = text[start:end]
    declared = [name for names in MOVED.values() for name in names if re.search(r"\b%s\b" % name, body)]
    assert not declared, "NvbMapper declares state that its owners hold: %s" % declared
    assert re.search(r"\bdyn_event\b", body), "nvb_mapper_wait_for's hand-over event stays on NvbMapper"


def test_moved_state_is_gone_from_the_api():
    text = _read("nvb_api.cu")
    word = r"\b(?:%s)\b" % "|".join(name for names in MOVED.values() for name in names)
    found = [_line(text, m.start()) for m in re.finditer(word, text)]
    assert not found, "moved members still named at nvb_api.cu lines %s" % found


def _arrays(text, cls):
    """The array members (named with a trailing underscore) that the body of class `cls` declares."""
    (a, b), = owner_spans(text, (r"\b(?:class|struct)\s+%s(?=\s*\{)" % cls,))
    names = set()
    for decl in re.findall(r"\b(?:DeviceArray<[^;{}]*?>|Geometry)\s+([\w\s,]+);", text[a:b]):
        names.update(n.strip() for n in decl.split(",") if n.strip().endswith("_"))
    return names


def test_owned_arrays_grow_only_inside_their_owner():
    text = _read("nvb_api.cu")
    classes = set(re.findall(r"\b(?:class|struct)\s+(\w+)\s*\{", text))
    declared = {c: _arrays(text, c) for c in classes}
    stray = []
    for owner in OWNERS:
        assert declared[owner], "no arrays in %s" % owner
        for m in re.finditer(r"\b(%s)\s*\.\s*grow\w*\s*\(" % "|".join(sorted(declared[owner])), text):
            homes = [c for c in classes if m.group(1) in declared[c]]
            if not any(a <= m.start() < b for c in homes for a, b in _spans(text, c)):
                stray.append("%s: %d" % (m.group(1), _line(text, m.start())))
    assert not stray, "arrays grown outside the class that declares them:\n" + "\n".join(stray)


def test_doubling_growth_is_written_once():
    text = _read("nvb_api.cu")
    found = [_line(text, m.start()) for m in re.finditer(r"grow\(m, \w+, std::max\(\w+, 2 \*", text)]
    assert not found, "hand-written doubling growth at nvb_api.cu lines %s" % found


def test_slot_sort_is_called_only_inside_its_owner():
    text = _read("nvb_api.cu")
    spans = _spans(text, "SlotOrder")
    assert spans, "no SlotOrder in nvb_api.cu"
    for call in ("launchGroundSortBlocks", "groundSortTempBytes"):
        calls = [m.start() for m in re.finditer(r"\b%s\s*\(" % call, text)]
        assert calls, call
        stray = [_line(text, c) for c in calls if not any(a <= c < b for a, b in spans)]
        assert not stray, "%s( outside SlotOrder at nvb_api.cu lines %s" % (call, stray)
    # only the sort knows that the sorted slots follow the unsorted ones
    stray = [_line(text, m.start()) for m in re.finditer(r"\+\s*hw\b", text) if not any(a <= m.start() < b for a, b in spans)]
    assert not stray, "the sort's `+ hw` layout read outside SlotOrder at nvb_api.cu lines %s" % stray


def test_union_state_words_by_name():
    merge = _read("nvb_merge.cu")
    found = ["nvb_merge.cu:%d" % _line(merge, m.start()) for m in re.finditer(r"\b(?:state|st)\s*\[\s*\d", merge)]
    api = _read("nvb_api.cu")
    spans = _spans(api, "BlockUnion") + owner_spans(api, (r"\bnvb_blocks_union\w*\s*\(",))
    found += ["nvb_api.cu:%d" % _line(api, m.start()) for m in re.finditer(r"\b(?:state|st)\s*\[\s*\d", api)
              if any(a <= m.start() < b for a, b in spans)]
    assert not found, "union state words by number:\n" + "\n".join(found)
    header = _read("nvb_internal.cuh")
    assert re.search(r"static_assert\(sizeof\(UnionState\) == 8 \* sizeof\(int\)", header)
