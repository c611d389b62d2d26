"""Block-index lists cross the C ABI through one intake and one output path. A caller's list is checked, range-checked and
made a set only in takeBlockList, and records are written back as xyz triples only in writeBlockList, so no entry point
applies its own version of those rules. No compute calls: this reads the source and runs without a GPU."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
API = os.path.join(ROOT, "isaac_ros_nvblox_b200", "csrc", "nvb_api.cu")


def function_bodies(text):
    """{name: body} of every top-level function definition in `text` (a line `type name(...) {` at column 0)."""
    out = {}
    for m in re.finditer(r"^[A-Za-z][\w:<>*& ]*?\b(\w+)\([^;{]*\)\s*\{\s*$", text, re.M):
        depth, i = 1, m.end()
        while depth and i < len(text):
            depth += {"{": 1, "}": -1}.get(text[i], 0)
            i += 1
        out[m.group(1)] = text[m.start():i]
    return out


def outside(text, name, pattern):
    """The lines of `text` outside function `name` that match `pattern`."""
    rest = text.replace(function_bodies(text).get(name, ""), "")
    return [line.strip() for line in rest.splitlines() if re.search(pattern, line)]


RANGE_CHECK = r"indexInRange\(\s*\w+\[3 \* i\]"
UNIQUE = r"std::unique\b"
TRIPLE_WRITE = r"(_xyz_host|\bout_xyz)\[3 \* i \+ 2\] ="


def test_parser_finds_functions():
    text = ("int a(int x) {\n  if (x) {\n    return 1;\n  }\n  return 0;\n}\n"
            "int32_t nvb_b(NvbMapper* m, const int32_t* xyz_host, int32_t n) {\n  return indexInRange(xyz_host[3 * i], 0, 0);\n}\n")
    bodies = function_bodies(text)
    assert set(bodies) == {"a", "nvb_b"}
    assert outside(text, "a", RANGE_CHECK) == ["return indexInRange(xyz_host[3 * i], 0, 0);"]
    assert outside(text, "nvb_b", RANGE_CHECK) == []


def test_patterns_match_the_hand_written_forms():
    assert re.search(RANGE_CHECK, "if (!indexInRange(blocks_xyz_host[3 * i], blocks_xyz_host[3 * i + 1], z))")
    assert re.search(UNIQUE, "v.erase(std::unique(v.begin(), v.end()), v.end());")
    assert re.search(TRIPLE_WRITE, "removed_xyz_host[3 * i] = a, removed_xyz_host[3 * i + 2] = b;")
    assert re.search(TRIPLE_WRITE, "for (...) out_xyz[3 * i] = s.x, out_xyz[3 * i + 2] = s.z;")
    assert not re.search(TRIPLE_WRITE, "xyz[3 * i + 2] = p.z;")  # float point outputs are not block lists


def test_caller_lists_are_checked_only_by_the_intake():
    text = open(API).read()
    assert "takeBlockList" in function_bodies(text)
    assert outside(text, "takeBlockList", RANGE_CHECK) == []
    assert outside(text, "takeBlockList", UNIQUE) == []


def test_block_lists_are_written_only_by_the_output_function():
    text = open(API).read()
    assert "writeBlockList" in function_bodies(text)
    assert outside(text, "writeBlockList", TRIPLE_WRITE) == []
