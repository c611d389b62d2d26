"""Only the ESDF block-format header (nvb_esdf_block.cuh) knows where an ESDF voxel's words live in a block, and only the
C ABI's block copies and voxel queries turn blocks into the reference's 20-byte EsdfVoxel records. No compute calls: this
reads the CUDA sources and runs without a GPU."""
import glob
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "isaac_ros_nvblox_b200", "csrc")
HEADER = "nvb_esdf_block.cuh"


def _sources():
    paths = sorted(glob.glob(os.path.join(CSRC, "*.cu")) + glob.glob(os.path.join(CSRC, "*.cuh")))
    assert any(p.endswith(HEADER) for p in paths)
    return {os.path.basename(p): re.sub(r"//[^\n]*", "", open(p).read()) for p in paths}


def _function_body(text, name):
    m = re.search(r"\b%s\s*\([^)]*\)\s*\{" % name, text)
    assert m, name
    depth, i = 1, m.end()
    while depth:
        depth += {"{": 1, "}": -1}.get(text[i], 0)
        i += 1
    return text[m.end():i - 1]


def test_function_body_parser():
    text = "void f(int a) { if (a) { g(); } h(); } void k() { x(); }"
    assert _function_body(text, "f") == " if (a) { g(); } h(); "


# The old layout written out: a 20-byte stride, a 5-word stride (`v * 5 + 4`) or the flag bytes of a 20-byte record (`e[16]`,
# `e[17]`). "1.5 * n" (growth factors) is not a stride, and an array declared with 16 or 17 elements is not a subscript.
STRIDE = re.compile(r"\*\s*20\b|\b20\s*\*|(?<![\d.])\b5\s*\*|\*\s*5\b(?!\.)|\w\s*\[\s*1[67]\s*\]")
DECLARATION = re.compile(r"^\s*(?:__shared__\s+)?(?:(?:const|signed|unsigned)\s+)*(?:char|int|float)\s+\w+\s*(?:\[\d+\])+")


def test_stride_patterns():
    for bad in ("v * 5 + 4", "e[16]", "e[17] != 0", "5 * v", "blk + v * 20", "20 * v"):
        assert STRIDE.search(bad), bad
    for ok in ("(size_t)(1.5 * words) + 64", "v * 16", "kEsdfCellWords * v", "x[15]"):
        assert not STRIDE.search(ok), ok
    assert DECLARATION.search("  __shared__ int s_src[16], s_fs[16];") and not DECLARATION.search("  d = e[16];")


def test_no_twenty_byte_voxel_stride_outside_the_layout_header():
    for name, text in _sources().items():
        if name == HEADER:
            continue
        assert "kEsdfVoxelWords" not in text, name
        for line in text.splitlines():
            if STRIDE.search(line):
                assert "kWeldMax" in line or DECLARATION.search(line), (name, line.strip())


def test_records_only_at_the_api_boundary():
    allowed = {"nvb_util.cu": ("gatherBlocksKernel", "scatterBlocksKernel"), "nvb_query.cu": ("queryVoxelsKernel",)}
    for name, text in _sources().items():
        if name == HEADER:
            continue
        uses = len(re.findall(r"\b(?:kEsdfRecordWords|esdfVoxelToRecord|esdfVoxelFromRecord)\b", text))
        inside = sum(len(re.findall(r"\b(?:kEsdfRecordWords|esdfVoxelToRecord|esdfVoxelFromRecord)\b", _function_body(text, f)))
                     for f in allowed.get(name, ()))
        assert uses == inside, name
    assert "esdfVoxelToRecord" in _function_body(_sources()["nvb_util.cu"], "gatherBlocksKernel")
    assert "esdfVoxelFromRecord" in _function_body(_sources()["nvb_util.cu"], "scatterBlocksKernel")
