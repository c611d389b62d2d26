"""Device and pinned host memory of the CUDA sources has one owner each: cudaMalloc and cudaFree are called only by
DeviceArray, cudaFreeHost only by PinnedFree. Every other allocation goes through them, so no return path leaks and no
failed allocation leaves a pointer to freed memory behind. The stream-ordered forms (cudaMallocAsync, cudaFreeAsync) are
not covered. No compute calls: this reads the sources and runs without a GPU."""
import glob
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# call -> the definitions allowed to make it: the class body and its out-of-class members
OWNERS = {
    "cudaMalloc": (r"\bclass\s+DeviceArray\b", r"\bDeviceArray<\w+>::\w+\s*\("),
    "cudaFree": (r"\bclass\s+DeviceArray\b", r"\bDeviceArray<\w+>::\w+\s*\("),
    "cudaFreeHost": (r"\bstruct\s+PinnedFree\b",),
}


def strip_comments(text):
    """Comments become blank, keeping the line numbers."""
    return re.sub(r"//[^\n]*|/\*.*?\*/", lambda m: "\n" * m.group(0).count("\n"), text, flags=re.S)


def owner_spans(text, patterns):
    """[start, end) of each definition in `text` that one of `patterns` opens: from the match to the brace closing its body."""
    spans = []
    for pattern in patterns:
        for m in re.finditer(pattern, text):
            i = text.index("{", m.end())
            depth = 1
            j = i + 1
            while depth:
                depth += {"{": 1, "}": -1}.get(text[j], 0)
                j += 1
            spans.append((m.start(), j))
    return spans


def stray_calls(text):
    """(call, line) of every cudaMalloc(, cudaFree( and cudaFreeHost( call in `text` outside the call's owner."""
    text = strip_comments(text)
    out = []
    for call, patterns in OWNERS.items():
        spans = owner_spans(text, patterns)
        for m in re.finditer(r"\b%s\s*\(" % call, text):
            if not any(a <= m.start() < b for a, b in spans):
                out.append((call, text.count("\n", 0, m.start()) + 1))
    return out


def test_owner_parser():
    text = """
template <typename T>
class DeviceArray {
  ~DeviceArray() { cudaFree(p_); }  // cudaMalloc( in a comment
};
template <typename T>
cudaError_t DeviceArray<T>::grow(size_t n) {
  if (n) { cudaMalloc(&q, n); }
  cudaFree(p_);
}
struct PinnedFree {
  void operator()(void* p) const { cudaFreeHost(p); }
};
void leak() { cudaMalloc(&p, 4); cudaMallocAsync(&p, 4, s); cudaFreeAsync(p, s); cudaMallocHost(&h, 4); }
void drop() { cudaFree(p), cudaFreeHost(h); }
"""
    assert sorted(stray_calls(text)) == [("cudaFree", 15), ("cudaFreeHost", 15), ("cudaMalloc", 14)]


def test_device_and_pinned_memory_have_one_owner():
    csrc = os.path.join(ROOT, "isaac_ros_nvblox_b200", "csrc")
    sources = sorted(glob.glob(os.path.join(csrc, "*.cu")) + glob.glob(os.path.join(csrc, "*.cuh")))
    assert sources
    stray = ["%s:%d: %s" % (os.path.basename(p), line, call) for p in sources for call, line in stray_calls(open(p).read())]
    assert not stray, "allocations outside DeviceArray / PinnedFree:\n" + "\n".join(stray)
