"""Host-to-device copies of the CUDA sources are stream-ordered. The mapper's streams are non-blocking, so a blocking
cudaMemcpy from pageable memory is not ordered against them and may return before its DMA has landed. No compute calls:
this reads the sources and runs without a GPU."""
import glob
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def blocking_copies(text):
    """The argument lists of every blocking cudaMemcpy( call in `text`."""
    out = []
    for m in re.finditer(r"\bcudaMemcpy\(", text):
        depth, i = 1, m.end()
        while depth:
            depth += {"(": 1, ")": -1}.get(text[i], 0)
            i += 1
        out.append(text[m.end():i - 1])
    return out


def test_blocking_copy_parser():
    text = "cudaMemcpy(a, f(b), n, cudaMemcpyDeviceToHost); cudaMemcpyAsync(c, d, n, cudaMemcpyHostToDevice, s);"
    assert blocking_copies(text) == ["a, f(b), n, cudaMemcpyDeviceToHost"]


def test_no_blocking_host_to_device_copy():
    sources = sorted(glob.glob(os.path.join(ROOT, "isaac_ros_nvblox_b200", "csrc", "*.cu")))
    assert sources
    for path in sources:
        for args in blocking_copies(open(path).read()):
            assert "cudaMemcpyHostToDevice" not in args, "%s: blocking cudaMemcpy(%s)" % (os.path.basename(path), args)
