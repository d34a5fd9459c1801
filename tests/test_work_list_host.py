"""The work-list rule every persistent kernel and the host share (device_types.h): block b of a `grid`-block launch
walks the chunk [qw_chunk_begin(total, b, grid), qw_chunk_begin(total, b + 1, grid)) of the flat work list, and a
strided threshold sample takes item k * stride + phase of split s (phase = s % stride when stride > 1, else 0), where
the host sizes split s's share of the list with qw_sample_count. Pinned against a restatement, without a GPU."""
import ctypes as C
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SHIM = ('#include "device_types.h"\n'
        'extern "C" unsigned chunk_begin(unsigned total, unsigned b, unsigned grid) { return qw_chunk_begin(total, b, grid); }\n'
        'extern "C" unsigned sample_item(unsigned k, unsigned s, unsigned stride) { return qw_sample_item(k, s, stride); }\n'
        'extern "C" unsigned sample_count(unsigned n, unsigned s, unsigned stride) { return qw_sample_count(n, s, stride); }\n')


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    d = tmp_path_factory.mktemp("work_list")
    (d / "shim.cpp").write_text(SHIM)
    cxx = os.environ.get("CXX", "g++")
    subprocess.run([cxx, "-O2", "-Wall", "-Werror", "-std=c++17", "-fPIC", "-shared", "-I", os.path.join(ROOT, "quickwit_b200", "csrc"),
                    "-o", str(d / "shim.so"), str(d / "shim.cpp")], check=True)
    lib = C.CDLL(str(d / "shim.so"))
    for f in (lib.chunk_begin, lib.sample_item, lib.sample_count):
        f.restype = C.c_uint
        f.argtypes = [C.c_uint, C.c_uint, C.c_uint]
    return lib


@pytest.mark.parametrize("total", [0, 1, 7, 264, 1000, 6528, 2**31 + 5])
@pytest.mark.parametrize("grid", [1, 5, 132, 264, 1000, 1056])
def test_chunks_partition_the_work_list(shim, total, grid):
    bounds = [shim.chunk_begin(total, b, grid) for b in range(grid + 1)]
    assert bounds == [total * b // grid for b in range(grid + 1)]
    assert bounds[0] == 0 and bounds[-1] == total
    sizes = [e - b for b, e in zip(bounds, bounds[1:])]
    assert all(s >= 0 for s in sizes) and sum(sizes) == total
    # every block gets floor or ceil of total / grid items: the longest chunk is ceil(total / grid)
    assert max(sizes) == -(-total // grid) and min(sizes) == total // grid
    if grid <= total:
        assert min(sizes) >= 1  # a launch of at most `total` blocks leaves no block idle


@pytest.mark.parametrize("stride", [1, 2, 3, 16, 25, 32])
def test_sampled_items_of_each_split(shim, stride):
    for s in [0, 1, 2, 5, 15, 16, 31, 33, 100]:
        phase = s % stride if stride > 1 else 0
        for n in [0, 1, 2, phase, phase + 1, stride - 1, stride, stride + 1, 3 * stride + phase, 137, 204, 1000]:
            want = list(range(phase, n, stride))
            cnt = shim.sample_count(n, s, stride)
            assert cnt == len(want), (n, s, stride)
            assert [shim.sample_item(k, s, stride) for k in range(cnt)] == want, (n, s, stride)


def test_stride_one_takes_every_item(shim):
    for s in [0, 1, 7, 31]:
        for n in [0, 1, 16, 1000]:
            assert shim.sample_count(n, s, 1) == n
            assert [shim.sample_item(k, s, 1) for k in range(n)] == list(range(n))


def test_sampled_work_list_of_a_batch(shim):
    """The host's prefix over the splits' sampled counts and the kernels' walk of it visit each split's sampled items
    exactly once, whichever block a work item falls to: one split, empty splits, and a batch larger than the grid."""
    for items, stride, grid in [([1000], 16, 264), ([0, 137, 0, 0, 5, 137, 1, 0], 8, 7),
                                ([204] * 32, 25, 264), ([3, 0, 2], 1, 2), ([0, 0], 4, 3)]:
        fw = [0]
        for s, n in enumerate(items):
            fw.append(fw[-1] + shim.sample_count(n, s, stride))
        total = fw[-1]
        seen = {s: [] for s in range(len(items))}
        for b in range(grid):
            for w in range(shim.chunk_begin(total, b, grid), shim.chunk_begin(total, b + 1, grid)):
                s = max(i for i in range(len(items)) if fw[i] <= w)  # the split of work item w
                seen[s].append(shim.sample_item(w - fw[s], s, stride))
        for s, n in enumerate(items):
            phase = s % stride if stride > 1 else 0
            assert seen[s] == list(range(phase, n, stride)), (items, stride, grid, s)
