"""The scratch carving helper of kgv_internal.h (kgv_carve / kgv_reserve_carved), on the host: every array starts 256-byte aligned right
after the previous one and its padding, arrays never overlap, the measuring pass gives the size the carving pass fills, and an empty array
takes no space beyond alignment."""
import os
import subprocess

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
CUDA_HOME = os.environ.get("CUDA_HOME", "/usr/local/cuda")


def _al256(x):
    return (x + 255) & ~255


@pytest.fixture(scope="module")
def layouts(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("carve") / "scratch_carve_test")
    subprocess.run(["g++", "-std=c++17", "-O1", "-I" + os.path.join(CUDA_HOME, "include"), "-o", exe, os.path.join(HERE, "cpp", "scratch_carve_test.cpp")],
                   check=True, capture_output=True, text=True)
    out = subprocess.run([exe], check=True, capture_output=True, text=True).stdout
    res = []
    for line in out.splitlines():
        f = line.split()
        if f[0] == "layout":
            n, measured, need, end, null_measure = map(int, f[1:])
            res.append({"n": n, "measured": measured, "need": need, "end": end, "null_measure": null_measure, "arrays": []})
        else:
            res[-1]["arrays"].append((f[1], int(f[2]), int(f[3])))
    assert [r["n"] for r in res] == [0, 1, 7, 33, 1000]
    return res


def test_arrays_are_256_byte_aligned(layouts):
    for r in layouts:
        for name, off, _ in r["arrays"]:
            assert off % 256 == 0, (r["n"], name, off)


def test_each_array_starts_at_the_rounded_end_of_the_previous(layouts):
    # the offsets the call sites used to chain by hand: next = al256(previous offset + previous bytes), padding included
    for r in layouts:
        arr = r["arrays"]
        assert arr[0][1] == 0
        for (name, off, nbytes), (_, nxt, _) in zip(arr, arr[1:]):
            assert nxt == _al256(off + nbytes), (r["n"], name)


def test_arrays_never_overlap_and_padding_is_kept(layouts):
    for r in layouts:
        spans = sorted((off, off + nbytes) for _, off, nbytes in r["arrays"] if nbytes)
        for (_, e0), (s1, _) in zip(spans, spans[1:]):
            assert e0 <= s1, r["n"]
        assert spans[-1][1] <= r["need"]


def test_measuring_pass_gives_the_size_the_carving_pass_uses(layouts):
    for r in layouts:
        assert r["null_measure"] == 1  # measuring hands out no pointers
        last_name, last_off, last_bytes = r["arrays"][-1]
        assert r["measured"] == r["need"] == r["end"] == _al256(last_off + last_bytes), r["n"]


def test_zero_length_array_takes_no_space(layouts):
    for r in layouts:
        arr = r["arrays"]
        for i, (name, off, nbytes) in enumerate(arr):
            if nbytes == 0:
                assert arr[i + 1][1] == off, (r["n"], name)
