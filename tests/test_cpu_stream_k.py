"""The wgmma GEMM's tile schedule (csrc/stream_k.cuh), built for the host with g++: no GPU needed.

Ordered stream-K is bit-exact and deadlock-free only if the partition keeps its promises: every (tile, k-block) unit is run exactly once, a
tile is split between at most two CTAs, which are neighbours, the lower one holding k-blocks [0, j) as its FIRST piece (the head) and the
higher one holding [j, num_kb) as its LAST piece (the tail), so that a CTA waits only at its end and only on the CTA before it."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

from tests.helpers import ROOT

SMS = 132


@pytest.fixture(scope="module")
def sk(tmp_path_factory):
    gxx = shutil.which("g++")
    if not gxx:
        pytest.skip("g++ not installed")
    out = str(tmp_path_factory.mktemp("stream_k") / "stream_k_host.so")
    subprocess.check_call([gxx, "-O2", "-shared", "-fPIC", "-I", os.path.join(ROOT, "text-to-sound-synthesis_b200", "csrc"),
                           os.path.join(ROOT, "tests", "native", "stream_k_host.cpp"), "-o", out])
    lib = ctypes.CDLL(out)
    lib.sk_applies.argtypes = [ctypes.c_int] * 4
    lib.sk_pieces.argtypes = [ctypes.c_int] * 5 + [ctypes.POINTER(ctypes.c_int), ctypes.c_int]
    return lib


def pieces(lib, tiles, num_kb, grid, c, stream_k):
    buf = (ctypes.c_int * 3 * 4096)()
    n = lib.sk_pieces(tiles, num_kb, grid, c, int(stream_k), ctypes.cast(buf, ctypes.POINTER(ctypes.c_int)), 4096)
    assert n >= 0
    return [tuple(buf[i]) for i in range(n)]


def check_partition(lib, tiles, num_kb, grid, stream_k):
    owner = np.full((tiles, num_kb), -1, dtype=np.int64)
    for c in range(grid):
        ps = pieces(lib, tiles, num_kb, grid, c, stream_k)
        for i, (t, k0, k1) in enumerate(ps):
            assert 0 <= t < tiles and 0 <= k0 < k1 <= num_kb, (c, ps)
            assert (owner[t, k0:k1] == -1).all(), f"unit run twice: tile {t} k-blocks [{k0}, {k1}) by CTA {c}"
            owner[t, k0:k1] = c
            if k1 < num_kb:
                assert i == 0 and k0 == 0, f"CTA {c}: a head must be its first piece and start at k-block 0: {ps}"
            if k0 > 0:
                assert i == len(ps) - 1 and k1 == num_kb, f"CTA {c}: a tail must be its last piece and end the tile: {ps}"
        if not stream_k:
            assert all(k0 == 0 and k1 == num_kb for _, k0, k1 in ps)
    assert (owner >= 0).all(), "a unit nobody runs"
    for t in range(tiles):
        cs = sorted(set(owner[t].tolist()))
        assert len(cs) <= 2, f"tile {t} spans CTAs {cs}"
        if len(cs) == 2:
            # the tail's producer is the CTA before it: k-blocks [0, j) by c, [j, num_kb) by c + 1
            j = int(np.argmax(owner[t] != owner[t, 0]))
            assert cs[1] == cs[0] + 1 and (owner[t, :j] == cs[0]).all() and (owner[t, j:] == cs[1]).all(), (t, owner[t])
    return owner


# the f16x3 denoiser GEMMs at B = 16 (tiles_m = 34; num_kb = K / 64), the logits GEMM, and small / awkward shapes
SHAPES = [(272, 16), (816, 16), (1088, 16), (272, 64), (68, 16), (133, 2), (137, 3), (264, 5), (1000, 9), (7, 7), (3, 1000), (265, 1)]


@pytest.mark.parametrize("tiles,num_kb", SHAPES)
@pytest.mark.parametrize("grid", [1, 2, 7, 64, 131, 132])
def test_partition(sk, tiles, num_kb, grid):
    grid = min(grid, tiles)
    applies = bool(sk.sk_applies(tiles, num_kb, grid, SMS))
    assert applies == (grid < tiles < 3 * grid and tiles % grid != 0 and num_kb > 1)
    check_partition(sk, tiles, num_kb, grid, stream_k=False)
    if applies:
        owner = check_partition(sk, tiles, num_kb, grid, stream_k=True)
        # balanced: every CTA runs floor or ceil of units / grid k-blocks
        counts = np.bincount(owner.ravel(), minlength=grid)
        assert counts.min() >= (tiles * num_kb) // grid and counts.max() <= -(-tiles * num_kb // grid)


def test_partition_sweep(sk):
    rng = np.random.default_rng(0)
    for _ in range(300):
        grid = int(rng.integers(1, SMS + 1))
        tiles = int(rng.integers(grid + 1, 3 * grid + 3))
        num_kb = int(rng.integers(2, 40))
        if sk.sk_applies(tiles, num_kb, grid, SMS):
            check_partition(sk, tiles, num_kb, grid, stream_k=True)


def test_stream_k_needs_a_resident_grid(sk):
    # more CTAs than SMs: a CTA could wait on one that is not resident, so the schedule stays data-parallel
    assert not sk.sk_applies(272, 16, SMS + 1, SMS)
    assert sk.sk_applies(272, 16, SMS, SMS)
    assert not sk.sk_applies(264, 16, SMS, SMS)  # no partial wave
    assert not sk.sk_applies(816, 16, SMS, SMS)  # three waves or more: data-parallel
    assert not sk.sk_applies(200, 1 << 24, SMS, SMS)  # unit count beyond 32 bits
