"""The one rule that sizes the binning buffer (`_C._Workspace`, `_C.RASTER` / `_C.VOXEL`, the key functions): what a
shape without a hint gets, how a hint grows and shrinks, how much a speculative forward adds, and how shapes are keyed.
Every host caller (the autograd entry points, the raw-parameter path, the engines and NativeTrainStep) goes through it.
No GPU and no pinned memory needed."""
import pytest
import torch

from r2_gaussian_b200 import _C

W = _C._Workspace
DEV = torch.device("cuda", 0)


@pytest.fixture(autouse=True)
def fresh_workspace(monkeypatch):
    monkeypatch.setattr(W, "hints", {})
    monkeypatch.setattr(W, "_pinned", [])


def test_seeds_and_floor():
    assert (_C.RASTER.seed, _C.VOXEL.seed) == (12, 8)
    key = _C.raster_key(DEV, 1000, 64, 64)
    assert W.provision(key, 1000, _C.RASTER.seed) == 16384          # 12 000 instances: the floor wins
    assert W.first(1, _C.VOXEL.seed) == 16384
    assert W.provision(key, 100_000, _C.RASTER.seed) == 5 << 18      # 1.2 M rounded up to the 256 Ki grid
    assert W.first(100_000, _C.VOXEL.seed) == 7 << 17                 # 800 000 rounded up to the 128 Ki grid


@pytest.mark.parametrize("n", [1, 4095, 4096, 4097, 16384, 32769, 1_000_000, 12_345_678, 1 << 30])
def test_rounding_granularity(n):
    step = 1 << max(12, n.bit_length() - 3)       # an eighth of the next power of two, at least one 4 KiB page
    r = W._round(n)
    assert r % step == 0 and n <= r < n + step
    assert W._round(r) == r


def test_grow_at_once_shrink_only_below_half():
    key = _C.raster_key(DEV, 5000, 128, 128)
    W.update(key, 100_000)
    first = W.hints[key]
    assert first == W.grown(100_000) == W._round(121_024) and first > 100_000
    assert W.provision(key, 5000, _C.RASTER.seed) == first
    W.update(key, 200_000)                         # more instances: the hint grows at once
    grown = W.hints[key]
    assert grown == W.grown(200_000) > first
    W.update(key, 120_000)                         # fewer, but the new want is still at least half the hint: kept
    assert W.grown(120_000) >= grown // 2 and W.hints[key] == grown
    W.update(key, 50_000)                          # far fewer: the hint shrinks to the new want
    assert W.grown(50_000) < grown // 2 and W.hints[key] == W.grown(50_000)


def test_speculative_doubling():
    P = 20_000
    key = _C.voxel_key(DEV, P, 32, 32, 32, 2.0)
    no_hint = W.first(P, _C.VOXEL.seed)
    assert W.provision(key, P, _C.VOXEL.seed, speculative=True) == W._round(2 * no_hint)
    W.hints[key] = 409_600
    assert W.provision(key, P, _C.VOXEL.seed) == 409_600
    assert W.provision(key, P, _C.VOXEL.seed, speculative=True) == W._round(2 * 409_600)
    W.hints[key] = 16_384                          # twice the hint is below seed * P: the seed wins
    assert W.provision(key, P, _C.VOXEL.seed, speculative=True) == W._round(_C.VOXEL.seed * P)


def test_keys():
    a = _C.voxel_key(DEV, 1000, 64, 64, 64, 2.0)
    b = _C.voxel_key(DEV, 1000, 64, 64, 64, 1.0)   # same grid, half the voxel pitch
    assert a != b
    assert a == _C.voxel_key(DEV, 1000, 64, 64, 64, 2.0000000001)
    assert _C.raster_key(DEV, 1000, 64, 64) != _C.raster_key(torch.device("cuda", 1), 1000, 64, 64)
    assert _C.raster_key(DEV, 1000, 64, 48) != _C.raster_key(DEV, 1000, 48, 64)


def test_status_word_read_updates_the_hint_and_recycles():
    key = _C.raster_key(DEV, 1000, 64, 64)
    word = torch.tensor([30_000, 1], dtype=torch.int32)
    assert W.read(word, key) == (30_000, 1)
    assert W.hints[key] == W.grown(30_000)
    assert W._pinned == [word]


def test_speculative_switch(monkeypatch):
    monkeypatch.delenv("R2X_SPECULATIVE", raising=False)
    assert not _C.speculative.active()
    with _C.speculative(True):
        assert _C.speculative.active()
        with _C.speculative(False):
            assert not _C.speculative.active()
        monkeypatch.setenv("R2X_SPECULATIVE", "0")
        assert not _C.speculative.active()
    assert not _C.speculative.active()
