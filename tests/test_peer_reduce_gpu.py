"""r2x_peer_allreduce_sum_t, the exchange step of the Gaussian-sharded projector, against the rank-ordered float32 sum.

Everything runs in one process on one device: the `world` partial buffers are torch tensors, and each rank's flag array
(R2X_MAX_PEERS uint32 words) is set to the epoch, or one ahead of it, before the call.  The kernel's wait
(int32)(flag - epoch) >= 0 then holds on entry, so no call ever waits; the time-out is short (1e7 SM cycles, a few ms)
so that a wrongly set flag shows as status = 1 instead of a 2 s stall.  No case lets a peer stay away.

The sum is b[0] + b[1] + ... + b[world-1], left to right in float32, bit for bit (the library is built without -ftz and
fast-math: IEEE adds).  The cases: order-sensitive data that the reversed and the pairwise order sum differently; signed
zeros, subnormals, infinities and overflow; world sizes 1 to R2X_MAX_PEERS with every rank calling; lengths around the
float4 lanes, one CTA's span and the grid cap (grid-stride loops), each with and without a scalar tail; the epoch wrap;
and the refusals, which leave the output untouched."""
import ctypes as C
import os
import re

import numpy as np
import pytest

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TIMEOUT_CYCLES = 10 ** 7
SENTINEL = np.float32(-1234.5)


def _header_define(name):
    with open(os.path.join(ROOT, "include", "r2x.h")) as f:
        return int(re.search(rf"#define\s+{name}\s+(\d+)", f.read()).group(1))


MAX_PEERS = _header_define("R2X_MAX_PEERS")
ERR_INVALID = _header_define("R2X_ERR_INVALID")


def _lib():
    from r2_gaussian_b200._lib import load
    return load()


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@np.errstate(over="ignore", invalid="ignore")
def seq_sum(bufs):
    acc = bufs[0].copy()
    for b in bufs[1:]:
        acc = acc + b
    return acc


@np.errstate(over="ignore", invalid="ignore")
def pair_sum(bufs):
    if len(bufs) == 1:
        return bufs[0].copy()
    mid = len(bufs) // 2
    return pair_sum(bufs[:mid]) + pair_sum(bufs[mid:])


def same_bits(got, want):
    """Bit for bit, except that a NaN matches any NaN (the GPU's adds return the canonical NaN)."""
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    nan = np.isnan(want)
    return (np.array_equal(np.isnan(got), nan)
            and np.array_equal(got[~nan].view(np.uint32), want[~nan].view(np.uint32)))


class Peers:
    """`world` partial buffers, their flag arrays and an output, all on cuda:0.  Buffers hold max(n, 4) floats so
    that n = 0 still passes real pointers."""

    def __init__(self, parts):
        self.world, self.n = len(parts), int(parts[0].size)
        m = max(self.n, 4)
        self.host = [np.asarray(p, np.float32) for p in parts]
        self.bufs = []
        for p in self.host:
            t = torch.zeros(m, dtype=torch.float32, device="cuda")
            t[:self.n] = torch.from_numpy(p.copy())
            self.bufs.append(t)
        self.flags = torch.zeros((self.world, MAX_PEERS), dtype=torch.int32, device="cuda")
        self.out = torch.full((m,), float(SENTINEL), dtype=torch.float32, device="cuda")
        self.status = torch.zeros(1, dtype=torch.int32, device="cuda")

    def arm(self, rank, epoch, ahead=()):
        """flags[rank][q] = epoch for q < world, or epoch + 1 (mod 2^32) for q in `ahead`."""
        row = np.array([(epoch + (1 if q in ahead else 0)) & 0xFFFFFFFF for q in range(self.world)], np.uint32)
        self.flags[rank, :self.world] = torch.from_numpy(row.view(np.int32)).cuda()

    def flags_host(self):
        return self.flags.cpu().numpy().view(np.uint32)

    def call(self, rank, epoch, n=None, world=None, bufs=None, flags=None, out=None, status=None):
        world = self.world if world is None else world
        ptrs = [b.data_ptr() for b in self.bufs] if bufs is None else bufs
        fptrs = [self.flags[p].data_ptr() for p in range(self.world)] if flags is None else flags
        k = max(world, 1)
        ptrs = (ptrs + [None] * k)[:k]
        fptrs = (fptrs + [None] * k)[:k]
        return _lib().r2x_peer_allreduce_sum_t(
            torch.cuda.current_stream().cuda_stream, world, rank, (C.c_void_p * k)(*ptrs), (C.c_void_p * k)(*fptrs),
            epoch & 0xFFFFFFFF, self.out.data_ptr() if out is None else out, self.n if n is None else n,
            self.status.data_ptr() if status is None else status, TIMEOUT_CYCLES)

    def reduce_as(self, rank, epoch, ahead=()):
        """One armed call of `rank`; asserts status 0 and that its signal reached every peer's flag array (and changed
        nothing else there).  -> out[:n] as a host array."""
        self.arm(rank, epoch, ahead)
        before = self.flags_host()
        self.out.fill_(float(SENTINEL))
        assert self.call(rank, epoch) == 0
        torch.cuda.synchronize()
        assert int(self.status.item()) == 0, f"rank {rank}: a peer was reported missing"
        after = self.flags_host()
        assert np.all(after[:, rank] == np.uint32(epoch & 0xFFFFFFFF)), f"rank {rank}: the signal missed a peer"
        before[:, rank] = after[:, rank]
        assert np.array_equal(before, after), f"rank {rank}: a flag word other than column {rank} changed"
        out = self.out.cpu().numpy()
        assert np.all(out[self.n:] == SENTINEL), "the kernel wrote past n"
        return out[:self.n]


# ---- data ---------------------------------------------------------------------------------------------------------------
def order_sensitive(world, n, seed):
    """Values of very different magnitudes spread over the ranks: 1e8 + 1 - 1e8 is 0 in float32, 1e8 - 1e8 + 1 is 1."""
    r = np.random.default_rng(seed)
    pool = np.array([1e8, -1e8, 1.0, -1.0, 3.0, 0.5, 2.5e7, -3.3e7, 1e-3, 7.0], np.float32)
    parts = pool[r.integers(0, len(pool), (world, n))]
    parts *= (1.0 + r.random((world, n)) * 1e-3).astype(np.float32)
    return list(parts.astype(np.float32))


def specials(world, n, seed):
    """Signed zeros, subnormals, infinities (inf + -inf), sums that overflow to inf, and ordinary numbers."""
    r = np.random.default_rng(seed)
    fmax = np.finfo(np.float32).max
    tiny = np.finfo(np.float32).tiny
    pool = np.array([0.0, -0.0, tiny * 0.5, -tiny * 0.25, tiny * 2 ** -20, np.inf, -np.inf, fmax, -fmax, fmax * 0.75,
                     1.0, -2.0, 1e-38, -1e-38], np.float32)
    parts = pool[r.integers(0, len(pool), (world, n))]
    if world >= 2:
        # a few fixed patterns at the front: -0 + -0, -0 + 0, inf + -inf, max + max, subnormal + subnormal
        pats = [(-0.0, -0.0), (-0.0, 0.0), (np.inf, -np.inf), (fmax, fmax), (tiny * 0.5, tiny * 0.25),
                (tiny * 0.5, -tiny * 0.5)]
        for i, (a, b) in enumerate(pats[:n]):
            parts[:, i] = -0.0                   # x + -0 = x for every x, -0 and +0 included
            parts[0, i], parts[1, i] = a, b
    return list(parts.astype(np.float32))


def random_parts(world, n, seed):
    r = np.random.default_rng(seed)
    return list((r.standard_normal((world, n)) * (1 + np.arange(world))[:, None]).astype(np.float32))


# ---- rank order ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("world", [3, 4, 8, 16])
def test_sum_is_the_rank_ordered_float32_sum_bit_for_bit(world):
    n = 4 * 1031 + 3
    parts = order_sensitive(world, n, seed=world)
    want = seq_sum(parts)
    # the yardstick tells the orders apart: a kernel that summed in another order would fail here
    assert (seq_sum(parts[::-1]) != want).sum() > n // 20
    assert (pair_sum(parts) != want).sum() > n // 20
    pk = Peers(parts)
    for rank in range(world):
        got = pk.reduce_as(rank, epoch=1 + rank)
        assert same_bits(got, want), f"world {world}, rank {rank}: {int((got != want).sum())} elements differ"


@pytest.mark.parametrize("world", [2, 3, 16])
def test_signed_zeros_subnormals_infinities_and_overflow(world):
    n = 4 * 300 + 3
    parts = specials(world, n, seed=40 + world)
    want = seq_sum(parts)
    assert np.isnan(want).any() and np.isinf(want).any()
    assert (want == 0).any() and np.signbit(want[want == 0]).any() and (~np.signbit(want[want == 0])).any()
    sub = (want != 0) & (np.abs(want) < np.finfo(np.float32).tiny)
    assert sub.any(), "no subnormal result in the case"
    pk = Peers(parts)
    for rank in range(world):
        assert same_bits(pk.reduce_as(rank, epoch=7), want), f"world {world}, rank {rank}"


# ---- world sizes and lengths --------------------------------------------------------------------------------------------
def _lengths():
    """Small lengths (float4 lanes and the scalar tail), one CTA's float4 span (256 x 4 floats) and around it, and the
    grid cap: n / 4 > SMs x 256 forces grid-stride iterations (read from the device)."""
    span = 256 * 4
    grid = _sms() * span
    return [0, 1, 2, 3, 4, 5, 7, span - 1, span, span + 1, span + 3, span + 4, 2 * span + 2,
            grid + 3, 3 * grid + 4 + 1, 3 * grid + 4 * 77]


@pytest.mark.parametrize("world", [1, 2, 3, 8, 15, 16])
def test_every_world_size_rank_and_length(world):
    lengths = _lengths()
    assert any(n % 4 for n in lengths if n >= 4 * 256 * _sms())     # a grid-stride case with a tail
    for n in lengths:
        parts = random_parts(world, n, seed=1000 * world + n)
        if world == 1 and n:
            # NaN payloads and signalling NaNs survive: at world 1 the kernel only loads and stores
            payloads = np.array([0x7FC12345, 0xFFA00001, 0x7F800001, 0xFFFFFFFF], np.uint32).view(np.float32)
            parts[0][:min(n, 4)] = payloads[:min(n, 4)]
            parts[0][-1] = payloads[(n - 1) % 4]
        want = seq_sum(parts)
        pk = Peers(parts)
        for rank in range(world):
            got = pk.reduce_as(rank, epoch=3 + rank, ahead=set(range(0, world, 2)))
            if world == 1:
                assert np.array_equal(got.view(np.uint32), parts[0].view(np.uint32)), f"n {n}: not a bit copy"
            else:
                assert same_bits(got, want), f"world {world}, rank {rank}, n {n}"


def test_a_long_buffer_at_world_2():
    n = 2 ** 25 + 3
    parts = random_parts(2, n, seed=5)
    want = parts[0] + parts[1]
    pk = Peers(parts)
    for rank in (0, 1):
        assert same_bits(pk.reduce_as(rank, epoch=11), want), f"rank {rank}"


# ---- epochs -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("epoch", [1, 2 ** 31 - 1, 2 ** 31, 2 ** 32 - 1, 0])
def test_the_epoch_wraps_like_the_reducer_counter(epoch):
    """PeerReducer passes epoch & 0xFFFFFFFF: the wait must hold across 2^31 (signed difference) and 2^32 (wrap),
    with flags at the epoch or one ahead of it."""
    world, n = 3, 4 * 500 + 1
    parts = order_sensitive(world, n, seed=epoch & 0xFFFF)
    want = seq_sum(parts)
    pk = Peers(parts)
    for rank in range(world):
        for ahead in ((), {0, 1, 2}, {rank}):
            assert same_bits(pk.reduce_as(rank, epoch, ahead), want), f"epoch {epoch}, rank {rank}, ahead {ahead}"


# ---- refusals -----------------------------------------------------------------------------------------------------------
def test_refusals_leave_the_output_untouched():
    world, n = 3, 64
    pk = Peers(random_parts(world, n, seed=9))
    for rank in range(world):
        pk.arm(rank, 1)
    flags0 = pk.flags_host()
    good = [b.data_ptr() for b in pk.bufs]
    cases = {
        "world 0": dict(world=0, rank=0),
        f"world {MAX_PEERS + 1}": dict(world=MAX_PEERS + 1, rank=0),
        "rank -1": dict(rank=-1),
        "rank = world": dict(rank=world),
        "n -1": dict(n=-1),
        "null out": dict(out=0),
        "null status": dict(status=0),
        "null peer buffer": dict(bufs=[good[0], None, good[2]]),
        "null flag array": dict(flags=[pk.flags[0].data_ptr(), pk.flags[1].data_ptr(), None]),
        "misaligned buffer": dict(bufs=[good[0], good[1] + 4, good[2]]),
        "misaligned out": dict(out=pk.out.data_ptr() + 4),
    }
    for label, kw in cases.items():
        kw = dict(kw)
        rank = kw.pop("rank", 0)
        pk.out.fill_(float(SENTINEL))
        torch.cuda.synchronize()
        rc = pk.call(rank, 1, **kw)
        torch.cuda.synchronize()
        assert rc == ERR_INVALID, f"{label}: returned {rc}"
        assert np.all(pk.out.cpu().numpy() == SENTINEL), f"{label}: out was written"
        assert int(pk.status.item()) == 0, label
        assert np.array_equal(pk.flags_host(), flags0), f"{label}: a flag was written"
