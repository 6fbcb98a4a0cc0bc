"""The sm_90a data-movement kernels one launch at a time, at launch shapes chosen here, against a host reference.

The engine picks every launch shape for itself, so the suite's end-to-end tests only reach the shapes the default
options produce.  These tests drive the CUDA backend directly through tests/gpu_kernels/libsw_kernels_test.so (flat
C wrappers over gpu_cuda.cu, built by `make probe`) and check:

- the TMA bulk copy through each entry point (inline segment list, pinned segment list, balanced jobs) at
  stages 2 / 3 / 8 and stage sizes from 1 KiB to the shared-memory limit, and the SIMT copy in each alignment class;
- the bulk reductions (TMA and element-wise) of every element type on signed zeros, subnormals, infinities, NaN,
  overflow and integer wrap-around, against the exact sum rounded once to nearest-even;
- the put kernels' slot headers, payloads and RTS bodies on both sides of the inline-launch limits;
- the resident pull kernel serving published batches: tails, empty chunks, chunk-size clamps and the slot ring.

Every destination sits between bands of 0xEE that must come back untouched.  Every wait is bounded."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "tests", "gpu_kernels", "libsw_kernels_test.so")
WAIT_S = 30.0    # a launch here takes milliseconds; a wait that runs out is a failure, not a hang
CANARY = 0xEE
BAND = 4096      # canary bytes before the first and after the last destination of a buffer

# slot layout of the inbound ring (sw_device.h): the header words the matcher trusts, then the payload
SLOT_BYTES, SLOT_HDR, SLOT_MAGIC = 8192, 64, 0x53574D47
KIND_EAGER, KIND_RTS = 1, 2
# element types of a reduction (SW_DTYPE_* in include/starway_b200.h)
DTYPES = {"float32": 1, "float16": 2, "bfloat16": 3, "float64": 4, "int32": 5, "int64": 6}
ITEMSIZE = {"float32": 4, "float16": 2, "bfloat16": 2, "float64": 8, "int32": 4, "int64": 8}


# ---------------------------------------------------------------------------------------------------- plumbing
class Shim:
    def __init__(self, path):
        lib = ctypes.CDLL(path)
        vp, u32, u64, i32, sz = ctypes.c_void_p, ctypes.c_uint32, ctypes.c_uint64, ctypes.c_int, ctypes.c_size_t
        sigs = {
            "swk_init": (i32, [i32]),
            "swk_last_error": (ctypes.c_char_p, []),
            "swk_bulk_smem_limit": (i32, []),
            "swk_pull_default_ctas": (i32, []),
            "swk_pull_jobs": (i32, []),
            "swk_pull_slots": (i32, []),
            "swk_host_alloc": (vp, [sz]),
            "swk_host_free": (i32, [vp]),
            "swk_stream_create": (vp, []),
            "swk_stream_destroy": (i32, [vp]),
            "swk_wait": (i32, [vp, ctypes.c_double]),
            "swk_launch_bulk": (i32, [vp, vp, vp, vp, u32, vp, sz, i32, i32, i32, i32, i32]),
            "swk_launch_reduce": (i32, [vp, vp, vp, vp, u32, vp, sz, i32, i32, i32, i32, i32]),
            "swk_launch_put": (i32, [vp, vp, vp, vp, vp, vp, vp, vp, u32, vp, sz, vp, u64]),
            "swk_pull_create": (vp, [u32]),
            "swk_pull_launch": (i32, [vp, vp, u32, i32, i32, u32, u32]),
            "swk_pull_publish": (i32, [vp, vp, vp, vp, vp, u32, u32]),
            "swk_pull_stop": (None, [vp]),
            "swk_pull_stats": (i32, [vp, vp]),
            "swk_pull_destroy": (i32, [vp]),
        }
        for name, (res, args) in sigs.items():
            fn = getattr(lib, name)
            fn.restype, fn.argtypes = res, args
        self.lib = lib

    def __getattr__(self, name):
        return getattr(self.lib, "swk_" + name)

    def error(self):
        return (self.lib.swk_last_error() or b"").decode()


def ptr(a):
    """Address of a contiguous NumPy array (kept alive by the caller)."""
    assert a.flags["C_CONTIGUOUS"]
    return a.ctypes.data


def u64s(values):
    return np.ascontiguousarray(np.asarray(values, dtype=np.uint64))


@pytest.fixture(scope="module")
def torch():
    import torch

    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    torch.cuda.init()
    return torch


@pytest.fixture(scope="module")
def shim(torch):
    if not os.path.exists(LIB):
        subprocess.check_call(["make", "-C", ROOT, "-j", "8", "probe"])
    s = Shim(LIB)
    assert s.init(torch.cuda.current_device()) == 0, s.error()
    return s


@pytest.fixture(scope="module")
def stream(shim):
    st = shim.stream_create()
    assert st, shim.error()
    yield st
    if shim.wait(st, WAIT_S) == 0:
        shim.stream_destroy(st)


class Pinned:
    """Page-locked, device-mapped host memory from the backend's allocator."""

    def __init__(self, shim, nbytes):
        self.nbytes = nbytes
        self.addr = shim.host_alloc(nbytes)
        assert self.addr, shim.error()

    def view(self, dtype=np.uint8):
        return np.frombuffer((ctypes.c_uint8 * self.nbytes).from_address(self.addr), dtype=dtype)


@pytest.fixture(scope="module")
def pinned(shim, stream):
    p = Pinned(shim, 4 << 20)   # segment lists and put descriptors: the kernels read them from here
    yield p
    if shim.wait(stream, WAIT_S) == 0:
        shim.host_free(p.addr)


def run_launch(shim, stream, torch, launch):
    """Every buffer torch wrote is complete before the launch; the launch has completed when this returns."""
    torch.cuda.synchronize()
    r = launch()
    assert r >= 0, f"launch failed: {shim.error()}"
    w = shim.wait(stream, WAIT_S)
    assert w == 0, f"wait returned {w}: {shim.error()}"
    return r


def to_device(torch, host_bytes):
    return torch.from_numpy(np.ascontiguousarray(host_bytes)).cuda()


def canary_buffer(torch, nbytes):
    return torch.full((nbytes,), CANARY, dtype=torch.uint8, device="cuda")


def assert_bytes_equal(got, want, what):
    if np.array_equal(got, want):
        return
    bad = np.flatnonzero(got != want)
    i = int(bad[0])
    raise AssertionError(f"{what}: {bad.size} byte(s) differ, first at offset {i}: got {got[i]:#04x}, want "
                         f"{want[i]:#04x} (bytes {got[i:i + 8].tolist()} vs {want[i:i + 8].tolist()})")


@pytest.fixture(scope="module")
def src_pool(torch):
    """48 MiB of random bytes, on the device and on the host."""
    host = np.random.default_rng(0x5EED).integers(0, 256, 48 << 20, dtype=np.uint8)
    return host, to_device(torch, host)


# ---------------------------------------------------------------------------------------------------- bulk copy
def place(lengths, pieces=None, src_align=16, dst_align=16, src_skew=None, dst_skew=None, gap=48):
    """Lay jobs out in a source pool and a destination buffer with a gap of canary bytes between destinations.
    `pieces[j]` cuts job j into that many segments, contiguous in source and destination (16-byte multiples).
    Returns (segments as (src_off, dst_off, len), jobs as (src_off, dst_off, len), destination size)."""
    segs, jobs = [], []
    s_cur, d_cur = 0, BAND
    for j, n in enumerate(lengths):
        s_cur = -(-s_cur // src_align) * src_align + (src_skew(j) if src_skew else 0)
        d_cur = -(-d_cur // dst_align) * dst_align + (dst_skew(j) if dst_skew else 0)
        jobs.append((s_cur, d_cur, n))
        k = pieces[j] if pieces else 1
        cuts = sorted({0, n} | {(n * i // k) & ~15 for i in range(1, k)})
        for a, b in zip(cuts, cuts[1:]):
            segs.append((s_cur + a, d_cur + a, b - a))
        s_cur += n + gap + 16 * (j % 3)
        d_cur += n + gap + 16 * (j % 5)
    return segs, jobs, d_cur + BAND


def run_copy(shim, stream, pinned, torch, src_pool, segs, jobs, dst_size, mode, stages=8, stage_bytes=24576,
             ctas_per_sm=1, balance=0):
    host_src, dev_src = src_pool
    assert max(s + n for s, _, n in jobs) <= host_src.size
    dst = canary_buffer(torch, dst_size)
    base_s, base_d = dev_src.data_ptr(), dst.data_ptr()
    src = u64s([base_s + s for s, _, _ in segs])
    dsts = u64s([base_d + d for _, d, _ in segs])
    lens = u64s([n for _, _, n in segs])
    run_launch(shim, stream, torch, lambda: shim.launch_bulk(stream, ptr(src), ptr(dsts), ptr(lens), len(segs), pinned.addr,
                                                             pinned.nbytes, mode, stages, stage_bytes, ctas_per_sm, balance))
    want = np.full(dst_size, CANARY, dtype=np.uint8)
    for s, d, n in jobs:
        want[d:d + n] = host_src[s:s + n]
    assert_bytes_equal(dst.cpu().numpy(), want, "bulk copy destination")


def stage_sizes(shim):
    return {"1k": lambda stages: 1024, "24k": lambda stages: 24576,
            "max": lambda stages: (shim.bulk_smem_limit() // stages) & ~15}


def tma_lengths(sb, count):
    """16, stage_bytes +- 16, whole multiples of stage_bytes, and two segments of several MiB."""
    cycle = [16, sb - 16, sb + 16, sb, 2 * sb, 3 * sb, sb + 32, 48]
    out = [cycle[i % len(cycle)] for i in range(count)]
    out[count // 3] = (3 << 20) + 16
    out[2 * count // 3] = 5 << 20
    return out


@pytest.mark.parametrize("stage_size", ["1k", "24k", "max"])
@pytest.mark.parametrize("stages", [2, 3, 8])
@pytest.mark.parametrize("entry", ["inline_96_segments", "list_97_segments", "balanced_96_jobs", "balanced_97_jobs"])
def test_bulk_tma_copy_entry_points(shim, stream, pinned, torch, src_pool, entry, stages, stage_size):
    """Each TMA entry point at each pipeline depth (stages 2 is a look-ahead of 0) and stage size.
    inline: <= 96 segments travel as kernel parameters; list: 97 segments are read from pinned memory; balanced:
    contiguous segments merge into <= 96 jobs that every CTA splits by byte range, 97 jobs fall back to the list."""
    sb = stage_sizes(shim)[stage_size](stages)
    njobs = 97 if "97" in entry else 96
    balanced = entry.startswith("balanced")
    lengths = tma_lengths(sb, njobs)
    pieces = [1 + (j % 3) for j in range(njobs)] if balanced else None
    segs, jobs, size = place(lengths, pieces)
    if balanced:
        assert len(segs) > 96   # only the merge into jobs keeps this launch off the segment-list kernel
    run_copy(shim, stream, pinned, torch, src_pool, segs, jobs, size, mode=0, stages=stages, stage_bytes=sb,
             balance=int(balanced))


def test_bulk_tma_copy_many_segments_per_cta(shim, stream, pinned, torch, src_pool):
    """More segments than CTAs: each CTA walks several segments, zero-length ones among them."""
    n = 3000
    lengths = [(16 * (1 + (j * 37) % 700)) if j % 11 else 0 for j in range(n)]
    segs, jobs, size = place(lengths)
    run_copy(shim, stream, pinned, torch, src_pool, segs, jobs, size, mode=0, stages=4, stage_bytes=4096, ctas_per_sm=2)


@pytest.mark.parametrize("align", ["mutual_16", "mutual_4", "unaligned"])
def test_bulk_simt_copy_alignment_classes(shim, stream, pinned, torch, src_pool, align):
    """The SIMT copy in each alignment class of (src ^ dst): 16-byte vectors, 4-byte words, bytes.  Lengths 1..33 at
    every source misalignment (head bytes larger than the length among them), then bodies long enough for the
    unrolled loop, each with a tail."""
    flip = {"mutual_16": lambda j: 0, "mutual_4": lambda j: 4 * (1 + j % 3), "unaligned": lambda j: 1 + j % 3}[align]
    lengths = list(range(1, 34)) + [1000 + 7, 4096 * 3 + 5, 70000 + 3, (1 << 20) + 9, (2 << 20) + 15]
    segs, jobs, size = place(lengths, src_align=16, dst_align=16, src_skew=lambda j: j % 16,
                             dst_skew=lambda j: (j % 16) ^ flip(j), gap=40)
    for s, d, _ in segs:
        cls = (s ^ d) & 15
        assert {"mutual_16": cls == 0, "mutual_4": cls != 0 and cls & 3 == 0, "unaligned": cls & 3 != 0}[align]
    run_copy(shim, stream, pinned, torch, src_pool, segs, jobs, size, mode=1, ctas_per_sm=4)


@pytest.mark.parametrize("stages", [2, 8])
def test_tma_tuning_beyond_shared_memory_is_refused(shim, stream, pinned, torch, src_pool, stages):
    """A tuning whose stages need more shared memory than a CTA may have: launch_bulk and launch_reduce return -1
    and launch nothing."""
    limit = shim.bulk_smem_limit()
    assert limit > 200 * 1024, limit   # H100: 227 KiB opt-in per block, less the static mbarriers
    sb = ((limit // stages) & ~15) + 16
    segs, jobs, size = place([sb, 4096])
    dst = canary_buffer(torch, size)
    src = u64s([src_pool[1].data_ptr() + s for s, _, _ in segs])
    dsts = u64s([dst.data_ptr() + d for _, d, _ in segs])
    lens = u64s([n for _, _, n in segs])
    torch.cuda.synchronize()
    args = (stream, ptr(src), ptr(dsts), ptr(lens), len(segs), pinned.addr, pinned.nbytes)
    for balance in (0, 1):
        assert shim.launch_bulk(*args, 0, stages, sb, 1, balance) == -1
        assert "shared memory" in shim.error()
    assert shim.launch_reduce(*args, DTYPES["int32"], 0, stages, sb, 1) == -1
    assert "shared memory" in shim.error()
    assert shim.wait(stream, WAIT_S) == 0
    assert (dst.cpu().numpy() == CANARY).all()


# ---------------------------------------------------------------------------------------------------- reduce
BITS = {2: np.uint16, 4: np.uint32, 8: np.uint64}


def bf16_to_f64(bits):
    return (bits.astype(np.uint32) << 16).view(np.float32).astype(np.float64)


def f64_to_bf16(x):
    """Round to nearest even, through float32: the float32 rounding of a sum of two bfloat16 values is never a
    bfloat16 tie it was not already, so the two roundings give the once-rounded result."""
    u = x.astype(np.float32).view(np.uint32).astype(np.uint64)
    r = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)
    return np.where(np.isnan(x), np.uint16(0x7FC0), r)


def as_f64(name, bits):
    if name == "bfloat16":
        return bf16_to_f64(bits)
    return bits.view(name).astype(np.float64)


def from_f64(name, x):
    """The exact float64 sum rounded once to the element type (float64: numpy's own add already is that)."""
    if name == "bfloat16":
        return f64_to_bf16(x)
    return x.astype(name).view(BITS[ITEMSIZE[name]])


def reference_sum(name, a_bits, b_bits):
    """Bit patterns of a + b in `name`, and where the reference is NaN."""
    if name in ("int32", "int64"):
        u = np.uint32 if name == "int32" else np.uint64
        s = a_bits.view(u) + b_bits.view(u)   # modular: wraps like two's complement hardware
        return s.view(BITS[ITEMSIZE[name]]), np.zeros(s.size, dtype=bool)
    with np.errstate(all="ignore"):
        if name == "float64":
            x = a_bits.view(np.float64) + b_bits.view(np.float64)   # exact sum rounded once to float64
        else:
            # exact in float64 for float16; for float32 / bfloat16 the float64 rounding is innocuous (53 >= 2p + 2)
            x = as_f64(name, a_bits) + as_f64(name, b_bits)
        return from_f64(name, x), np.isnan(x)


def float_params(name):
    """(largest finite, smallest normal, smallest subnormal, machine epsilon) as float64."""
    if name == "bfloat16":
        return float(bf16_to_f64(np.array([0x7F7F], np.uint16))[0]), 2.0 ** -126, 2.0 ** -133, 2.0 ** -7
    fi = np.finfo(name)
    return float(fi.max), float(fi.tiny), float(fi.smallest_subnormal), float(fi.eps)


def special_pairs(name):
    """(dst, src) pairs at the edges of the type, as float64 values the type represents exactly (or integers)."""
    if name in ("int32", "int64"):
        bits = 32 if name == "int32" else 64
        hi, lo = (1 << (bits - 1)) - 1, -(1 << (bits - 1))
        return [(hi, 1), (1, hi), (hi, hi), (lo, -1), (lo, lo), (lo, hi), (-1, 1), (0, lo), (hi, lo), (-1, -1),
                (hi - 5, 10), (lo + 5, -10), (0, 0)]
    inf, nan = float("inf"), float("nan")
    big, tiny, sub, eps = float_params(name)
    top_half_ulp = big * eps / (2 - eps) / 2   # half the spacing of the largest binade
    pairs = [
        (0.0, 0.0), (0.0, -0.0), (-0.0, 0.0), (-0.0, -0.0),                          # signed zeros
        (sub, 0.0), (0.0, -sub), (sub, sub), (-sub, -sub), (sub, -sub), (-sub, sub),  # subnormals
        (tiny - sub, sub), (tiny, -sub), (-tiny, sub), (tiny - sub, tiny - sub), (3 * sub, -0.0), (tiny / 2, tiny / 4),
        (inf, 1.0), (-inf, 1.0), (inf, inf), (-inf, -inf), (inf, -inf), (-inf, inf), (inf, -big), (big, inf),
        (nan, 1.0), (1.0, nan), (nan, inf), (-inf, nan), (nan, nan),
        (big, big), (-big, -big), (big, -big), (big, top_half_ulp), (-big, -top_half_ulp),  # ties at the top: to inf
        (big, top_half_ulp / 2), (big - 2 * top_half_ulp, top_half_ulp),                    # stay finite / tie to even
        (1.0, eps / 2), (1.0 + eps, eps / 2), (1.0, eps * 0.75), (-1.0, -eps / 2), (1.0, -eps / 4),  # rounding of ties
    ]
    if name == "float16":   # sums past 65504
        pairs += [(65504.0, 16.0), (65504.0, 8.0), (60000.0, 6000.0), (-65504.0, -32.0), (65504.0, 65504.0),
                  (32768.0, 32768.0), (65504.0, -65504.0), (65504.0, 15.0)]
    return pairs


def encode(name, values):
    if name in ("int32", "int64"):
        return np.array([v & ((1 << (8 * ITEMSIZE[name])) - 1) for v in values], dtype=BITS[ITEMSIZE[name]])
    x = np.array(values, dtype=np.float64)
    bits = from_f64(name, x)
    if name != "float64":
        back = as_f64(name, bits)
        ok = (back == x) | (np.isnan(back) & np.isnan(x))
        assert ok.all(), f"{name}: value not representable: {x[~ok]}"
    return bits


def random_operands(name, n, rng):
    """Random bit patterns (every class of value) and random values of nearby magnitude (rounding decides)."""
    w = ITEMSIZE[name]
    raw = rng.integers(0, 1 << (8 * w), size=(2, n), dtype=np.uint64 if w == 8 else np.int64).astype(BITS[w])
    if name in ("int32", "int64"):
        return raw[0], raw[1]
    m = rng.standard_normal((2, n)) * np.exp2(rng.integers(-4, 5, size=(2, n)))
    near = [from_f64(name, m[i]) for i in range(2)]
    return np.concatenate([raw[0], near[0]]), np.concatenate([raw[1], near[1]])


def reduce_segments(name, mode, nelem):
    """Element counts per segment (a 16-byte multiple in TMA mode) and the source byte skew of each."""
    w = ITEMSIZE[name]
    if mode == 0:
        unit = 16 // w
        sched = [unit, 2 * unit, 64 * unit, 3 * unit, (4096 + 16) // w, (65536 + 48) // w, 5 * unit]
    else:
        sched = [1, 3, 7, 16 // w + 1, 1000 + 1, 33, (65536 + 2 * w) // w, 2]
    counts, used, i = [], 0, 0
    while used < nelem:
        c = min(sched[i % len(sched)], nelem - used)
        counts.append(c)
        used += c
        i += 1
    # SIMT reads a source at any byte offset: skew every other one; TMA sources stay 16-byte aligned
    skews = [(0 if mode == 0 or j % 2 == 0 else 1 + 2 * (j % 7)) for j in range(len(counts))]
    return counts, skews


def run_reduce(shim, stream, pinned, torch, name, mode, a_bits, b_bits, counts, skews, dst_gap, stages=3,
               stage_bytes=2048):
    """Reduce b into a, segment by segment; returns (got, want) element bits and the NaN mask, after checking every
    byte between and around the destinations."""
    w = ITEMSIZE[name]
    src_img = np.random.default_rng(7).integers(0, 256, a_bits.size * w + 64 * len(counts) + 256, dtype=np.uint8)
    dst_size = BAND + a_bits.size * w + dst_gap * len(counts) + 16 * len(counts) + BAND
    dst_img = np.full(dst_size, CANARY, dtype=np.uint8)
    segs, spans = [], []
    s_cur, d_cur, e = 0, BAND, 0
    for c, skew in zip(counts, skews):
        s_cur = -(-s_cur // 16) * 16 + skew
        d_cur = -(-d_cur // (16 if mode == 0 else w)) * (16 if mode == 0 else w)
        src_img[s_cur:s_cur + c * w] = b_bits[e:e + c].view(np.uint8)
        dst_img[d_cur:d_cur + c * w] = a_bits[e:e + c].view(np.uint8)
        segs.append((s_cur, d_cur, c * w))
        spans.append((d_cur, e, c))
        s_cur += c * w + 16
        d_cur += c * w + dst_gap
        e += c
    src, dst = to_device(torch, src_img), to_device(torch, dst_img)
    sp = u64s([src.data_ptr() + s for s, _, _ in segs])
    dp = u64s([dst.data_ptr() + d for _, d, _ in segs])
    ln = u64s([n for _, _, n in segs])
    run_launch(shim, stream, torch, lambda: shim.launch_reduce(stream, ptr(sp), ptr(dp), ptr(ln), len(segs), pinned.addr,
                                                               pinned.nbytes, DTYPES[name], mode, stages, stage_bytes, 4))
    got_img = dst.cpu().numpy()
    want_bits, nan = reference_sum(name, a_bits, b_bits)
    want_img = dst_img.copy()
    got_bits = np.empty_like(want_bits)
    for d, e0, c in spans:
        want_img[d:d + c * w] = want_bits[e0:e0 + c].view(np.uint8)
        got_bits[e0:e0 + c] = got_img[d:d + c * w].view(BITS[w])
    # outside the destinations: nothing written
    outside = np.ones(dst_size, dtype=bool)
    for d, _, c in spans:
        outside[d:d + c * w] = False
    assert_bytes_equal(got_img[outside], want_img[outside], "bytes around the reduce destinations")
    return got_bits, want_bits, nan


def describe(a, b, got, want, idx):
    rows = []
    for i in idx[:8]:
        rows.append(f"  [{i}] {int(a[i]):#x} + {int(b[i]):#x}: got {int(got[i]):#x}, want {int(want[i]):#x}")
    return "\n".join(rows)


def is_nan_bits(name, bits):
    if name == "bfloat16":
        return np.isnan(bf16_to_f64(bits))
    return np.isnan(bits.view(name))


@pytest.mark.parametrize("mode", [0, 1], ids=["tma", "simt"])
@pytest.mark.parametrize("name", list(DTYPES))
def test_reduce_matches_the_rounded_exact_sum(shim, stream, pinned, torch, name, mode):
    """dst += src for every element type on both kernels, bit for bit against the exact sum rounded once to
    nearest-even (integers: modulo 2^bits).  Signed zeros, subnormals, infinities, NaN (any NaN where the reference
    is NaN), sums past the largest finite value, and random operands where the rounding decides."""
    rng = np.random.default_rng(DTYPES[name] * 10 + mode)
    pairs = special_pairs(name)
    sa, sb = encode(name, [p[0] for p in pairs]), encode(name, [p[1] for p in pairs])
    ra, rb = random_operands(name, 20000, rng)
    a_bits, b_bits = np.concatenate([sa, sb, ra]), np.concatenate([sb, sa, rb])   # every special pair both ways
    pad = -a_bits.size % 8                                                         # whole 16-byte TMA segments
    a_bits, b_bits = np.concatenate([a_bits, ra[:pad]]), np.concatenate([b_bits, rb[:pad]])
    counts, skews = reduce_segments(name, mode, a_bits.size)
    got, want, nan = run_reduce(shim, stream, pinned, torch, name, mode, a_bits, b_bits, counts, skews, dst_gap=48)
    exact = ~nan
    bad = np.flatnonzero(exact & (got != want))
    assert bad.size == 0, f"{name} {bad.size} sums differ:\n" + describe(a_bits, b_bits, got, want, bad)
    bad = np.flatnonzero(nan & ~is_nan_bits(name, got))
    assert bad.size == 0, f"{name}: {bad.size} sums should be NaN:\n" + describe(a_bits, b_bits, got, want, bad)


@pytest.mark.parametrize("mode", [0, 1], ids=["tma", "simt"])
@pytest.mark.parametrize("name", list(DTYPES))
def test_reduce_overlapping_destinations_in_one_launch(shim, stream, pinned, torch, name, mode):
    """64 segments of one launch add into the same 1 MiB destination, and two more overlap each other at a 16-byte
    offset.  Integer-valued operands keep every partial sum exact, so the result does not depend on the order the
    memory system applies the adds in."""
    w = ITEMSIZE[name]
    n = (1 << 20) // w
    span = {"bfloat16": 2, "float16": 15}.get(name, 1000)   # |any partial sum| <= 65 * span stays exact
    rng = np.random.default_rng(100 + DTYPES[name] * 2 + mode)
    step = 48 // w                                            # source k starts 48 bytes after source k - 1
    pool_vals = rng.integers(-span, span + 1, n + 64 * step + 16 // w)
    init_vals = rng.integers(-span, span + 1, n)
    off_vals = rng.integers(-span, span + 1, (2, 4096))       # the pair of segments 16 bytes apart

    def bits(v):
        return encode(name, v.tolist()) if name == "bfloat16" else (
            v.astype(name).view(BITS[w]) if name.startswith("float") else v.astype(np.int64).astype(name).view(BITS[w]))

    pool, init, offs = bits(pool_vals), bits(init_vals), [bits(off_vals[0]), bits(off_vals[1])]
    src = to_device(torch, np.concatenate([pool, offs[0], offs[1]]).view(np.uint8))
    region2 = BAND + n * w + 64                                 # second destination, after the 1 MiB one
    dst_size = region2 + 4096 * w + 16 + BAND
    dst_img = np.full(dst_size, CANARY, dtype=np.uint8)
    dst_img[BAND:BAND + n * w] = init.view(np.uint8)
    dst_img[region2:region2 + 4096 * w + 16] = 0
    dst = to_device(torch, dst_img)
    pool_bytes = pool.size * w
    segs = [(k * 48, BAND, n * w) for k in range(64)]
    segs += [(pool_bytes, region2, 4096 * w), (pool_bytes + 4096 * w, region2 + 16, 4096 * w)]
    sp = u64s([src.data_ptr() + s for s, _, _ in segs])
    dp = u64s([dst.data_ptr() + d for _, d, _ in segs])
    ln = u64s([c for _, _, c in segs])
    run_launch(shim, stream, torch, lambda: shim.launch_reduce(stream, ptr(sp), ptr(dp), ptr(ln), len(segs), pinned.addr,
                                                               pinned.nbytes, DTYPES[name], mode, 8, 24576, 1))
    total = init_vals.astype(np.int64).copy()
    for k in range(64):
        total += pool_vals[k * step:k * step + n]
    two = np.zeros(4096 + 16 // w, dtype=np.int64)
    two[:4096] += off_vals[0]
    two[16 // w:] += off_vals[1]
    want = dst_img.copy()
    want[BAND:BAND + n * w] = bits(total).view(np.uint8)
    want[region2:region2 + 4096 * w + 16] = bits(two).view(np.uint8)
    assert_bytes_equal(dst.cpu().numpy(), want, f"{name} overlapping reductions")


# ---------------------------------------------------------------------------------------------------- put
PUT_LENGTHS = [0, 1, 15, 16, 8127, 8128]


def put_cases():
    out = []
    for n in (1, 31, 32, 33, 200):
        for rts in (0, 1, 16, 17):
            if rts <= n and (rts != 1 or n == 1):
                out.append(pytest.param(n, rts, id=f"n{n}-rts{rts}"))
    return out


@pytest.mark.parametrize("n,n_rts", put_cases())
def test_put_writes_header_and_payload_of_every_slot(shim, stream, pinned, torch, src_pool, n, n_rts):
    """Eager and RTS puts into the slots of a ring: the header words the matcher trusts (tag, length, seq,
    magic << 32 | kind) exactly, the payload or the 128-byte RTS body, and nothing else in the slot.  n <= 32 with
    <= 16 RTS takes the single-CTA kernel with descriptors as parameters, which also writes the done flag."""
    host_src, dev_src = src_pool
    rng = np.random.default_rng(n * 100 + n_rts)
    ring = canary_buffer(torch, (n + 2) * SLOT_BYTES)        # a canary slot before and after
    order = rng.permutation(n) + 1                           # message i lands in slot order[i]
    is_rts = np.zeros(n, dtype=np.uint8)
    is_rts[rng.choice(n, n_rts, replace=False)] = 1
    bodies = Pinned(shim, max(1, n_rts) * 128)
    body_bytes = rng.integers(0, 256, max(1, n_rts) * 128, dtype=np.uint8)
    bodies.view()[:] = body_bytes
    flag = Pinned(shim, 64)
    try:
        src, dst, tag, seq, lens, msg_len, expect = [], [], [], [], [], [], []
        r = 0
        for i in range(n):
            slot = ring.data_ptr() + int(order[i]) * SLOT_BYTES
            t = int(rng.integers(0, 1 << 63)) << 1 | (i & 1)
            sq = (1 << 40) + 3 * i + 1
            if is_rts[i]:
                src.append(bodies.addr + 128 * r)
                lens.append(128)
                ml = int(rng.integers(8129, 1 << 34))
                expect.append(("rts", r))
                r += 1
            else:
                ln = PUT_LENGTHS[i % len(PUT_LENGTHS)]
                off = 1 + 2 * int(rng.integers(0, 1 << 20)) if i % 4 else 16 * int(rng.integers(0, 1 << 16))
                src.append(dev_src.data_ptr() + off)
                lens.append(ln)
                ml = ln
                expect.append(("eager", off))
            dst.append(slot)
            tag.append(t)
            seq.append(sq)
            msg_len.append(ml)
        a_src, a_dst, a_tag, a_seq, a_ml = u64s(src), u64s(dst), u64s(tag), u64s(seq), u64s(msg_len)
        a_len = np.ascontiguousarray(np.array(lens, dtype=np.uint32))
        done_value = 0xD0E0_0000_0000_0000 | (n << 8) | n_rts
        ret = run_launch(shim, stream, torch, lambda: shim.launch_put(
            stream, ptr(a_src), ptr(a_dst), ptr(a_tag), ptr(a_seq), ptr(a_len), ptr(is_rts), ptr(a_ml), n, pinned.addr,
            pinned.nbytes, flag.addr, done_value))
        inline = n <= 32 and n_rts <= 16
        assert ret == (1 if inline else 0)
        assert int(flag.view(np.uint64)[0]) == (done_value if inline else 0)

        img = ring.cpu().numpy()
        for k in (0, n + 1):
            assert (img[k * SLOT_BYTES:(k + 1) * SLOT_BYTES] == CANARY).all(), f"canary slot {k} written"
        for i in range(n):
            s = img[int(order[i]) * SLOT_BYTES:(int(order[i]) + 1) * SLOT_BYTES]
            words = s[:32].view(np.uint64)
            kind = KIND_RTS if is_rts[i] else KIND_EAGER
            assert words.tolist() == [tag[i], msg_len[i], seq[i], (SLOT_MAGIC << 32) | kind], f"header of message {i}"
            assert (s[32:SLOT_HDR] == CANARY).all(), f"header padding of message {i}"
            what, where = expect[i]
            if what == "rts":
                body = body_bytes[128 * where:128 * where + 128]
            else:
                body = host_src[where:where + lens[i]]
            assert_bytes_equal(s[SLOT_HDR:SLOT_HDR + body.size], body, f"payload of message {i} ({what}, {lens[i]} B)")
            assert (s[SLOT_HDR + body.size:] == CANARY).all(), f"bytes after the payload of message {i}"
    finally:
        if shim.wait(stream, WAIT_S) == 0:
            shim.host_free(bodies.addr)
            shim.host_free(flag.addr)


# ---------------------------------------------------------------------------------------------------- pull
def pull_batches(shape, ctas, rng):
    """Message lengths of each batch of a shape."""
    jobs = 64
    if shape == "one_job":
        return [[(1 << 20) + 5]]
    if shape == "full_batch":
        return [[[16, 17, 1, 4096, 65536 + 3, 8191, 15, 300000 + 11][j % 8] for j in range(jobs)]]
    if shape == "tails_only":   # every message < 16 B: no body bytes at all, one empty chunk
        return [list(range(1, 16)), [1] * jobs]
    if shape == "ragged_lengths":
        return [[16 * int(rng.integers(1, 4000)) + 1 + (j % 15) for j in range(jobs)] for _ in range(3)]
    if shape == "chunk_clamps":
        # the publisher's chunk is total / (ctas - 1) rounded up to 1 KiB, clamped to [8 KiB, 256 KiB]: totals whose
        # share lands just inside and just outside each clamp
        out = []
        for share in (6000, 7168, 9000, 261000, 262144, 270000):
            total = share * (ctas - 1)
            k = 1 + int(rng.integers(0, 6))
            each = total // k
            out.append([each + (j % 3) for j in range(k - 1)] + [total - each * (k - 1) + 7])
        return out
    if shape == "ring_wrap":   # 20 batches in one launch: the 8-slot ring wraps twice
        return [[int(rng.integers(1, 40000)) for _ in range(1 + b % 5)] for b in range(20)]
    raise ValueError(shape)


PULL_SHAPES = ["one_job", "full_batch", "tails_only", "ragged_lengths", "chunk_clamps", "ring_wrap"]


@pytest.mark.parametrize("shape", PULL_SHAPES)
@pytest.mark.parametrize("grid", ["ctas2", "ctas3_min_stages", "default_ctas"])
def test_pull_kernel_copies_published_batches(shim, torch, grid, shape):
    """The resident pull kernel, started first on its own stream, serves batches published from the device: whole
    messages land (bodies by the copy CTAs, tails by CTA 0), nothing outside them is written, and its statistics
    count every job, batch and body byte.  The launch ends with its stop word."""
    default = shim.pull_default_ctas()
    ctas, stages, stage_bytes = {"ctas2": (2, 8, 24576), "ctas3_min_stages": (3, 3, 1024),
                                 "default_ctas": (default, 8, 24576)}[grid]
    assert 2 <= ctas <= default
    rng = np.random.default_rng(PULL_SHAPES.index(shape) * 10 + len(grid))
    batches = pull_batches(shape, ctas, rng)
    assert all(len(b) <= shim.pull_jobs() for b in batches)
    if shape == "ring_wrap":
        assert len(batches) > 2 * shim.pull_slots()
    lengths = [n for b in batches for n in b]
    _, jobs, size = place(lengths, gap=64)
    src_bytes = max(s + n for s, _, n in jobs) + 64
    host_src = rng.integers(0, 256, src_bytes, dtype=np.uint8)
    src, dst = to_device(torch, host_src), canary_buffer(torch, size)
    torch.cuda.synchronize()

    sess = shim.pull_create(len(batches))
    assert sess, shim.error()
    s_pull, s_pub = shim.stream_create(), shim.stream_create()
    assert s_pull and s_pub, shim.error()
    finished = False
    try:
        assert shim.pull_launch(sess, s_pull, ctas, stages, stage_bytes, 20_000_000, 25_000_000) == 0, shim.error()
        k = 0
        for b in batches:
            part = jobs[k:k + len(b)]
            k += len(b)
            sp = u64s([src.data_ptr() + s for s, _, _ in part])
            dp = u64s([dst.data_ptr() + d for _, d, _ in part])
            ln = u64s([n for _, _, n in part])
            assert shim.pull_publish(sess, s_pub, ptr(sp), ptr(dp), ptr(ln), len(part), ctas) == 0, shim.error()
        published = shim.wait(s_pub, WAIT_S)
        running = shim.wait(s_pull, 0.0)   # -2: still resident, as it must be until its stop word
        shim.pull_stop(sess)
        ended = shim.wait(s_pull, WAIT_S)
        assert published == 0, f"publishing did not finish: {shim.error()}"
        assert running == -2, "the pull kernel left before its stop word"
        assert ended == 0, f"pull kernel did not leave after its stop word: {shim.error()}"
        finished = True
    finally:
        if not finished:
            shim.pull_stop(sess)
            finished = shim.wait(s_pull, WAIT_S) == 0 and shim.wait(s_pub, WAIT_S) == 0
    stats = np.zeros(8, dtype=np.uint64)
    assert shim.pull_stats(sess, ptr(stats)) == 0, shim.error()
    assert shim.pull_destroy(sess) == 0
    shim.stream_destroy(s_pull)
    shim.stream_destroy(s_pub)

    want = np.full(size, CANARY, dtype=np.uint8)
    for s, d, n in jobs:
        want[d:d + n] = host_src[s:s + n]
    assert_bytes_equal(dst.cpu().numpy(), want, f"pull destination ({shape}, {ctas} CTAs)")
    nbytes, _, nbatches, njobs, _, _, _, tickets = (int(x) for x in stats)
    assert njobs == len(lengths)
    assert nbatches == len(batches)
    assert nbytes == sum(n & ~15 for n in lengths)
    assert tickets == len(batches) + 1   # the batches and the launch's EXIT marker
