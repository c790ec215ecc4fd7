"""`quantize_fp8` on a CUDA tensor: the native quantiser (tsb200_quantize_fp8) against its definition, the torch
expression that `quantize_fp8` runs on the CPU.

Every case compares x8 as uint8 and scale as int32 bit patterns with `quantize_fp8(x.cpu(), per_row)`. NaN equals NaN
in any encoding: the sign of a NaN the CPU makes depends on the host's default NaN (x86 makes inf / inf negative), and
the e4m3 helpers the kernels share write 0x7f.

The kernel reads 16-byte units when x, its row stride and K * element size are multiples of 16 bytes, and elements
otherwise. The layouts below take both: contiguous and row-strided inputs with K * size % 16 == 0 the vector path, a
base offset by one element (and any odd K) the element-wise path.
"""
import pytest
import torch

import pytorch_sparse_b200 as ts
from pytorch_sparse_b200 import ops

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
DTYPES = (torch.bfloat16, torch.float16, torch.float32, torch.float64)
KS = (1, 15, 16, 48, 128, 256, 400, 2048, 4096, 10000)
NS = (0, 1, 7, 4099)


def cpu_ref(x, per_row):
    return ts.quantize_fp8(x.detach().cpu(), per_row)


def assert_same_bits(x8, s, ref8, refs, what=""):
    a, b = x8.cpu().view(torch.uint8), ref8.cpu().view(torch.uint8)
    assert a.shape == b.shape and x8.dtype == torch.float8_e4m3fn, what
    nan = ((a & 0x7F) == 0x7F) & ((b & 0x7F) == 0x7F)
    bad = ~((a == b) | nan)
    if bool(bad.any()):
        i = tuple(int(j) for j in bad.nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())} e4m3 bytes differ, first at {i}: "
                             f"0x{int(a[i]):02x} vs 0x{int(b[i]):02x}")
    assert s.dtype == torch.float32 and s.shape == refs.shape, what
    sa, sb = s.cpu().view(torch.int32), refs.cpu().view(torch.int32)
    bad = sa != sb
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} scales differ: {s.cpu()[bad][:4]} vs {refs[bad][:4]}"


def make_rows(N, K, dtype, g):
    """Random rows with magnitudes 2^-e ... 2^e (e = 12 for f16, 60 otherwise) from row to row, a few all-zero rows
    and -0 entries; built in fp64 on the CPU and rounded once to `dtype`."""
    e = 12 if dtype == torch.float16 else 60
    x = torch.randn(N, K, generator=g, dtype=torch.float64)
    x *= torch.exp2(torch.randint(-e, e + 1, (N, 1), generator=g).double())
    if N > 3:
        x[N // 3] = 0.0
        x[N // 2, ::3] = -0.0
    return x.to(dtype)


def place(xc, layout):
    """The CPU matrix `xc` on the GPU as a contiguous tensor, a column slice of a wider one (row-strided, rows 16-byte
    aligned when K * size is), or a slice starting one element in (no row is 16-byte aligned)."""
    N, K = xc.shape
    if layout == "contiguous":
        return xc.to(DEV)
    wide = torch.full((N, K + 24), float("nan"), dtype=xc.dtype, device=DEV)
    off = 0 if layout == "strided" else 1
    x = wide[:, off:off + K]
    x.copy_(xc)
    return x


@pytest.mark.parametrize("layout", ["contiguous", "strided", "misaligned"])
@pytest.mark.parametrize("K", KS)
@pytest.mark.parametrize("per_row", [True, False], ids=["rowscale", "tensorscale"])
@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: str(d).split(".")[1])
def test_matches_cpu(dtype, per_row, K, layout):
    g = torch.Generator().manual_seed(K * 7 + DTYPES.index(dtype))
    for N in NS:
        if N == 0 and not per_row:
            continue                                 # raises, like the CPU path (test_error_cases)
        x = place(make_rows(N, K, dtype, g), layout)
        x8, s = ts.quantize_fp8(x, per_row)
        assert x8.is_contiguous() and x8.data_ptr() % 16 == 0
        assert_same_bits(x8, s, *cpu_ref(x, per_row), f"N={N}")


def test_edge_rows():
    """All zero, all -0, NaN first / inside / last, +-inf, inf with NaN, fp32 subnormals (the scale is subnormal too),
    the smallest subnormal (its scale rounds to 0, so every quotient is inf), and quotients on e4m3 rounding midpoints:
    with amax 448 the scale is exactly 1, with 896 exactly 2, so the quotient is the midpoint itself, half of them
    rounding down to an even mantissa and half up."""
    K = 48
    mids = torch.tensor([1.0625, 1.1875, 2.125, 3.125, 13.5, 27.0, 100.0, 200.0, 0.5 + 2.0 ** -5, 2.0 ** -10,
                         3 * 2.0 ** -10, 5 * 2.0 ** -10, 9 * 2.0 ** -10])
    rows = []
    for scale in (1.0, 2.0):
        r = torch.zeros(K)
        r[0] = 448.0 * scale
        r[1:1 + mids.numel()] = mids * scale
        r[1 + mids.numel():1 + 2 * mids.numel()] = -mids * scale
        rows.append(r)
    nan, inf = float("nan"), float("inf")
    special = [torch.zeros(K), torch.full((K,), -0.0)]
    for pos in (0, K // 2, K - 1):
        r = torch.randn(K)
        r[pos] = nan
        special.append(r)
    for v in (inf, -inf):
        r = torch.randn(K)
        r[5] = v
        special.append(r)
    r = torch.randn(K)
    r[3], r[9] = inf, nan
    special.append(r)
    r = torch.randn(K) * 1e-40                       # fp32 subnormals
    special.append(r)
    r = torch.full((K,), 2.0 ** -149)                # the smallest one
    special.append(r)
    x32 = torch.stack(rows + special + [torch.randn(K) * 10.0 ** e for e in (-30, -10, 0, 10, 30)])
    for dtype in (torch.float32, torch.bfloat16, torch.float16, torch.float64):
        xc = x32.to(dtype)
        for layout in ("contiguous", "misaligned"):
            x = place(xc, layout)
            for per_row in (True, False):
                assert_same_bits(*ts.quantize_fp8(x, per_row), *cpu_ref(x, per_row), f"{dtype} {layout} {per_row}")
    # the midpoint rows really sit on midpoints with scale 1 / 2
    _, s = ts.quantize_fp8(x32.to(DEV), True)
    assert s[0].item() == 1.0 and s[1].item() == 2.0


def test_tensor_scale_spans_1e30():
    """Rows from 1e-30 to 1e30 across the tensor: with one scale most quotients underflow to e4m3 subnormals and 0."""
    g = torch.Generator().manual_seed(3)
    N, K = 601, 128
    ex = torch.linspace(-30, 30, N, dtype=torch.float64).view(-1, 1)
    xc = torch.randn(N, K, generator=g, dtype=torch.float64) * torch.pow(10.0, ex)
    for dtype in (torch.float32, torch.bfloat16, torch.float64):
        x = xc.to(dtype).to(DEV)
        x8, s = ts.quantize_fp8(x, False)
        assert_same_bits(x8, s, *cpu_ref(x, False), str(dtype))
        b = x8.view(torch.uint8).cpu() & 0x7F
        assert bool(((b > 0) & (b < 8)).any()) and bool((b == 0).any())    # subnormals and zeros both occur


def test_more_than_2_31_elements():
    """A bf16 [2^24 + 64, 128] tensor (2^31 + 8192 elements, 4.3 GB, 6.5 GB with x8): the rows around element 2^31
    (the start of row 2^24) against the CPU quantiser of those rows; the per-tensor scale against the CPU amax."""
    K = 128
    N = (1 << 31) // K + 64
    r0 = (1 << 31) // K
    x = torch.empty(N, K, dtype=torch.bfloat16, device=DEV).uniform_(-1.0, 1.0)
    x[r0 + 1, 17] = -1000.0                         # the tensor's amax, past element 2^31
    x[r0 - 2] = 0.0                                 # an all-zero row just before it
    rows = slice(r0 - 4, r0 + 4)

    x8, s = ts.quantize_fp8(x, True)
    assert_same_bits(x8[rows], s[rows], *cpu_ref(x[rows], True), "per row")
    assert_same_bits(x8[:4], s[:4], *cpu_ref(x[:4], True), "per row, first rows")
    assert_same_bits(x8[-4:], s[-4:], *cpu_ref(x[-4:], True), "per row, last rows")
    del x8, s

    amax = max(x[i:i + (1 << 20)].cpu().abs().amax().float() for i in range(0, N, 1 << 20))
    s_ref = torch.where(amax > 0, amax / 448.0, torch.ones_like(amax))
    x8, s = ts.quantize_fp8(x, False)
    ref8 = (x[rows].cpu().float() / s_ref).to(torch.float8_e4m3fn)
    assert_same_bits(x8[rows], s, ref8, s_ref, "per tensor")
    assert float(amax) == 1000.0
    del x, x8, s
    torch.cuda.empty_cache()                         # hand the 6.5 GB back to the device for the tests that follow


@pytest.mark.parametrize("layout", ["contiguous", "strided"])
@pytest.mark.parametrize("dtype", (torch.bfloat16, torch.float16, torch.float32), ids=lambda d: str(d).split(".")[1])
def test_peak_memory(dtype, layout):
    """No float temporaries: the peak allocation above the input is x8, the scales and the amax word (<= 1 MB)."""
    N, K = 100_000, 256
    x = place(torch.randn(N, K).to(dtype), layout)
    for per_row in (True, False):
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        x8, s = ts.quantize_fp8(x, per_row)
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated() - base
        assert peak <= N * K + 4 * N + (1 << 20), (per_row, peak)
        del x8, s


@pytest.mark.parametrize("per_row", [True, False], ids=["rowscale", "tensorscale"])
def test_cuda_graph_capture(per_row):
    g = torch.Generator().manual_seed(5)
    N, K = 3000, 256
    x = torch.randn(N, K, generator=g).bfloat16().to(DEV)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        ts.quantize_fp8(x, per_row)                  # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        x8, s = ts.quantize_fp8(x, per_row)
    for i in range(2):
        x.copy_(torch.randn(N, K, generator=g).bfloat16().to(DEV) * (10.0 ** i))
        graph.replay()
        torch.cuda.synchronize()
        assert_same_bits(x8, s, *ts.quantize_fp8(x, per_row), "replay vs eager")
        assert_same_bits(x8, s, *cpu_ref(x, per_row), "replay vs cpu")


def test_requires_grad_keeps_history():
    """Under grad mode an x that requires grad takes the torch expression on the GPU, as before: its scale keeps a
    grad_fn (and divides by 448 as torch's CUDA division by a scalar does, so it is compared within one ulp)."""
    x = torch.randn(40, 32, device=DEV, requires_grad=True)
    for per_row in (True, False):
        x8, s = ts.quantize_fp8(x, per_row)
        assert s.grad_fn is not None
        assert torch.allclose(s.detach().cpu(), cpu_ref(x, per_row)[1], rtol=2.0 ** -23, atol=0)
        with torch.no_grad():
            x8, s = ts.quantize_fp8(x, per_row)
        assert s.grad_fn is None
        assert_same_bits(x8, s, *cpu_ref(x, per_row))


def test_scripted_runs_the_op():
    scripted = torch.jit.script(ts.quantize_fp8)
    x = torch.randn(33, 48, device=DEV).half()
    for per_row in (True, False):
        assert_same_bits(*scripted(x, per_row), *cpu_ref(x, per_row))
    assert_same_bits(*torch.ops.tsb200.quantize_fp8(x, True), *cpu_ref(x, True))


def test_operand_of_a_hop():
    """The native operand fed to spmm_fp8_quant gives the same hop, bit for bit, as the CPU-made operand."""
    g = torch.Generator().manual_seed(11)
    N, K, E = 5000, 128, 60_000
    row = torch.randint(N, (E,), generator=g)
    col = torch.randint(N, (E,), generator=g)
    adj = ts.SparseTensor(row=row.to(DEV), col=col.to(DEV), value=torch.rand(E, generator=g).to(DEV),
                          sparse_sizes=(N, N)).coalesce()
    x = (torch.randn(N, K, generator=g) * torch.exp2(torch.randint(-8, 9, (N, 1), generator=g).float())).to(DEV)
    for per_row in (True, False):
        x8, s = ts.quantize_fp8(x, per_row)
        c8, cs = cpu_ref(x, per_row)
        assert_same_bits(x8, s, c8, cs)
        y8, ys = adj.spmm_fp8_quant(x8, s)
        r8, rs = adj.spmm_fp8_quant(c8.to(DEV), cs.to(DEV))
        assert torch.equal(y8.view(torch.uint8), r8.view(torch.uint8)) and torch.equal(ys, rs)


def test_error_cases():
    def same_error(shape, per_row):
        with pytest.raises(Exception) as cpu_err:
            ts.quantize_fp8(torch.zeros(shape), per_row)
        with pytest.raises(cpu_err.type, match="amax"):
            ts.quantize_fp8(torch.zeros(shape, device=DEV), per_row)

    with pytest.raises(ValueError):
        ts.quantize_fp8(torch.ones(3, device=DEV))
    with pytest.raises(ValueError):
        ts.quantize_fp8(torch.ones(2, 3, 4, device=DEV))
    same_error((3, 0), True)                          # IndexError
    same_error((3, 0), False)                         # RuntimeError
    same_error((0, 0), True)
    same_error((0, 5), False)
    x8, s = ts.quantize_fp8(torch.zeros(0, 5, device=DEV), True)
    assert x8.shape == (0, 5) and x8.dtype == torch.float8_e4m3fn and s.shape == (0,) and s.dtype == torch.float32
    with pytest.raises(RuntimeError, match="bfloat16, torch.float16 or torch.float32"):
        ops.quantize_fp8(torch.ones(2, 3, dtype=torch.float64, device=DEV))
    # integer and fp8 inputs go through .float(), as on the CPU
    xi = torch.randint(-300, 300, (9, 17), device=DEV)
    assert_same_bits(*ts.quantize_fp8(xi), *cpu_ref(xi, True))
    assert_same_bits(*ts.quantize_fp8(xi.t()), *cpu_ref(xi.t(), True))     # last dimension not contiguous
