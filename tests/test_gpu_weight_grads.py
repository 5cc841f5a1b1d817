"""GPU (H100): the weight-gradient path of the CUDA backward (DESIGN.md section 4.2) at kernel precision.  Every weight
gradient is a row reduction dW[k][n] = alpha sum_rows X[row][k] D[row][n]: eqd_tn_gemm (csrc/bwd_reduce.cu) writes one
fp32 partial per row chunk, eqd_grad_reduce sums the chunks in fp64 in a fixed order and scatters them through the index
maps of training.layer_reductions / HEAD_REDUCTION into the flat gradient.

  1. The two kernels called directly.  Every chunk partial is held per element to a bound counted from the kernel's
     operation order: the within-chunk sum is a sequential fmaf chain over m = rows_per_chunk rows, then one multiply by
     alpha, so |P - alpha sum x d| <= (gamma_m (1 + u) + u) |alpha| sum |x d|  (u = 2^-24, gamma_m = m u / (1 - m u)).
     The column sums: each thread adds m / 16 rows, then the 16 row groups are added in a fixed order, then alpha:
     gamma_{m/16 + 16} in place of gamma_m.  Both bounds add (|alpha| m (1 + gamma_m) + 1) 2^-150 for gradual
     underflow: the rbf features exp(-d^2 / sigma) of distant node pairs are subnormal in fp32, and their products with
     dz1 round to 0 (the relative bound alone then reads 1 / (gamma_m + u) = 65 281 at m = 256).  A per-chunk bound is
     what makes one missing row visible; a bound on the whole sum is too loose at 500 chunks.  eqd_grad_reduce must
     equal, bit for bit,
     float32(prior + float32(sum_c float64(partial[c stride + src]))) summed sequentially over c.
  2. Every reduction of a real TrainEngine.backward, recorded through a stand-in for TrainEngine.lib: each eqd_tn_gemm
     call's partials and column sums against per-chunk fp64 of the operands it read (cloned at the call, on the stream
     the backward runs on), with the row count and alpha the reduction table prescribes; and the flat gradient's
     reduction-owned elements bitwise equal to a numpy fold of the recorded eqd_grad_reduce calls in call order, from a
     non-zero starting buffer.  Elements no reduction owns keep their starting value, except those that
     eqd_bwd_head_dropout (the keypoint key / query projections) and eqd_bwd_embed write; their own tests cover them.
  3. Whole-layer composition: training.layer_backward on seeded h_in, x_in, h0 and upstream gradients, with aggr and mu
     from the fp64 forward of tests/layer_norm_ref.layer_forward rounded to fp32 (a consistent stash, no forward-kernel
     error), against fp64 autograd of that forward, every parameter gradient of the layer at 1e-5 of the tensor's
     largest fp64 magnitude (the bound the stage kernels meet).  The layers run at leakyrelu_neg_slope = 1, where the
     layer is smooth: at the shipped 0.01 a pre-activation within fp32 rounding of 0 can take the other branch in the
     kernels' fp32 recompute, and summed into a weight gradient that is what forces the 3e-3 of the model-level tests.
     The kernel tests cover the branch itself at the shipped slope.

Batches: `bench` is bench.py --workload train's 32-pair batch (17 407 nodes, 174 k edges: 454 chunks of 384 rows per
edge reduction), `train` test_gpu_backward_kernels.py's 100 pairs of 200 + 200 nodes (N = 40 000, E = 400 000).

Measured on an H100 80GB HBM3 (700 W power limit), worst fraction of the bound (`pytest -s` prints every value):
  part 1   tn_gemm partials at most 0.086, column sums 0.095; grad_reduce bitwise
  part 2   partials 0.342, column sums 0.324 (46 or 73 eqd_tn_gemm calls per case); the flat gradient bitwise equal to
           the fold of 82 or 130 eqd_grad_reduce calls
  part 3   att_mlp_Q.0.weight of layer 0 7.4e-6 of max |ref| (K 4.0e-6), every other parameter gradient under 1.4e-6
The file runs in about 30 s on that GPU.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import dropout_masks as dm
import golden_io as gio
import layer_norm_ref as nr
from equidock_public_b200 import _native as nat
from equidock_public_b200 import synthetic
from equidock_public_b200 import training as tr
from equidock_public_b200.engine import GraphPlan
from equidock_public_b200.training import BackwardWorkspace, TrainEngine, tn_gemm_shapes
from test_gpu_backward_kernels import Report, _batch, _gen
from test_gpu_forward_kernels import _coords
from test_gpu_trainer_step import _device_batch, _shard

pytestmark = pytest.mark.gpu

F64 = torch.float64
U = 2.0 ** -24
ETA = 2.0 ** -150                 # half the spacing of fp32 subnormals: the absolute error of one rounding
SENT = -777.25                    # finite pre-fill of floats a kernel must leave untouched
GUARD = 67                        # sentinel floats past every output
P_DROP, DROP_SEED, DROP_RANK, DROP_LAYER = 0.25, 0x5EED_0123_4567_89AB, 3, 2

_CACHE = {}


def _gamma(m):
    return m * U / (1.0 - m * U)


def _tn_rel(m):
    """Relative bound (of |alpha| sum |terms|) of a sum of m sequentially rounded terms followed by the alpha multiply."""
    return _gamma(m) * (1.0 + U) + U


def _tn_abs(m, alpha):
    """Absolute part of the same bound: each of the m roundings may lose up to half the subnormal spacing (2^-150) when
    its result underflows, the alpha multiply once more."""
    return (abs(alpha) * m * (1.0 + _gamma(m)) + 1.0) * ETA


def _chunking(rows, K, nc):
    lib = nat.load()
    rpc, nch = C.c_int32(0), C.c_int32(0)
    floats = int(lib.eqd_tn_partial_floats(rows, K, nc, C.byref(rpc), C.byref(nch)))
    return rpc.value, nch.value, floats


def _fraction(got, ref, bound):
    """max |got - ref| / bound; where the bound is 0 the kernel must be exact.  Non-finite values count as infinite."""
    diff = torch.nan_to_num((got.to(F64) - ref).abs(), nan=float('inf'))
    exact = bound == 0
    if bool((diff[exact] != 0).any()):
        return float('inf')
    return float((diff[~exact] / bound[~exact]).max()) if bool((~exact).any()) else 0.0


def _chunk_fractions(X, D, K, nc, rows, alpha, part, colsum, rpc, nch):
    """Per-chunk fp64 of alpha X^T D (X [rows][>= K], D [rows][>= nc]) against the kernel's partials / column sums:
    (fraction of the partials' bound, fraction of the column sums' bound or None)."""
    pad = nch * rpc - rows
    chunks = lambda t, w: torch.nn.functional.pad(t[:rows, :w].to(F64), (0, 0, 0, pad)).view(nch, rpc, w)
    Xc, Dc = chunks(X, K), chunks(D, nc)
    a = float(np.float32(alpha))
    ref = a * torch.bmm(Xc.transpose(1, 2), Dc)
    bnd = _tn_rel(rpc) * abs(a) * torch.bmm(Xc.abs().transpose(1, 2), Dc.abs()) + _tn_abs(rpc, a)
    fp = _fraction(part[:nch * K * nc].view(nch, K, nc), ref, bnd)
    fc = None
    if colsum is not None:
        mc = rpc // 16 + 16
        fc = _fraction(colsum[:nch * nc].view(nch, nc), a * Dc.sum(1),
                       _tn_rel(mc) * abs(a) * Dc.abs().sum(1) + _tn_abs(mc, a))
    return fp, fc


def _report(name, rows):
    """rows: (tag, fraction of the bound); all must be <= 1."""
    lines = [f'{"ok " if f <= 1.0 else "BAD"} {name} {tag:44s} {f:.3f}' for tag, f in rows]
    print('\n' + '\n'.join(lines))
    print(f'{name}: worst fraction of the bound {max(f for _, f in rows):.3f}')
    bad = [ln for ln in lines if ln.startswith('BAD')]
    assert not bad, '\n'.join(bad)


# ---- batches ------------------------------------------------------------------------------------------------------

def _bench_graph(dev):
    if 'bench' not in _CACHE:
        g = _device_batch(_shard(0, 1)[0], dev)[0]
        _CACHE['bench'] = (g, GraphPlan.from_graph(g, dev, 10))
    return _CACHE['bench']


def _graph(kind, dev):
    if kind == 'bench':
        return _bench_graph(dev)
    if kind == 'train':
        return _batch('train', dev)
    if kind not in _CACHE:
        if kind == 'tail1':        # N = 57 < 256 (one partial node chunk); E = 9 * 57 = 513 = 2 * 256 + 1
            pairs = [synthetic.synthetic_pair(np.random.default_rng(41), 30, 27, 9)]
        elif kind == 'one1':       # a pair of two 1-node proteins (no edges) among ordinary pairs
            rng = np.random.default_rng(42)
            pairs = [synthetic.synthetic_pair(rng, 70, 45, 10), synthetic.synthetic_pair(rng, 1, 1, 10),
                     synthetic.synthetic_pair(rng, 12, 130, 10)]
        elif kind == 'mid':        # 16 pairs of 200 + 200 nodes: 6 400 nodes, 64 000 edges
            pairs = synthetic.synthetic_batch(16, seed=43)
        else:
            raise ValueError(kind)
        g = gio.make_batch(pairs, dev)
        _CACHE[kind] = (g, GraphPlan.from_graph(g, dev, 10))
    return _CACHE[kind]


def _n_e(kind, dev):
    if kind == 'bench330':         # the 330-pair bench batch's edge count
        return 132_000, 1_320_000
    plan = _graph(kind, dev)[1]
    return plan.N, plan.E


# ---- part 1: eqd_tn_gemm and eqd_grad_reduce called directly ----------------------------------------------------

def _tn_run(rows, K, nc, alpha=1.0, with_colsum=True, ldx=None, ldd=None, seed=0, dev=None):
    """One eqd_tn_gemm on seeded data with sentinel-guarded outputs; returns the fractions of the bounds (partials,
    column sums), the partial and colsum buffers and the chunk count."""
    lib = nat.load()
    ldx, ldd = ldx or K, ldd or nc
    rpc, nch, floats = _chunking(rows, K, nc)
    assert floats == nch * K * nc
    r = _gen(seed, dev)
    X, D = r(max(rows, 1), ldx), r(max(rows, 1), ldd, s=0.5) + 0.25
    part = torch.full((floats + GUARD,), SENT, device=dev)
    cs = torch.full((nch * nc + GUARD,), SENT, device=dev)
    got = C.c_int32(-5)
    st = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    nat.check(lib.eqd_tn_gemm(nat.ptr(X), ldx, K, nat.ptr(D), ldd, nc, rows, alpha, nat.ptr(part),
                              nat.ptr(cs) if with_colsum else None, C.byref(got), st), 'eqd_tn_gemm')
    torch.cuda.synchronize()
    assert got.value == nch, ('chunk count differs from eqd_tn_partial_floats', got.value, nch)
    assert bool((part[floats:] == SENT).all()), 'floats past nchunks * K * ncols of partial were written'
    assert bool((cs[nch * nc:] == SENT).all()), 'floats past nchunks * ncols of colsum were written'
    if not with_colsum:
        assert bool((cs == SENT).all()), 'colsum written although NULL was passed'
    if rows == 0:
        assert nch == 0 and bool((part == SENT).all())
        return 0.0, 0.0, part, cs, nch
    fp, fc = _chunk_fractions(X, D, K, nc, rows, alpha, part, cs if with_colsum else None, rpc, nch)
    return fp, fc, part, cs, nch


# (rows, K, ncols, alpha, colsum, ldx, ldd)
TN_CASES = ([(n, 64, 64, 1.0, True, None, None) for n in (1, 63, 64, 65, 255, 256, 257)]
            + [(256 * 3 + d, 64, 64, 0.75, True, None, None) for d in (-1, 0, 1)]         # rpc 256, 3 chunks
            + [(384 * 454 + d, 64, 64, 1.0, True, None, None) for d in (-1, 0, 1)]       # rpc 384, 454 chunks (bench E)
            + [(1000, K, nc, 1.0, False, None, None) for K in (44, 64, 72) for nc in (64, 72, 320, 344)]
            + [(1000, 44, 64, 0.75, True, 72, 80), (777, 72, 344, 0.5, True, 76, 348)])  # ld > K, ld > ncols


TN_IDS = [f'{c[0]}x{c[1]}x{c[2]}-a{round(100 * c[3])}-cs{int(c[4])}-ld{c[5] or 0}' for c in TN_CASES]


@pytest.mark.parametrize('rows,K,nc,alpha,with_cs,ldx,ldd', TN_CASES, ids=TN_IDS)
def test_tn_gemm_chunk_partials_vs_fp64(rows, K, nc, alpha, with_cs, ldx, ldd, cuda_device):
    fp, fc = _tn_run(rows, K, nc, alpha, with_cs, ldx, ldd, seed=rows % 9973 + K + nc, dev=cuda_device)[:2]
    _report('tn_gemm', [('partial', fp)] + ([('colsum', fc)] if with_cs else []))


# (rows, K, ncols): small and partial chunks, and the training shapes of 100 pairs of 200 + 200 nodes
TN_REDUCE_SHAPES = ((1000, 64, 64), (37, 44, 64), (5000, 72, 344), (300, 72, 72), (400000, 64, 64), (400000, 44, 64),
                    (40000, 64, 320), (40000, 72, 344), (40000, 64, 72))


def test_tn_gemm_and_reduce_vs_fp64(cuda_device):
    """eqd_tn_gemm (alpha 0.5, column sums on) followed by eqd_grad_reduce of its partials and column sums into one
    gradient buffer: the partials per chunk against fp64 within the bound above, the reduced gradient bitwise equal to
    the numpy fold of those partials, through permuted destination maps onto a non-zero prior."""
    lib, dev = nat.load(), cuda_device
    rows_out = []
    for i, (rows, K, nc) in enumerate(TN_REDUCE_SHAPES):
        fp, fc, part, cs, nch = _tn_run(rows, K, nc, 0.5, True, seed=700 + i, dev=dev)
        rows_out += [(f'{rows}x{K}x{nc} partial', fp), (f'{rows}x{K}x{nc} colsum', fc)]
        rng = np.random.default_rng(700 + i)
        total = K * nc + nc + 3
        prior = rng.standard_normal(total).astype(np.float32)
        dst = rng.permutation(total)[:K * nc + nc].astype(np.int32)
        grad = torch.from_numpy(prior).to(dev)
        T = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.int32)).to(dev)
        src_p, src_c = T(np.arange(K * nc)), T(np.arange(nc))
        dst_p, dst_c = T(dst[:K * nc]), T(dst[K * nc:])
        nat.check(lib.eqd_grad_reduce(nat.ptr(part), nch, K * nc, nat.ptr(src_p), nat.ptr(dst_p), K * nc,
                                      nat.ptr(grad), None), 'eqd_grad_reduce')
        nat.check(lib.eqd_grad_reduce(nat.ptr(cs), nch, nc, nat.ptr(src_c), nat.ptr(dst_c), nc, nat.ptr(grad), None),
                  'eqd_grad_reduce')
        ref = prior.copy()
        _fold(ref, part[:nch * K * nc].view(nch, K * nc).cpu().numpy(), dst[:K * nc])
        _fold(ref, cs[:nch * nc].view(nch, nc).cpu().numpy(), dst[K * nc:])
        got = grad.cpu().numpy()
        assert np.array_equal(got.view(np.uint32), ref.view(np.uint32)), \
            f'{rows}x{K}x{nc}: {int((got != ref).sum())} reduced elements differ from the fp64 fold'
    _report('tn_gemm + grad_reduce', rows_out)


@pytest.mark.parametrize('batch', ['bench', 'train', 'bench330'])
def test_tn_gemm_training_shapes_vs_fp64(batch, cuda_device):
    """Every (rows, K, ncols) of training.tn_gemm_shapes for the batch, with alpha 0.75 (the DIPS skip_weight_h)."""
    N, E = _n_e(batch, cuda_device)
    shapes = tn_gemm_shapes(N, E) if batch != 'bench330' else [(E, 44, 64), (E, 64, 64)]
    rows = []
    for i, (n, K, nc) in enumerate(shapes):
        fp, fc = _tn_run(n, K, nc, 0.75, True, seed=500 + i, dev=cuda_device)[:2]
        rows += [(f'{n}x{K}x{nc} partial', fp), (f'{n}x{K}x{nc} colsum', fc)]
    if batch == 'bench':
        assert _chunking(E, 64, 64)[1] == 454
    _report(f'tn_gemm[{batch}]', rows)


def test_tn_gemm_zero_rows_and_refusals(cuda_device):
    lib, dev = nat.load(), cuda_device
    X, D = torch.randn(300, 80, device=dev), torch.randn(300, 80, device=dev)
    part, cs = torch.full((64 * 64 * 4,), SENT, device=dev), torch.full((64 * 4,), SENT, device=dev)
    nch = C.c_int32(-5)
    nat.check(lib.eqd_tn_gemm(nat.ptr(X), 64, 64, nat.ptr(D), 64, 64, 0, 1.0, nat.ptr(part), nat.ptr(cs), C.byref(nch),
                              None), 'eqd_tn_gemm')
    torch.cuda.synchronize()
    assert nch.value == 0 and bool((part == SENT).all()) and bool((cs == SENT).all())
    off = lambda t, b: C.c_void_p(t.data_ptr() + b)
    bad = {'K % 4': (nat.ptr(X), 64, 42, nat.ptr(D), 64, 64), 'ncols % 4': (nat.ptr(X), 64, 64, nat.ptr(D), 64, 62),
           'ldx % 4': (nat.ptr(X), 66, 64, nat.ptr(D), 64, 64), 'ldd % 4': (nat.ptr(X), 64, 64, nat.ptr(D), 66, 64),
           'X misaligned': (off(X, 4), 64, 64, nat.ptr(D), 64, 64), 'D misaligned': (nat.ptr(X), 64, 64, off(D, 8), 64, 64)}
    for what, (xp, ldx, K, dp, ldd, nc) in bad.items():
        rc = lib.eqd_tn_gemm(xp, ldx, K, dp, ldd, nc, 200, 1.0, nat.ptr(part), nat.ptr(cs), C.byref(nch), None)
        assert rc == -1, (what, rc)
    torch.cuda.synchronize()
    assert bool((part == SENT).all()) and bool((cs == SENT).all()), 'a refused call wrote its outputs'


def _fold(grad, vals, dst):
    """numpy restatement of eqd_grad_reduce: grad[dst] = f32(grad[dst] + f32(sum_c f64(vals[c]))), c in order."""
    t = np.zeros(vals.shape[1], np.float64)
    for c in range(vals.shape[0]):
        t = t + vals[c].astype(np.float64)
    grad[dst] = grad[dst] + t.astype(np.float32)


@pytest.mark.parametrize('nch,stride', [(1, 4096), (7, 4096), (454, 4096), (521, 22016), (132, 272)])
def test_grad_reduce_bitwise_vs_numpy(nch, stride, cuda_device):
    lib, dev = nat.load(), cuda_device
    rng = np.random.default_rng(nch + stride)
    # a wide dynamic range, so that an fp32 accumulation or another order differs in the last bits
    part = (rng.standard_normal(nch * stride) * 2.0 ** rng.integers(-12, 12, nch * stride)).astype(np.float32)
    n = stride * 3 // 4
    src = rng.permutation(stride)[:n].astype(np.int32)
    total = 2 * stride + 5
    dst = rng.permutation(total)[:n].astype(np.int32)
    prior = (rng.standard_normal(total) * 10).astype(np.float32)
    grad = torch.from_numpy(prior).to(dev)
    T = lambda a: torch.from_numpy(a).to(dev)
    pt, st_, dt = T(part), T(src), T(dst)
    nat.check(lib.eqd_grad_reduce(nat.ptr(pt), nch, stride, nat.ptr(st_), nat.ptr(dt), n, nat.ptr(grad), None),
              'eqd_grad_reduce')
    ref = prior.copy()
    _fold(ref, part.reshape(nch, stride)[:, src], dst)
    got = grad.cpu().numpy()
    assert np.array_equal(got.view(np.uint32), ref.view(np.uint32)), \
        f'{int((got != ref).sum())} elements differ from the fp64 fold'
    untouched = np.ones(total, bool)
    untouched[dst] = False
    assert np.array_equal(got[untouched].view(np.uint32), prior[untouched].view(np.uint32))
    if nch > 1:   # the test data tells an fp32 accumulation apart
        vals = part.reshape(nch, stride)[:, src]
        t32, t64 = np.zeros(n, np.float32), np.zeros(n, np.float64)
        for c in range(nch):
            t32, t64 = t32 + vals[c], t64 + vals[c]
        assert not np.array_equal(t32, t64.astype(np.float32))
    # nchunks = 0 and n = 0 are no-ops
    before = grad.clone()
    nat.check(lib.eqd_grad_reduce(nat.ptr(pt), 0, stride, nat.ptr(st_), nat.ptr(dt), n, nat.ptr(grad), None), 'r0')
    nat.check(lib.eqd_grad_reduce(nat.ptr(pt), nch, stride, nat.ptr(st_), nat.ptr(dt), 0, nat.ptr(grad), None), 'r1')
    torch.cuda.synchronize()
    assert torch.equal(grad, before)


# ---- part 2: every reduction of a real backward -----------------------------------------------------------------

def _owner(ptr, tensors):
    """(tensor, byte offset) of the tensor in ``tensors`` whose storage holds device address ``ptr``."""
    for t in tensors:
        base = t.data_ptr()
        if base <= ptr < base + t.numel() * t.element_size():
            return t, ptr - base
    raise AssertionError(f'pointer {ptr:#x} is in none of the known buffers')


def _floats_at(ptr, count, tensors):
    t, off = _owner(ptr, tensors)
    raw = t.reshape(-1).view(torch.uint8)
    assert off % 4 == 0 and off + 4 * count <= raw.numel()
    return raw[off:off + 4 * count].view(torch.float32).clone()


def _ints_at(ptr, count, tensors):
    t, off = _owner(ptr, tensors)
    assert t.dtype == torch.int32 and off == 0 and t.numel() == count
    return t.clone()


class _RecordingLib:
    """Stands in for TrainEngine.lib.  At each eqd_tn_gemm it checks the partials / column sums the call left against
    per-chunk fp64 of the operands it read (cloned on the current stream, the backward's); at each eqd_grad_reduce it
    records the values the call sums, (nchunks, n) fp32, and the destination indices."""

    def __init__(self, lib, eng, fwd_box, expected):
        self._lib, self._eng, self._fwd, self._expected = lib, eng, fwd_box, expected
        self.tn, self.reduce = [], []

    def __getattr__(self, name):
        return getattr(self._lib, name)

    def _buffers(self):
        ws, fwd = self._eng._ws, self._fwd[0]
        bufs = [v for v in vars(ws).values() if torch.is_tensor(v)] + list(ws.dh)
        return bufs + [fwd['stash'], fwd['h']]

    def _maps(self):
        out = []
        for maps in [self._eng._head_maps] + list(self._eng._maps.values()):
            for pair in maps.values():
                out += [t for mp in pair if mp is not None for t in mp]
        return out

    def eqd_tn_gemm(self, X, ldx, K, D, ldd, ncols, nrows, alpha, partial, colsum, nch, stream):
        rc = self._lib.eqd_tn_gemm(X, ldx, K, D, ldd, ncols, nrows, alpha, partial, colsum, nch, stream)
        label, rows, a = self._expected[len(self.tn)]
        ws = self._eng._ws
        rpc, n_ch, _ = _chunking(rows, K, ncols)
        got = (int(nrows), float(np.float32(alpha)), nch._obj.value)
        want = (rows, float(np.float32(a)), n_ch)
        assert got == want, f'{label}: eqd_tn_gemm called with (rows, alpha) -> chunks {got}, expected {want}'
        assert partial.value == ws.partial.data_ptr() and (colsum is None or colsum.value == ws.colsum.data_ptr())
        bufs = self._buffers()
        Xr = _floats_at(X.value, rows * ldx, bufs).view(rows, ldx)
        Dr = _floats_at(D.value, rows * ldd, bufs).view(rows, ldd)
        fp, fc = _chunk_fractions(Xr, Dr, K, ncols, rows, a, ws.partial, ws.colsum if colsum is not None else None,
                                  rpc, n_ch)
        self.tn.append((label, n_ch, fp, fc))
        return rc

    def eqd_grad_reduce(self, partial, nchunks, stride, src, dst, n, grad, stream):
        if n > 0 and nchunks > 0:
            ws = self._eng._ws
            buf, off = _owner(partial.value, [ws.partial, ws.colsum, ws.vec])
            assert off == 0
            maps = self._maps()
            s, d = _ints_at(src.value, n, maps).long(), _ints_at(dst.value, n, maps)
            idx = torch.arange(nchunks, device=buf.device)[:, None] * stride + s[None, :]
            self.reduce.append((buf.reshape(-1)[idx].cpu().numpy(), d.cpu().numpy()))
        return self._lib.eqd_grad_reduce(partial, nchunks, stride, src, dst, n, grad, stream)


def _expected_calls(eng, N, E):
    """(label, rows, alpha) of every eqd_tn_gemm of one TrainEngine.backward, in launch order."""
    out = [('head', N, 1.0)]
    layers = eng.iegmn.iegmn_layers
    for li in reversed(range(len(layers))):
        tp = eng.layer_pack(layers[li])
        sk = float(layers[li].packed(eng.device).struct.dev.skip_weight_h)
        # alpha = skip_weight_h on node_mlp.4 (node2) of a 64-wide layer only: h' = skip node_mlp(.) + (1 - skip) h
        out += [(f'L{li} {r.name}', N if r.rows == 'N' else E, sk if r.name == 'node2' and tp.dh == nat.HID else 1.0)
                for r in tp.reductions if r.X is not None]
    return out


def _model(case, dev):
    if case == 'db5':
        return gio.build_model('db5', dev).train()
    if case == 'dips':
        return gio.build_model('dips', dev).train()
    if case == 'dips-ln-drop':
        return nr.build_model('dips', dev, nr.args_with('dips', 'LN', dropout=P_DROP, final_h_layer_norm='LN'),
                              seed=7).train()
    raise ValueError(case)


BACKWARD_CASES = [('db5', 'bench'), ('dips', 'train'), ('dips-ln-drop', 'mid'), ('dips', 'tail1'), ('db5', 'one1')]


@pytest.mark.parametrize('case,batch', BACKWARD_CASES)
def test_backward_reductions_vs_fp64_and_bitwise_fold(case, batch, cuda_device):
    dev = cuda_device
    g, _ = _graph(batch, dev)
    model = _model(case, dev)
    eng = TrainEngine(model)
    torch.manual_seed(3)                 # the dropout seed and the SVD guard's CPU draws
    fwd = eng.forward(g)
    plan = fwd['plan']
    N, E, B = plan.N, plan.E, plan.n_pairs
    if batch == 'tail1':
        assert N < 256 and E % _chunking(E, 64, 64)[0] == 1
    if batch == 'one1':
        assert 1 in plan.n_lig_list and 1 in plan.n_rec_list
    box = [fwd]
    rec = _RecordingLib(eng.lib, eng, box, None)
    eng._ws, eng._ws_plan = BackwardWorkspace(plan, dev, fwd['head'].n_heads), plan    # for _expected_calls' packs
    rec._expected = _expected_calls(eng, N, E)
    eng.lib = rec
    r = _gen(900, dev)
    flat0 = r(eng.layout.total, s=0.01)
    torch.manual_seed(4)
    flat = eng.backward(fwd, r(plan.N_l, 3, s=0.01), r(2 * B, fwd['head'].n_heads, 3, s=0.01).double(),
                        flat=flat0.clone())
    torch.cuda.synchronize()
    assert len(rec.tn) == len(rec._expected)
    if batch == 'bench':
        assert {nch for label, nch, _, _ in rec.tn if 'edge' in label} == {454}

    rows = []
    for label, nch, fp, fc in rec.tn:
        rows.append((f'{label} partial ({nch} chunks)', fp))
        if fc is not None:
            rows.append((f'{label} colsum', fc))
    _report(f'backward[{case}, {batch}] N={N} E={E}', rows)

    # the flat gradient: the reductions' elements bitwise equal to the fold, the rest as it started (except the
    # keypoint key / query projections and the embedding, which other kernels write)
    ref = flat0.cpu().numpy().copy()
    owned = np.zeros(ref.size, bool)
    for vals, dst in rec.reduce:
        assert np.unique(dst).size == dst.size
        _fold(ref, vals, dst)
        owned[dst] = True
    got = flat.cpu().numpy()
    diff = owned & (got.view(np.uint32) != ref.view(np.uint32))
    assert not diff.any(), f'{int(diff.sum())} reduction-owned gradient elements differ from the fp64 fold'
    other = np.zeros(ref.size, bool)
    params = dict(model.named_parameters())
    for name in ('iegmn_original.att_mlp_key_ROT.0.weight', 'iegmn_original.att_mlp_query_ROT.0.weight',
                 'iegmn_original.residue_emb_layer.weight'):
        o = eng.layout.name_offset[name]
        other[o:o + params[name].numel()] = True
    assert not (owned & other).any()
    rest = ~owned & ~other
    assert np.array_equal(got[rest].view(np.uint32), flat0.cpu().numpy()[rest].view(np.uint32)), \
        'elements no reduction owns changed'
    print(f'fold: {len(rec.reduce)} eqd_grad_reduce calls, {int(owned.sum())} elements bitwise equal')


# ---- part 3: one whole layer against fp64 autograd -------------------------------------------------------------------

def _layer_model(kind, dev):
    key = ('layer model', kind)
    if key not in _CACHE:
        if kind == 'dips-ln':
            model = nr.build_model('dips', dev, nr.args_with('dips', 'LN', final_h_layer_norm='LN'), seed=9)
        else:
            model = gio.build_model(kind, dev)
        _CACHE[key] = (model, TrainEngine(model))
    return _CACHE[key]


LAYER_CASES = [('dips', 0, 'bench', False), ('dips', 4, 'bench', False), ('dips', 0, 'train', False),
               ('dips', 4, 'train', False), ('db5', 1, 'bench', False), ('dips-ln', 4, 'bench', False),
               ('dips', 0, 'bench', True)]


@pytest.mark.parametrize('kind,li,batch,drop', LAYER_CASES)
def test_layer_backward_param_grads_vs_fp64(kind, li, batch, drop, cuda_device):
    dev, lib = cuda_device, nat.load()
    g, plan = _graph(batch, dev)
    model, eng = _layer_model(kind, dev)
    mod = model.iegmn_original.iegmn_layers[li]
    lay, tp = mod.packed(dev), eng.layer_pack(mod)
    N, E, B, dh, dhp = plan.N, plan.E, plan.n_pairs, tp.dh, tp.dhp
    desc = nat.EqdLayer.from_buffer_copy(lay.struct)
    desc.dev.leaky_slope = 1.0
    masks = None
    if drop:
        desc.dropout = nat.dropout_descriptor(P_DROP, DROP_SEED, DROP_LAYER, DROP_RANK)
        bm = dm.BatchMasks(P_DROP, DROP_SEED, DROP_RANK, N, E, 1)
        masks = lambda layer, site, w=64: bm(layer, site, w).to(dev)
    skip, eta = float(lay.struct.dev.skip_weight_h), float(lay.struct.dev.x_connection_init)

    r = _gen(3000 + 10 * li + len(batch), dev)
    h0 = r(N, nat.H0)
    h = h0 if li == 0 else r(N, dh, s=0.7)
    x = _coords(g, dev)
    dh_out, dx_out = r(N, 64, s=0.1), r(N, 3).double()

    # fp64 forward and autograd on the same inputs
    p = {k: v.detach().to(F64).clone().requires_grad_(True) for k, v in mod.state_dict().items()}
    src, dst = plan.col_src.long(), plan.edge_dst.long()
    he = torch.cat([plan.he_l[:plan.E_l], plan.he_r[:plan.E_r]]).to(F64)
    seg = np.concatenate([[0], np.cumsum(list(plan.n_lig_list) + list(plan.n_rec_list))]).tolist()
    taps = {}
    x_new, h_new = nr.layer_forward(p, x, h.to(F64), x, h0.to(F64), src, dst, he, seg, B, 1.0, skip, eta, masks,
                                    DROP_LAYER, taps)
    ((x_new * dx_out).sum() + (h_new * dh_out.to(F64)).sum()).backward()

    # the CUDA layer backward with the fp64 forward's aggr / mu as its stash
    pad = lambda t, w: torch.cat([t.float(), torch.zeros(N, w - t.shape[1], device=dev)], 1).contiguous()
    h_in, h0_in = pad(h, dhp), pad(h0, nat.H0_PAD)
    aggr, mu = taps['aggr'].detach().float().contiguous(), pad(taps['mu'].detach(), dhp)
    ws = BackwardWorkspace(plan, dev)
    ws.dh0.zero_()
    flat = torch.zeros(eng.layout.total, device=dev)
    dh_in, dx_in = torch.empty(N, dhp, device=dev), torch.empty(N, 3, dtype=F64, device=dev)
    st = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    tr.layer_backward(lib, plan, lay, tp, ws, h0_in if li == 0 else h_in, x.contiguous(), aggr, mu, h0_in,
                      dh_out.clone(), dx_out.contiguous(), dh_in, dx_in, flat, st, desc=desc)
    torch.cuda.synchronize()

    rep = Report(f'layer_backward[{kind} L{li}, {batch}{", dropout" if drop else ""}] N={N} E={E}')
    for name, prm in mod.named_parameters():
        o = eng.layout.offset[id(prm)]
        rep.rel(name, flat[o:o + prm.numel()].view(prm.shape), p[name].grad)
    rep.check()
