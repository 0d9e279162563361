"""GPU tests of the spconv drop-in (gs_b200.spconv, csrc/sp_conv.cu) against the float64 oracle
(oracle/spconv_oracle.py).  The neighbour map must equal the oracle's brute-force map element for element; outputs and
gradients must lie within the rounding bound of their summation, |got - ref| <= gamma * sum |W| |x| with
gamma = (terms + 1) * 2^-24 (+ 2^-11 |ref| for the one rounding to fp16), and repeat with the same bits."""
import numpy as np
import pytest
import torch

from oracle import spconv_oracle as O

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
U = 2.0 ** -24

# TRELLIS / Stable3DGen channel pairs: SLat flow io blocks and the mesh decoder's subdivision stages
TRELLIS_PAIRS = [(128, 128), (128, 1024), (1024, 1024), (2048, 128), (256, 128), (768, 192), (192, 192), (192, 96),
                 (96, 96)]


def _S():
    from gs_b200 import spconv
    return spconv


def _sp():
    import spconv.pytorch as sp
    return sp


def _t(a, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    return t.to(dtype) if dtype is not None else t


def _np(t):
    return t.detach().float().cpu().numpy().astype(np.float64)


def _case(name):
    return next((i, s, b) for n, i, s, b in O.edge_sets() if n == name)


def _inputs(rng, N, Cin, Cout, k, dtype):
    x = _t(rng.standard_normal((N, Cin)).astype(np.float32), dtype)
    w = _t((rng.uniform(-1, 1, (Cout, k, k, k, Cin)) / np.sqrt(k ** 3 * Cin)).astype(np.float32), dtype)
    b = _t(rng.uniform(-1, 1, Cout).astype(np.float32), dtype)
    return x, w, b


def _check(got, ref, bound, terms, fp16, what):
    g = _np(got)
    tol = (terms + 1) * U * bound + (2.0 ** -11 * np.abs(ref) if fp16 else 0)
    err = np.abs(g - ref)
    bad = np.argwhere(~(err <= tol))
    assert bad.size == 0, f"{what}: {len(bad)} outside the bound, first {bad[:3].tolist()}, err {err.max():.3g}"


def _fwd(ind, spatial, B, x, w, b, k):
    S = _S()
    m = S.build_map(_t(ind), spatial, B, k)
    return S.submconv3d(x, w, b, m), m


@pytest.mark.parametrize("name", [s[0] for s in O.edge_sets()])
def test_map_equals_brute_force(name):
    ind, spatial, B = _case(name)
    m = _S().build_map(_t(ind), spatial, B, 3)
    want = O.brute_map(ind, spatial, B, 3)
    got = m.nbr.cpu().numpy()
    assert (got == want).all(), f"{name}: {(got != want).sum()} entries differ, first {np.argwhere(got != want)[:3].tolist()}"
    mask = m.mask.cpu().numpy().view(np.uint32)
    bits = ((want >= 0) << np.arange(27)).sum(1).astype(np.uint32)
    assert (mask & 0x07FFFFFF == bits).all()
    dup = np.array([want[i, 13] not in (-1, i) for i in range(len(ind))])
    assert ((mask >> 31).astype(bool) == dup).all()


def test_map_on_subdivided_shell():
    rng = np.random.default_rng(0)
    ind = O.subdivide(O.sphere_shell(32, batch=2))
    ind = ind[rng.permutation(len(ind))]
    m = _S().build_map(_t(ind), (64, 64, 64), 2, 3)
    assert (m.nbr.cpu().numpy() == O.brute_map(ind, (64, 64, 64), 2, 3)).all()


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("k", [1, 3])
@pytest.mark.parametrize("cin,cout", [(1, 1), (3, 13), (13, 3), (96, 129), (129, 96), (8, 40)])
def test_forward_channels(dtype, k, cin, cout):
    rng = np.random.default_rng(cin * 1000 + cout)
    ind, spatial, B = _case("random_dups_unsorted")
    x, w, b = _inputs(rng, len(ind), cin, cout, k, dtype)
    out, m = _fwd(ind, spatial, B, x, w, b, k)
    ref, bound = O.forward(_np(x), _np(w), _np(b), O.brute_map(ind, spatial, B, k))
    _check(out, ref, bound, k ** 3 * cin, dtype == torch.float16, f"{dtype} k{k} {cin}->{cout}")


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("cin,cout", TRELLIS_PAIRS)
def test_forward_trellis_pairs(dtype, cin, cout):
    rng = np.random.default_rng(cin + cout)
    ind = O.sphere_shell(24)
    ind = ind[rng.permutation(len(ind))][:700]
    x, w, b = _inputs(rng, len(ind), cin, cout, 3, dtype)
    out, _ = _fwd(ind, (24, 24, 24), 1, x, w, b, 3)
    ref, bound = O.forward(_np(x), _np(w), _np(b), O.brute_map(ind, (24, 24, 24), 1, 3))
    _check(out, ref, bound, 27 * cin, dtype == torch.float16, f"{dtype} {cin}->{cout}")


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("name", [s[0] for s in O.edge_sets()])
def test_forward_edge_sets(dtype, name):
    ind, spatial, B = _case(name)
    rng = np.random.default_rng(5)
    x, w, b = _inputs(rng, len(ind), 24, 40, 3, dtype)
    out, _ = _fwd(ind, spatial, B, x, w, b, 3)
    ref, bound = O.forward(_np(x), _np(w), _np(b), O.brute_map(ind, spatial, B, 3))
    _check(out, ref, bound, 27 * 24, dtype == torch.float16, f"{dtype} {name}")


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_isolated_is_centre_tap_plus_bias(dtype):
    ind, spatial, B = _case("isolated")
    rng = np.random.default_rng(1)
    x, w, b = _inputs(rng, len(ind), 16, 8, 3, dtype)
    out, _ = _fwd(ind, spatial, B, x, w, b, 3)
    ref = _np(x) @ _np(w)[:, 1, 1, 1, :].T + _np(b)
    bound = np.abs(_np(x)) @ np.abs(_np(w)[:, 1, 1, 1, :]).T + np.abs(_np(b))
    _check(out, ref, bound, 16, dtype == torch.float16, "isolated")


@pytest.mark.parametrize("k", [1, 3])
def test_empty_input(k):
    S = _S()
    m = S.build_map(torch.zeros(0, 4, dtype=torch.int32, device=DEV), (4, 4, 4), 1, k)
    x = torch.zeros(0, 5, device=DEV, requires_grad=True)
    w = torch.randn(7, k, k, k, 5, device=DEV, requires_grad=True)
    b = torch.randn(7, device=DEV, requires_grad=True)
    out = S.submconv3d(x, w, b, m)
    assert out.shape == (0, 7)
    out.sum().backward()
    assert x.grad.shape == (0, 5) and float(w.grad.abs().sum()) == 0 and float(b.grad.abs().sum()) == 0


def test_noncontiguous_inference_mode_side_stream():
    ind, spatial, B = _case("faces_unsorted")
    rng = np.random.default_rng(2)
    x, w, b = _inputs(rng, len(ind), 32, 16, 3, torch.float16)
    ref, _ = _fwd(ind, spatial, B, x, w, b, 3)
    wide = torch.zeros(len(ind), 64, dtype=torch.float16, device=DEV)
    wide[:, 1:33] = x
    xs = wide[:, 1:33]
    assert not xs.is_contiguous()
    with torch.inference_mode():
        out1, _ = _fwd(ind, spatial, B, xs, w, b, 3)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        out2, _ = _fwd(ind, spatial, B, x, w, b, 3)
    s.synchronize()
    assert torch.equal(out1, ref) and torch.equal(out2, ref)


def _backward(ind, spatial, B, x, w, b, k, go):
    x, w, b = (t.detach().clone().requires_grad_(True) for t in (x, w, b))
    out, _ = _fwd(ind, spatial, B, x, w, b, k)
    out.backward(go)
    return x.grad, w.grad, b.grad


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("k", [1, 3])
@pytest.mark.parametrize("name,cin,cout", [("shell16", 13, 29), ("shell16", 64, 96), ("faces_unsorted", 96, 32),
                                           ("random_dups_unsorted", 40, 24), ("outside_rows", 8, 8)])
def test_backward(dtype, k, name, cin, cout):
    if dtype == torch.float16 and name == "random_dups_unsorted":
        pytest.skip("fp16 rounds the duplicates' summed upstream gradient once more; fp32 covers duplicates")
    ind, spatial, B = _case(name)
    rng = np.random.default_rng(cin * cout + k)
    x, w, b = _inputs(rng, len(ind), cin, cout, k, dtype)
    go = _t(rng.standard_normal((len(ind), cout)).astype(np.float32), dtype)
    gx, gw, gb = _backward(ind, spatial, B, x, w, b, k, go)
    gx2, gw2, gb2 = _backward(ind, spatial, B, x, w, b, k, go)
    assert torch.equal(gx, gx2) and torch.equal(gw, gw2) and torch.equal(gb, gb2), "backward bits differ between runs"
    dx, dW, db, dxb, dWb = O.backward(_np(x), _np(w), O.brute_map(ind, spatial, B, k), _np(go))
    f16 = dtype == torch.float16
    N = len(ind)
    _check(gx, dx, dxb, k ** 3 * cout + 8, f16, "dgrad")
    _check(gw, dW, dWb, N + 256, f16, "wgrad")
    _check(gb, db, np.abs(_np(go)).sum(0), N + 256, f16, "dbias")


def test_wgrad_many_chunks():
    rng = np.random.default_rng(9)
    ind = O.subdivide(O.sphere_shell(24))
    ind = ind[rng.permutation(len(ind))]
    x, w, b = _inputs(rng, len(ind), 16, 16, 3, torch.float32)
    go = _t(rng.standard_normal((len(ind), 16)).astype(np.float32))
    gx, gw, gb = _backward(ind, (48, 48, 48), 1, x, w, b, 3, go)
    dx, dW, db, dxb, dWb = O.backward(_np(x), _np(w), O.brute_map(ind, (48, 48, 48), 1, 3), _np(go))
    _check(gx, dx, dxb, 27 * 16, False, "dgrad")
    _check(gw, dW, dWb, len(ind) + 256, False, "wgrad")
    _check(gb, db, np.abs(_np(go)).sum(0), len(ind) + 256, False, "dbias")


def test_trellis_subdivide_block_pattern(monkeypatch):
    """SparseSubdivideBlock3d on the spconv backend: the tensor built as SparseTensor.__init__ / replace build it, a
    3x3x3 -> 3x3x3 pair on one indice_key plus the 1x1 skip, all in fp16.  The map is built once and the cached-map
    output has the same bits as fresh maps."""
    sp, S = _sp(), _S()
    torch.manual_seed(0)
    coords = _t(O.subdivide(O.sphere_shell(16, batch=2)))
    feats = torch.randn(coords.shape[0], 96, device=DEV, dtype=torch.float16)
    spatial_shape = list(coords.max(0)[0] + 1)[1:]
    data = sp.SparseConvTensor(feats.reshape(feats.shape[0], -1), coords, spatial_shape, 2)
    data._features = feats
    conv1 = sp.SubMConv3d(96, 48, 3, indice_key="res_32", algo=sp.ConvAlgo.Native).to(DEV).half()
    conv2 = sp.SubMConv3d(48, 48, 3, indice_key="res_32", algo=sp.ConvAlgo.Native).to(DEV).half()
    skip = sp.SubMConv3d(96, 48, 1, indice_key="res_32").to(DEV).half()
    calls = []
    real = S.build_map
    monkeypatch.setattr(S, "build_map", lambda *a, **kw: calls.append(a[-1] if len(a) > 3 else 3) or real(*a, **kw))

    def replace(d, f):
        new = sp.SparseConvTensor(d.features.reshape(d.features.shape[0], -1), d.indices, d.spatial_shape,
                                  d.batch_size, d.grid, d.voxel_num, d.indice_dict)
        new._features = f
        return new

    h = conv1(data)
    h = replace(h, torch.nn.functional.silu(h.features))
    h = conv2(h)
    out = h.features + skip(data).features
    assert calls.count(3) == 1, calls
    assert "res_32" in data.indice_dict
    m = S.build_map(coords, spatial_shape, 2, 3)
    fresh = S.submconv3d(torch.nn.functional.silu(S.submconv3d(feats, conv1.weight, conv1.bias, m)), conv2.weight,
                         conv2.bias, S.build_map(coords, spatial_shape, 2, 3)) + \
        S.submconv3d(feats, skip.weight, skip.bias, S.build_map(coords, spatial_shape, 2, 1))
    assert torch.equal(out, fresh)
