"""The gradient kernels of the degradations, executed from their CUDA source on the CPU (tests/simt_cpu) and compared with
float64 numpy: cd_blur_apply_adjoint (A^T G A per plane, one CTA per plane up to 128², row strips above) and cd_lerp2_adjoint
(both gradients of the noise / fade lerps).

The adjoint is checked two ways: against float64 A^T G A, and through the adjoint identity <A X A^T, G> = <X, A^T G A> with
the emulated forward.  The operators are dense random matrices and the Exponential_reflect blur operators; neither is
symmetric, so an operator that was not transposed shows.  S = 132 leaves a partial strip, ring chunk and 128-column slice;
the S = 256 cases run one plane product each (the emulator takes about a second per strip product there)."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(__file__), 'simt_cpu'))

from test_blur_large_cpu import P, images, operators, ref_apply  # noqa: E402


@pytest.fixture(scope='module', params=['ascending', 'descending'])
def lib(request):
    """threads of a block resumed in ascending / descending order: a missing barrier shows under at least one of them"""
    import build
    lib = C.CDLL(build.build_all())
    lib.simt_set_reverse_order(int(request.param == 'descending'))
    yield lib
    lib.simt_set_reverse_order(0)


def ref_adjoint(g, ops, idx, collapse=False):
    """float64 A_idx^T G A_idx per plane (idx < 0: G); collapse: G -> mean(G) 11^T first"""
    G = g.double().numpy()
    if idx < 0:
        return G
    if collapse:
        G = np.broadcast_to(G.mean(axis=(-2, -1), keepdims=True), G.shape)
    A = ops[idx].double().numpy()
    return np.einsum('ji,...jk,kl->...il', A, G, A)


def apply(lib, x, ops, t=None, t_scalar=0, collapse=0):
    B, Cc, S, _ = x.shape
    out = torch.full_like(x, float('nan'))
    assert lib.cd_blur_apply(P(x), P(out), P(ops), P(t), t_scalar, B, Cc, S, ops.shape[0], collapse, 0, C.c_void_p(0)) == 0
    return out


def adjoint(lib, g, ops, t=None, t_scalar=0, collapse=0):
    B, Cc, S, _ = g.shape
    out = torch.full_like(g, float('nan'))
    assert lib.cd_blur_apply_adjoint(P(g), P(out), P(ops), P(t), t_scalar, B, Cc, S, ops.shape[0], collapse, C.c_void_p(0)) == 0
    return out


def rel(got, want):
    want = np.asarray(want, dtype=np.float64)
    return float(np.abs(got.double().numpy() - want).max() / max(1e-30, np.abs(want).max()))


def dot(a, b):
    return float((a.double() * b.double()).sum())


def shape_of(S):
    """(t, channels): three samples with a t = -1 row up to 132, one product plane at 256"""
    return (torch.tensor([2, -1, 0], dtype=torch.int64), 2) if S <= 132 else (torch.tensor([-1, 2], dtype=torch.int64), 1)


@pytest.mark.parametrize('S,kind', [(32, 'blur'), (32, 'dense'), (128, 'dense'), (132, 'blur'), (132, 'dense'), (256, 'dense')])
def test_adjoint_per_sample_t(lib, S, kind):
    T = 4
    ops = operators(S, T, kind, seed=11)
    t, Cc = shape_of(S)
    g = images(len(t), Cc, S, seed=12)
    out = adjoint(lib, g, ops, t=t)
    for b in range(len(t)):
        assert rel(out[b], ref_adjoint(g[b], ops, int(t[b]))) < 2e-6, b
        if int(t[b]) >= 0:                                                   # the forward operator is not the answer
            assert rel(out[b], ref_apply(g[b], ops, int(t[b]))) > 1e-2, b
    assert torch.equal(out[t == -1], g[t == -1])                             # t = -1 copies the plane
    # <A X A^T, G> = <X, A^T G A> with the emulated forward
    x = images(len(t), Cc, S, seed=13)
    lhs, rhs = dot(apply(lib, x, ops, t=t), g), dot(x, out)
    assert abs(lhs - rhs) < 1e-5 * (abs(lhs) + abs(rhs) + 1), (lhs, rhs)


@pytest.mark.parametrize('S', [32, 132])
def test_adjoint_scalar_index(lib, S):
    ops = operators(S, 3, 'dense', seed=14)
    g = images(2, 2, S, seed=15)
    assert rel(adjoint(lib, g, ops, t_scalar=1), ref_adjoint(g, ops, 1)) < 2e-6
    assert torch.equal(adjoint(lib, g, ops, t_scalar=-1), g)


@pytest.mark.parametrize('S,kind', [(32, 'blur'), (128, 'dense'), (132, 'blur'), (132, 'dense')])
def test_adjoint_collapse(lib, S, kind):
    """`discrete`: at t = T-1 the forward replaces the plane by its mean, so the adjoint maps G to A^T (mean(G) 11^T) A; the
    other planes are untouched by the option, and the identity holds against the collapsing forward"""
    T = 3
    ops = operators(S, T, kind, seed=16)
    t = torch.tensor([T - 1, 1, -1], dtype=torch.int64)
    g = images(3, 2, S, seed=17)
    plain = adjoint(lib, g, ops, t=t)
    coll = adjoint(lib, g, ops, t=t, collapse=1)
    assert rel(coll[0], ref_adjoint(g[0], ops, T - 1, collapse=True)) < 2e-6
    assert rel(coll[0], ref_adjoint(g[0], ops, T - 1)) > 1e-2                 # the collapse was applied
    assert torch.equal(coll[1:], plain[1:])
    x = images(3, 2, S, seed=18)
    lhs, rhs = dot(apply(lib, x, ops, t=t, collapse=1), g), dot(x, coll)
    assert abs(lhs - rhs) < 1e-5 * (abs(lhs) + abs(rhs) + 1), (lhs, rhs)


def test_adjoint_refuses_unsupported_sizes(lib):
    for S in (516, 130):
        g = torch.zeros(1, 1, S, S)
        ops = torch.zeros(1, S, S)
        assert lib.cd_blur_apply_adjoint(P(g), P(g.clone()), P(ops), P(None), 0, 1, 1, S, 1, 0, C.c_void_p(0)) != 0
        buf = C.create_string_buffer(512)
        lib.cd_last_error(buf, 512)
        assert b'cd_blur_apply_adjoint: image size %d unsupported' % S in buf.value


# ---- cd_lerp2_adjoint ----------------------------------------------------------------------------------------------------
def lerp2_adjoint(lib, g, t, t_scalar, wa, wb, per_pixel, want=(True, True)):
    B, Cc, H, W = g.shape
    ga = torch.full_like(g, float('nan')) if want[0] else None
    gb = torch.full_like(g, float('nan')) if want[1] else None
    assert lib.cd_lerp2_adjoint(P(g), P(t), t_scalar, P(wa), P(wb), B, Cc, C.c_int64(H * W), per_pixel, P(ga), P(gb),
                                C.c_void_p(0)) == 0
    return ga, gb


def test_lerp2_adjoint_per_sample():
    """cd_noise_lerp's coefficients: one scalar per sample from the [T] tables"""
    import build
    lib = C.CDLL(build.build_all())
    gen = torch.Generator().manual_seed(20)
    T, B, Cc, S = 7, 3, 3, 12
    wa, wb = torch.rand(T, generator=gen), torch.rand(T, generator=gen)
    g = torch.randn(B, Cc, S, S, generator=gen)
    t = torch.tensor([4, 0, 6], dtype=torch.int64)
    ga, gb = lerp2_adjoint(lib, g, t, 0, wa, wb, 0)
    wa64, wb64 = wa.double()[t].view(-1, 1, 1, 1), wb.double()[t].view(-1, 1, 1, 1)
    assert rel(ga, wa64 * g.double()) < 1e-7 and rel(gb, wb64 * g.double()) < 1e-7
    assert rel(gb, wa64 * g.double()) > 1e-2                                  # the coefficients are not swapped
    ga, gb = lerp2_adjoint(lib, g, None, 5, wa, wb, 0, want=(False, True))
    assert ga is None and rel(gb, float(wb[5]) * g.double()) < 1e-7


def test_lerp2_adjoint_per_pixel():
    """cd_fade_lerp's coefficients: [T][H][W] tables indexed by the sample's t and the pixel"""
    import build
    lib = C.CDLL(build.build_all())
    gen = torch.Generator().manual_seed(21)
    T, B, Cc, S = 5, 2, 3, 8
    wa, wb = torch.rand(T, S, S, generator=gen), torch.rand(T, S, S, generator=gen)
    g = torch.randn(B, Cc, S, S, generator=gen)
    t = torch.tensor([3, 1], dtype=torch.int64)
    ga, gb = lerp2_adjoint(lib, g, t, 0, wa, wb, 1)
    assert rel(ga, wa.double()[t][:, None] * g.double()) < 1e-7
    assert rel(gb, wb.double()[t][:, None] * g.double()) < 1e-7
    assert rel(ga, wa.double()[t].transpose(1, 2)[:, None] * g.double()) > 1e-2    # the pixel index is not transposed
    ga, gb = lerp2_adjoint(lib, g, None, 2, wa, wb, 1, want=(True, False))
    assert gb is None and rel(ga, wa.double()[2] * g.double()) < 1e-7
