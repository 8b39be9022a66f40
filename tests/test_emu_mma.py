"""tests/emu/host_emu.h's mma_tf32 (the model every tensor-core kernel's emulator test rests on) against a plain 16 x 8
x 8 product.  The fragments are laid out here from the PTX ISA's tables for mma.m16n8k8 with .tf32 operands
(groupID = lane >> 2, tig = lane % 4):
  A: a_i at row groupID + 8 (i % 2), column tig + 4 (i // 2)
  B: b_i at row tig + 4 i, column groupID
  C, D: c_i at row groupID + 8 (i // 2), column 2 tig + i % 2"""
import pytest
import torch

from tests.emu_harness import shared


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    return shared("emu_mma.cpp", tmp_path_factory)


def a_at(lane, i):
    return (lane >> 2) + 8 * (i % 2), (lane & 3) + 4 * (i // 2)


def b_at(lane, i):
    return (lane & 3) + 4 * i, lane >> 2


def c_at(lane, i):
    return (lane >> 2) + 8 * (i // 2), 2 * (lane & 3) + i % 2


def _run(lib, A, Bm, C):
    a = torch.tensor([[A[a_at(l, i)] for i in range(4)] for l in range(32)], dtype=torch.float32)
    b = torch.tensor([[Bm[b_at(l, i)] for i in range(2)] for l in range(32)], dtype=torch.float32)
    d = torch.tensor([[C[c_at(l, i)] for i in range(4)] for l in range(32)], dtype=torch.float32)
    assert lib.emu_mma_tf32(a.data_ptr(), b.data_ptr(), d.data_ptr()) == 0
    D = torch.empty(16, 8, dtype=torch.float32)
    for l in range(32):
        for i in range(4):
            D[c_at(l, i)] = d[l, i]
    return D


def _tf32(x):
    return (x.float().view(torch.int32) & -0x2000).view(torch.float32).double()


def test_product_against_a_plain_loop(lib):
    """random fp32 operands with all mantissa bits set: D = trunc_tf32(A) trunc_tf32(B) + C, summed exactly and rounded
    once to fp32"""
    g = torch.Generator().manual_seed(0)
    A, Bm, C = (torch.randn(*s, generator=g) for s in ((16, 8), (8, 8), (16, 8)))
    D = _run(lib, A, Bm, C)
    ref = torch.zeros(16, 8, dtype=torch.float64)
    for r in range(16):
        for n in range(8):
            ref[r, n] = C[r, n].double() + sum(_tf32(A[r, k]) * _tf32(Bm[k, n]) for k in range(8))
    assert torch.equal(D, ref.float())
    assert not torch.equal(D, (A.double() @ Bm.double() + C.double()).float())   # the truncation is there


@pytest.mark.parametrize("lane", range(32))
def test_each_fragment_register_lands_where_the_isa_says(lib, lane):
    """one nonzero A register (lane, i) times a one-hot B column picks out exactly the D element of (row, column)"""
    for i in range(4):
        r, k = a_at(lane, i)
        n = (r + k) % 8
        A, Bm, C = torch.zeros(16, 8), torch.zeros(8, 8), torch.zeros(16, 8)
        A[r, k], Bm[k, n] = 3.0, 0.5
        D = _run(lib, A, Bm, C)
        want = torch.zeros(16, 8)
        want[r, n] = 1.5
        assert torch.equal(D, want), (lane, i, r, k, n)
