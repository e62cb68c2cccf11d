"""gemm_bf16 sends a call to the wgmma kernel only when every epilogue tensor has the layout the kernel's vector
and TMA accesses assume: unit column stride and, from N >= 32 on, 16-byte bases and row pitches (x0 and xl
sharing one pitch).  Anything else runs the reference epilogue."""
import torch

from hugectr_b200.ops import gemm as G


def _bf(*shape):
    return torch.zeros(*shape, dtype=torch.bfloat16)


def test_aligned_epilogue_tensors_are_eligible():
    M, N = 64, 96
    assert G.epi_eligible(M, N, _bf(M, N), bias=torch.zeros(N), mask=_bf(M, N), x0=_bf(M, N), xl=_bf(M, N),
                          aux=_bf(M, N))


def test_misaligned_base_or_pitch_is_not_eligible():
    M, N = 64, 96
    big = _bf(M, N + 8)
    assert not G.epi_eligible(M, N, big[:, 1:N + 1])                     # base off by 2 bytes
    assert not G.epi_eligible(M, N, _bf(M, N), x0=_bf(M, N + 4)[:, :N], xl=_bf(M, N))   # pitch 200 B
    assert not G.epi_eligible(M, N, _bf(M, N), mask=_bf(M, N + 4)[:, :N])
    assert not G.epi_eligible(M, N, _bf(M, N), aux=big[:, 1:N + 1])
    assert not G.epi_eligible(M, N, _bf(M, N), bias=torch.zeros(N + 1)[1:])
    assert not G.epi_eligible(M, N, _bf(N, M).t())                       # column stride != 1
    assert not G.epi_eligible(M, N, _bf(M, N), x0=_bf(M, N + 8)[:, :N], xl=_bf(M, N))   # x0 / xl pitches differ


def test_narrow_outputs_need_no_vector_alignment():
    # below 32 columns the kernel's epilogue uses scalar accesses only (e.g. the N = 1 output layer)
    M = 64
    assert G.epi_eligible(M, 1, _bf(M, 1), bias=torch.zeros(1))
    assert G.epi_eligible(M, 24, _bf(M, 25)[:, 1:])
