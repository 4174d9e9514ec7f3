"""Ragged log-mel extraction without a GPU: the C layout of T2MelSpecArgs.lengths, the workspace queries, and the host
validation of ``TacotronSTFT.mel_spectrogram``'s lengths."""
import pytest
import torch

import tacotron2_b200 as t2
from tacotron2_b200 import _capi
from tacotron2_b200.layers import _sample_lengths


def test_workspace_queries():
    """The query with lengths covers the frame counts and the per-row scales of both products; the one without is the
    size it always was, which a NULL-lengths call keeps needing."""
    L = _capi.lib()
    for B, n in [(1, 513), (7, 67150), (64, 220500)]:
        plain = L.t2_mel_spectrogram_workspace_bytes(B, n, 1024, 256, 80)
        ragged = L.t2_mel_spectrogram_workspace_bytes_lengths(B, n, 1024, 256, 80)
        F = n // 256 + 1
        signal = B * (n + 1024 + F * (2 * 513 + 513 + 80)) * 4
        assert plain > signal and ragged >= signal + (B * F + 1026) * 4 + B * 4


def test_lengths_are_validated_on_the_host():
    assert _sample_lengths([513, 2000], 2, 2000, 1024) == [513, 2000]
    assert _sample_lengths(torch.tensor([600, 700], dtype=torch.int16), 2, 2000, 1024) == [600, 700]
    with pytest.raises(ValueError, match="length 512 of row 1"):
        _sample_lengths([513, 512], 2, 2000, 1024)
    with pytest.raises(ValueError, match="length 2001 of row 0"):
        _sample_lengths([2001, 513], 2, 2000, 1024)
    with pytest.raises(ValueError):
        _sample_lengths([600], 2, 2000, 1024)
    with pytest.raises(ValueError):
        _sample_lengths(torch.tensor([[600, 600]]), 2, 2000, 1024)
    for bad in (torch.tensor([600.0, 600.0]), torch.tensor([True, True]), [600, 600.0]):
        with pytest.raises(TypeError):
            _sample_lengths(bad, 2, 2000, 1024)


def test_mel_spectrogram_with_lengths_needs_cuda():
    with pytest.raises(RuntimeError, match="CUDA"):
        t2.TacotronSTFT().mel_spectrogram(torch.zeros(2, 2000), [600, 2000])
