"""Batch collation for the training path: the caller-side data format of Tacotron2.parse_batch (model.py:473-485).

``TextMelCollate`` produces exactly the 5-tuple the reference's collate function produces (data_utils.py:67-111): rows
sorted by decreasing text length (the packed-sequence precondition of Encoder.forward), right zero-padded text / mel,
gate targets that are 1 from the last real frame on, per-row output lengths.  Differences, none visible to train.py:
the padded tensors can be allocated in pinned host memory (``pin_memory=True``) so ``parse_batch``'s ``.cuda(non_blocking
=True)`` copies (utils.to_gpu) are asynchronous, and padding is done with ``pad_sequence`` instead of per-row Python loops.
Audio loading / STFT / text normalisation stay outside this package (SURVEY.md section 8: out of scope)."""
import torch
from torch.nn.utils.rnn import pad_sequence


class TextMelCollate:
    def __init__(self, n_frames_per_step, pin_memory=False):
        self.n_frames_per_step = n_frames_per_step
        self.pin_memory = bool(pin_memory) and torch.cuda.is_available()

    def __call__(self, batch):
        """batch: list of (text (T_i,) int64, mel (n_mel, L_i) float32).  Returns text_padded (B, T_max) int64,
        input_lengths (B) int64 (descending), mel_padded (B, n_mel, L_max') float32, gate_padded (B, L_max') float32,
        output_lengths (B) int64; L_max' = L_max rounded up to a multiple of n_frames_per_step."""
        input_lengths, order = torch.sort(torch.tensor([len(x[0]) for x in batch], dtype=torch.long), dim=0, descending=True)
        order = order.tolist()
        texts = [batch[i][0] for i in order]
        mels = [batch[i][1] for i in order]
        text_padded = pad_sequence([t.long() for t in texts], batch_first=True)                    # (B, T_max)
        output_lengths = torch.tensor([m.size(1) for m in mels], dtype=torch.long)
        max_len = int(output_lengths.max())
        rem = max_len % self.n_frames_per_step
        if rem:
            max_len += self.n_frames_per_step - rem
        mel_padded = pad_sequence([m.t().float() for m in mels], batch_first=True)                  # (B, L_max, n_mel)
        if mel_padded.size(1) < max_len:
            mel_padded = torch.nn.functional.pad(mel_padded, (0, 0, 0, max_len - mel_padded.size(1)))
        mel_padded = mel_padded.transpose(1, 2).contiguous()                                         # (B, n_mel, L_max')
        frame = torch.arange(max_len).unsqueeze(0)
        gate_padded = (frame >= (output_lengths - 1).unsqueeze(1)).float()                           # data_utils.py:107
        out = (text_padded, input_lengths, mel_padded, gate_padded, output_lengths)
        if self.pin_memory:
            out = tuple(t.pin_memory() for t in out)
        return out


class DeviceTextMelCollate:
    """``TextMelCollate`` for samples that already live on the GPU (e.g. mels straight out of ``TacotronSTFT.mel_spectrogram``):
    one concatenation + ``t2_collate`` (rank by text length, pad, gate targets) instead of per-row host loops and five H2D
    copies.  Same 5-tuple as the reference's collate function (data_utils.py:73-111), on the device, no host synchronisation:
    the lengths come from the tensor shapes.  Rows with equal text length keep their input order.

    With ``stft`` (a ``TacotronSTFT`` on the GPU) the samples are ``(text_ids, audio)`` pairs, audio 1-D in [-1, 1] on the
    device (the reference's ``TextMelLoader.get_mel`` with ``load_mel_from_disk=False``): the clips are zero-padded into
    one batch and turned into mels by one ragged ``stft.mel_spectrogram(audio, lengths)`` call, each clip's mel bit for bit
    its own B = 1 call, before the collation.  The range check of that call waits for the GPU once."""

    def __init__(self, n_frames_per_step, stft=None):
        self.n_frames_per_step = n_frames_per_step
        self.stft = stft

    def _mels(self, batch):
        """(text, audio) pairs -> (text, mel) pairs, every mel a (n_mel, n_i // hop + 1) view of one ragged call."""
        audio = [x[1] for x in batch]
        if any(a.dim() != 1 for a in audio):
            raise ValueError("DeviceTextMelCollate: with an stft the samples must be (text, 1-D audio) pairs")
        n = [int(a.numel()) for a in audio]
        y = pad_sequence([a.to(torch.float32) for a in audio], batch_first=True)
        mel = self.stft.mel_spectrogram(y, n)
        hop = self.stft.hop_length
        return [(x[0], mel[b, :, :n[b] // hop + 1]) for b, x in enumerate(batch)]

    def __call__(self, batch):
        import ctypes as C
        from . import _capi
        if self.stft is not None:
            batch = self._mels(batch)
        L = _capi.lib()
        dev = batch[0][1].device
        if dev.type != "cuda":
            raise RuntimeError("DeviceTextMelCollate: the samples must be CUDA tensors (use TextMelCollate for host batches)")
        B, n_mel = len(batch), int(batch[0][1].shape[0])
        tlen, mlen = [int(x[0].numel()) for x in batch], [int(x[1].shape[1]) for x in batch]
        text_flat = torch.cat([x[0].reshape(-1).to(device=dev, dtype=torch.int64) for x in batch])
        mel_flat = torch.cat([x[1].to(dtype=torch.float32).contiguous().reshape(-1) for x in batch])
        off = lambda v: torch.tensor([0] + list(torch.tensor(v).cumsum(0).tolist()), dtype=torch.int64).to(dev, non_blocking=True)
        text_off, mel_off = off(tlen), off(mlen)
        T_max, L_pad = max(tlen), max(mlen)
        if L_pad % self.n_frames_per_step:
            L_pad += self.n_frames_per_step - L_pad % self.n_frames_per_step
        i64, f32 = dict(device=dev, dtype=torch.int64), dict(device=dev, dtype=torch.float32)
        order = torch.empty(B, device=dev, dtype=torch.int32)
        out = (torch.empty(B, T_max, **i64), torch.empty(B, **i64), torch.empty(B, n_mel, L_pad, **f32), torch.empty(B, L_pad, **f32),
               torch.empty(B, **i64))
        a = _capi.T2CollateArgs()
        a.text_flat, a.text_offsets, a.mel_flat, a.mel_offsets = (t.data_ptr() for t in (text_flat, text_off, mel_flat, mel_off))
        a.B, a.n_mel, a.T_max, a.L_pad, a.order = B, n_mel, T_max, L_pad, order.data_ptr()
        a.text_padded, a.input_lengths, a.mel_padded, a.gate_padded, a.output_lengths = (t.data_ptr() for t in out)
        _capi.call(L.t2_collate, dev, C.byref(a))
        self.order = order
        return out
