"""The finality window behind the streams that follow ``Tacotron2.inference_stream`` (``WaveGlow.infer_stream``,
``Denoiser.stream``): what an item makes final, the window a stage runs over, and what the stream must keep."""
import torch


class FinalWindow:
    """Input that arrives in consecutive items along `axis`, for an output whose unit t (`unit` input elements) depends
    on the input units t - left ... t + right.  While the stream goes on, the output up to the held input less `right`
    units is final; once it has finished, all of it is.  The window of a final span is every kept element, [base, held):
    the buffer keeps only the input later windows can still need, at most the two halos plus one item."""

    def __init__(self, what, key, axis, left, right, unit=1):
        self.what, self.key, self.axis, self.left, self.right, self.unit = what, key, axis, left, right, unit
        self.kept = None
        self.base = self.held = 0       # kept holds the input elements [base, held)
        self.done = 0                   # the output units [0, done) are final and handed out

    def check(self, item):
        """Raises unless item[key], the item's input span (s0, s1), starts where the input held so far ends."""
        if item[self.key][0] != self.held:
            raise ValueError("%s must be consecutive (%s %s after %d)" % (self.what, self.key, item[self.key], self.held))

    def add(self, item, x):
        """Appends x, the data of a checked item, to the kept input: the first x is kept as it is, later ones take its
        device and dtype.  Returns the output units (d0, d1) the item makes final, or None when it makes none and the
        stream goes on."""
        if self.kept is None:
            self.kept = x
        else:
            drop = self.unit * max(0, self.done - self.left) - self.base      # no later window starts before done - left
            kept = self.kept.narrow(self.axis, drop, self.kept.shape[self.axis] - drop)
            self.kept = torch.cat((kept, x.to(device=kept.device, dtype=kept.dtype)), self.axis)
            self.base += drop
        self.held = item[self.key][1]
        finished, n = bool(item["finished"]), self.held // self.unit
        d0, d1 = self.done, n if finished else max(self.done, n - self.right)
        if d1 == d0 and not finished:
            return None
        self.done = d1
        return d0, d1

    def lengths(self, lengths, open_end):
        """Window-relative row ends, int32 on the kept input's device, from lengths (B,) in units with -1 for live rows:
        row b ends at unit * lengths[b] - base, or at 0 when that is before the window.  A live row, or one that ends
        past the window, gets `open_end`: how the stage's library marks a row that runs through the window."""
        lengths = lengths.to(self.kept.device)
        ends = (self.unit * lengths - self.base).clamp(min=0)
        past = (lengths < 0) | (ends > self.held - self.base)
        return torch.where(past, torch.full_like(lengths, open_end), ends).to(torch.int32).contiguous()
