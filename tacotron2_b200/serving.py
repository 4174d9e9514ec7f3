"""Continuous batching for Tacotron2 inference: a fixed number of decoder rows ("slots") stays in flight, and a slot whose
request has stopped takes the next queued text at the next chunk boundary.

``InferenceServer`` is the scheduler: the FIFO queue, the slot table, each request's step count and limit, the per-chunk
prenet mask and the hand-over of results.  It is plain Python over a backend object and imports without CUDA; the backend
that drives the engine is ``EngineBackend`` (``Tacotron2.inference_server`` builds both).

Step numbering: every chunk runs as local steps [0, n) of the resumable decoder into chunk-sized buffers.  The decoder
kernel keeps no step counter in its saved state, so a slot's position in its own request is known to the scheduler alone:
request r that has run s steps has, in the next chunk, its step s + i at local step i.

Seeded requests (``submit(..., seed=s)``) draw the prenet dropout of ``inference(text[None], seeds=[s])``: each chunk
hands the kernel every slot's seed and its request's step count s, and the slot's local step i draws its request's step
s + i under that seed."""
import collections
import numbers

import torch

from ._engine import seed_pattern

WARNING = "Warning! Reached max decoder steps"      # the line Decoder.inference prints (model.py:446)


class Request:
    """One queued or running utterance."""

    def __init__(self, rid, text, limit, keep, seed=None):
        self.id, self.text, self.limit, self.keep, self.seed = rid, text, limit, keep, seed
        self.steps = 0            # decoder steps of this request that earlier chunks ran
        self.slot = None
        self.out = None           # the backend's output buffers of this request
        self.length = None        # frames, once it has left its slot
        self.hit_max_steps = False


def chunk_seed(session_seed, chunk_index):
    """Philox seed of one chunk: the session's seed advanced by a 64-bit odd constant per chunk, so no two chunks of a
    session draw the same stream although each numbers its steps from 0."""
    return (session_seed + 0x9E3779B97F4A7C15 * (chunk_index + 1)) & 0xFFFFFFFFFFFFFFFF


class InferenceServer:
    """slots decoder rows in flight over a FIFO queue of texts.

    ``submit`` queues a text, ``step`` runs one chunk and returns the requests that finished in it, ``run`` steps until
    the queue is empty and every slot is idle.  backend: ``admit(pairs)``, ``launch(n, chunk_index, keep, slots)``,
    ``collect(entries)``, ``read()`` and ``finish(requests)`` (see EngineBackend)."""

    def __init__(self, backend, slots, max_text_len, chunk_steps, max_decoder_steps):
        slots, max_text_len, chunk_steps = int(slots), int(max_text_len), int(chunk_steps)
        if slots < 1:
            raise ValueError("tacotron2_b200: slots must be >= 1 (got %d)" % slots)
        if max_text_len < 1:
            raise ValueError("tacotron2_b200: max_text_len must be >= 1 (got %d)" % max_text_len)
        if chunk_steps < 1:
            raise ValueError("tacotron2_b200: chunk_steps must be >= 1 (got %d)" % chunk_steps)
        self.backend = backend
        self.slots, self.max_text_len, self.chunk_steps = slots, max_text_len, chunk_steps
        self.max_decoder_steps = int(max_decoder_steps)
        self.queue = collections.deque()
        self.table = [None] * slots          # slot -> Request
        self.injected = None                 # whether this session's requests carry prenet masks (fixed by the first)
        self.seeded = None                   # whether they carry seeds (fixed by the first)
        self.chunks = 0                      # chunks launched
        self.row_steps = 0                   # slots x decoder steps launched, over 64-row slices that ran
        self._next_id = 0

    # -- queue --------------------------------------------------------------------------------------
    def submit(self, text_ids, max_decoder_steps=None, prenet_keep=None, seed=None):
        """Queues one text: a 1-D integer tensor of 1..max_text_len symbol ids.  max_decoder_steps: this request's own
        limit (default: the model's).  Returns the request id.  Everything is checked here, before anything runs.

        seed: an integer in [0, 2**64).  The request then equals ``inference(text_ids[None], seeds=[seed])`` under its own
        limit, bit for bit, whatever slot, chunk or neighbours it gets, and its result carries ``seed``.

        prenet_keep is the test hook, the counterpart of ``dropout_masks(prenet=...)``: this request's (steps, 2, 256)
        uint8 keep mask with steps >= its limit; row t is the mask of its own step t.  A session takes masks for all of
        its requests or for none, and likewise seeds."""
        if not torch.is_tensor(text_ids):
            text_ids = torch.as_tensor(text_ids)
        if text_ids.dtype.is_floating_point or text_ids.dtype.is_complex or text_ids.dtype == torch.bool:
            raise TypeError("tacotron2_b200: text_ids must hold integers (got %s)" % text_ids.dtype)
        if text_ids.dim() != 1:
            raise ValueError("tacotron2_b200: text_ids must be 1-D (got shape %s)" % (tuple(text_ids.shape),))
        n = int(text_ids.numel())
        if n < 1:
            raise ValueError("tacotron2_b200: text_ids is empty")
        if n > self.max_text_len:
            raise ValueError("tacotron2_b200: text of %d symbols is longer than this server's max_text_len = %d"
                             % (n, self.max_text_len))
        limit = self.max_decoder_steps if max_decoder_steps is None else int(max_decoder_steps)
        if limit < 1:
            raise ValueError("tacotron2_b200: max_decoder_steps must be >= 1 (got %d)" % limit)
        if prenet_keep is not None:
            if prenet_keep.dim() != 3 or tuple(prenet_keep.shape[1:]) != (2, 256) or prenet_keep.shape[0] < limit:
                raise ValueError("tacotron2_b200: prenet_keep must have shape (steps >= %d, 2, 256) (got %s)"
                                 % (limit, tuple(prenet_keep.shape)))
            prenet_keep = prenet_keep.to(device="cpu", dtype=torch.uint8).contiguous()
        if seed is not None:
            if torch.is_tensor(seed):
                if seed.numel() != 1 or seed.dtype == torch.bool or seed.dtype.is_floating_point or seed.dtype.is_complex:
                    raise TypeError("tacotron2_b200: seed must be one integer (got a %s tensor of shape %s)"
                                    % (seed.dtype, tuple(seed.shape)))
                seed = int(seed.item()) & 0xFFFFFFFFFFFFFFFF if seed.dtype == torch.int64 else int(seed.item())
            if isinstance(seed, bool) or not isinstance(seed, numbers.Integral):
                raise TypeError("tacotron2_b200: seed must be an integer (got %r)" % (seed,))
            seed = int(seed)
            seed_pattern(seed, "tacotron2_b200")
            if prenet_keep is not None:
                raise ValueError("tacotron2_b200: seed and prenet_keep exclude each other")
        if self.seeded is None:
            self.seeded = seed is not None
        elif self.seeded != (seed is not None):
            raise ValueError("tacotron2_b200: a server takes a seed for every request or for none")
        if self.injected is None:
            self.injected = prenet_keep is not None
        elif self.injected != (prenet_keep is not None):
            raise ValueError("tacotron2_b200: a server takes prenet_keep for every request or for none")
        rid = self._next_id
        self._next_id += 1
        self.queue.append(Request(rid, text_ids.detach().to(device="cpu", dtype=torch.int64), limit, prenet_keep, seed))
        return rid

    def idle(self):
        return not self.queue and all(r is None for r in self.table)

    # -- one chunk ----------------------------------------------------------------------------------
    def chunk_mask(self, occupied):
        """(chunk_steps + 1, 2, slots, 256) uint8: [i, :, slot] is the mask of the occupant's own step steps + i (ones
        past its mask).  The kernel reads rows 1..chunk_steps: a step draws the mask of the step after it."""
        n = self.chunk_steps
        keep = torch.ones(n + 1, 2, self.slots, 256, dtype=torch.uint8)
        for slot, r in occupied:
            rows = r.keep[r.steps:r.steps + n + 1]
            keep[:rows.shape[0], :, slot] = rows
        return keep

    def step(self):
        """Admits queued requests into the idle slots, runs one chunk of chunk_steps decoder steps, and returns the
        results of the requests that finished in it (slot order).  Nothing to run: returns []."""
        admitted = []
        for slot in range(self.slots):
            if self.table[slot] is None and self.queue:
                r = self.queue.popleft()
                r.slot = slot
                self.table[slot] = r
                admitted.append((slot, r))
        if admitted:
            self.backend.admit(admitted)
        occupied = [(slot, r) for slot, r in enumerate(self.table) if r is not None]
        if not occupied:
            return []
        n = self.chunk_steps
        keep = self.chunk_mask(occupied) if self.injected else None
        if self.seeded:     # every slot's request seed and the steps it ran before this chunk (idle slots: 0, 0)
            seeds, step0 = [0] * self.slots, [0] * self.slots
            for slot, r in occupied:
                seeds[slot], step0[slot] = r.seed, r.steps
            self.backend.launch(n, self.chunks, keep, [slot for slot, _ in occupied], row_seeds=(seeds, step0))
        else:
            self.backend.launch(n, self.chunks, keep, [slot for slot, _ in occupied])
        self.chunks += 1
        # before the host knows where a row fired: all the frames the chunk can hold of the request; what lies past
        # its length is cut when the result is made
        self.backend.collect([(slot, r, r.steps, min(n, r.limit - r.steps)) for slot, r in occupied])
        fired, ran = self.backend.read()
        self.row_steps += sum(min(64, self.slots - 64 * i) * ran[i] for i in {slot // 64 for slot, _ in occupied})
        finished = []
        for slot, r in occupied:
            k = ran[slot // 64]                      # a slice stops early once every row of it has fired
            f = fired[slot]
            if f > 0 and r.steps + f <= r.limit:
                r.length = r.steps + f
            elif r.steps + k >= r.limit:
                r.length, r.hit_max_steps = r.limit, True
            else:
                r.steps += k
                continue
            finished.append(r)
            self.table[slot] = None
        results = self.backend.finish(finished) if finished else []
        for r in finished:
            if r.hit_max_steps:
                print(WARNING)
        return results

    def run(self):
        """Generator: finished requests in the order they finish, until the queue is empty and every slot is idle."""
        while not self.idle():
            for res in self.step():
                yield res


class EngineBackend:
    """The device side of an InferenceServer on one Tacotron2 (eval mode): the slots' encoder memory, one DecoderStream
    whose rows are the slots, each request's own output buffers, and the postnet of finished requests."""

    def __init__(self, model, slots, max_text_len, chunk_steps, seed=None, window=None):
        """window: None or the (back, front) attention window of every request; it needs no state of its own, since the
        kernel finds each slot's window from the attention weights that admit zeroes and the stream saves."""
        from ._engine import next_seed
        self.model = model
        eng = self.eng = model._t2_engine()
        dev = eng.device
        self.dtype = model._t2_out_dtype()
        self.slots, self.T_cap, self.n_mel = slots, max_text_len, eng.hp.n_mel_channels
        self.seed = next_seed() if seed is None else int(seed)
        memory = torch.zeros(slots, max_text_len, model.encoder.lstm.hidden_size * 2, device=dev, dtype=torch.float32)
        lengths = torch.ones(slots, device=dev, dtype=torch.int32)       # an idle slot attends to one zero position
        keep = torch.ones(chunk_steps + 1, 2, slots, 256, device=dev, dtype=torch.uint8)
        self.stream = eng.decoder_stream(memory, chunk_steps + 1, prenet_keep=keep,
                                         gate_threshold=model.decoder.gate_threshold, memory_lengths=lengths, window=window)
        self.keep_ptr = self.stream.args.dec.prenet_keep
        # a seeded session's per-slot seeds (64-bit patterns) and request step counts, rewritten before every chunk
        self.row_seeds = torch.zeros(slots, device=dev, dtype=torch.int64)
        self.row_step0 = torch.zeros(slots, device=dev, dtype=torch.int32)

    def admit(self, pairs):
        """pairs: (slot, request), slots ascending.  The new texts run through the encoder as one ragged batch; their
        memory rows (zero past each text's length) and lengths replace the slots', and the slots' decoder state is reset."""
        from ._engine import f32_buffer
        self.eng = self.model._t2_engine()
        st, dev = self.stream, self.eng.device
        lens = [int(r.text.numel()) for _, r in pairs]
        T = max(lens)
        ids = torch.zeros(len(pairs), T, dtype=torch.int64)
        for i, (_, r) in enumerate(pairs):
            ids[i, :lens[i]] = r.text
        lengths = torch.tensor(lens, dtype=torch.int32)
        mem = self.eng.encoder(text=ids.to(dev), lengths=lengths, training=False, per_row=True)
        if self.dtype != torch.float32:           # a .half() model hands its memory to the decoder in half
            mem = mem.to(self.dtype).float()
        rows = torch.tensor([slot for slot, _ in pairs], device=dev)
        block = torch.zeros(len(pairs), self.T_cap, mem.shape[2], device=dev, dtype=torch.float32)
        block[:, :T] = mem
        st.memory.index_copy_(0, rows, block)
        st.len32.index_copy_(0, rows, lengths.to(dev))
        for i, (_, r) in enumerate(pairs):
            r.out = (f32_buffer(dev, r.limit, self.n_mel), f32_buffer(dev, r.limit), f32_buffer(dev, r.limit, lens[i]))
        st.admit([slot for slot, _ in pairs])

    def launch(self, n, chunk_index, keep, slots, row_seeds=None):
        """row_seeds: None or (seeds, step0), one entry per slot (see the module docstring)."""
        st = self.stream
        if keep is not None:
            st.keep.copy_(keep)
        st.args.dec.prenet_keep = self.keep_ptr if keep is not None else None
        step0 = None
        if row_seeds is not None:
            seeds, steps = row_seeds
            self.row_seeds.copy_(torch.tensor([seed_pattern(v, "tacotron2_b200") for v in seeds], dtype=torch.int64))
            self.row_step0.copy_(torch.tensor(steps, dtype=torch.int32))
            step0 = self.row_step0
        st.args.dec.row_seeds = self.row_seeds.data_ptr() if row_seeds is not None else None
        live = {slot // 64 for slot in slots}
        st.launch_chunk(n, chunk_seed(self.seed, chunk_index), [i for i in range(st.n_slices) if i not in live],
                        row_step0=step0)

    def collect(self, entries):
        """entries: (slot, request, its steps before the chunk, frames to take)."""
        self.stream.collect([(slot, cnt, r.out[2].shape[1], r.out[0][s:], r.out[1][s:], r.out[2][s:])
                             for slot, r, s, cnt in entries if cnt > 0])

    def read(self):
        return self.stream.read_chunk()

    def finish(self, requests):
        """Results of the requests that left their slots: outputs cut at each one's length, the postnet over its own
        frames (the requests of one chunk as one ragged batch)."""
        dev, dt = self.eng.device, self.dtype
        Lmax = max(r.length for r in requests)
        mel_in = torch.zeros(len(requests), Lmax, self.n_mel, device=dev, dtype=torch.float32)
        for i, r in enumerate(requests):
            m = r.out[0][:r.length]
            mel_in[i, :r.length] = m if dt == torch.float32 else m.to(dt).float()
        post = self.eng.postnet(mel_in, torch.tensor([r.length for r in requests], dtype=torch.int32), True, False, None,
                                per_row=True)
        results = []
        for i, r in enumerate(requests):
            L = r.length
            mel, gate, align = r.out
            results.append(dict(id=r.id, mel_outputs=mel[:L].t().unsqueeze(0).to(dt),
                                mel_outputs_postnet=post[i:i + 1, :, :L].to(dt),
                                gate_outputs=gate[:L].view(1, L, 1).to(dt), alignments=align[:L].unsqueeze(0).to(dt),
                                mel_length=L, hit_max_steps=r.hit_max_steps))
            if r.seed is not None:
                results[-1]["seed"] = r.seed
            r.out = None
        return results
