"""Host rebuild of the engine's in-kernel dropout masks.

Every production dropout decision in libt2b200 is ``philox_keep(seed, site, idx, p)``: Philox4x32-10 (Salmon et al.,
"Parallel random numbers: as easy as 1, 2, 3", SC'11) with counter ``(idx >> 2 lo, idx >> 2 hi, site, 0x7ac07201)`` and
key ``(seed lo, seed hi)``; lane ``idx & 3`` of the output block gives ``u = (o >> 8) * 2^-24`` and the element is kept
when ``u >= p`` (both in fp32).  The functions here compute the same bits with torch int64 arithmetic (CPU or GPU) and
lay them out as ``tacotron2_b200.dropout_masks`` takes them, so a test can feed the masks a Philox run drew back into
the same kernels and into the oracle.  Each builder documents its site numbering and element index; those are the
engine's convention (the kernels of the forward AND the backward pass of each layer must agree with it)."""
import torch

_M32 = 0xFFFFFFFF
_MUL = (0xD2511F53, 0xCD9E8D57)       # Philox4x32 round multipliers
_WEYL = (0x9E3779B9, 0xBB67AE85)      # key schedule increments (golden ratio, sqrt(3) - 1)
COUNTER_TAG = 0x7ac07201              # the engine's fixed fourth counter word


def _mulhilo(a, m):
    """(hi, lo) 32-bit halves of a * m for int64 tensors a < 2^32 and a constant m < 2^32, without int64 overflow."""
    m_hi, m_lo = m >> 16, m & 0xFFFF
    t_lo = a * m_lo                                   # < 2^48
    t_hi = a * m_hi                                   # < 2^48, weight 2^16
    s = t_lo + ((t_hi & 0xFFFF) << 16)                # bits 0..48 of the product
    return ((t_hi >> 16) + (s >> 32)) & _M32, s & _M32


def philox4x32_10(ctr, key):
    """ctr: 4 int64 tensors (or ints) holding 32-bit words, key: 2 such.  Returns the 4 output words (int64 tensors)."""
    x = [torch.as_tensor(c, dtype=torch.int64) for c in ctr]
    k0, k1 = int(key[0]) & _M32, int(key[1]) & _M32
    for _ in range(10):
        hi0, lo0 = _mulhilo(x[0], _MUL[0])
        hi1, lo1 = _mulhilo(x[2], _MUL[1])
        x = [hi1 ^ x[1] ^ k0, lo1, hi0 ^ x[3] ^ k1, lo0]
        k0, k1 = (k0 + _WEYL[0]) & _M32, (k1 + _WEYL[1]) & _M32
    return x


def uniform(seed, site, idx):
    """The fp32 uniform u in [0, 1) the engine draws for element `idx` (int64 tensor) of dropout site `site` (int or
    int64 tensor broadcastable against idx)."""
    idx = torch.as_tensor(idx, dtype=torch.int64)
    idx, site = torch.broadcast_tensors(idx, torch.as_tensor(site, dtype=torch.int64, device=idx.device))
    blk = idx >> 2
    o = philox4x32_10((blk & _M32, blk >> 32, site, torch.full_like(blk, COUNTER_TAG)),
                      (seed & _M32, (seed >> 32) & _M32))
    word = torch.stack(o, -1).gather(-1, (idx & 3).unsqueeze(-1)).squeeze(-1)
    return (word >> 8).to(torch.float32) * (1.0 / 16777216.0)


def keep(seed, site, idx, p):
    """Bool tensor: philox_keep(seed, site, idx, p) for every element of idx."""
    return uniform(seed, site, idx) >= torch.tensor(p, dtype=torch.float32)


def _stream(seed, sites, n, p, device):
    """Keep bits of elements 0..n-1 of every site in `sites` (list): uint8 (len(sites), n).  Whole Philox blocks are
    generated once and all four lanes used, so the cost is one Philox call per four elements."""
    nb = (n + 3) // 4
    blk = torch.arange(nb, dtype=torch.int64, device=device)
    out = torch.empty(len(sites), nb * 4, dtype=torch.uint8, device=device)
    thr = torch.tensor(p, dtype=torch.float32, device=device)
    step = max(1, (1 << 22) // nb)                    # bound the int64 temporaries to a few tens of MB
    for s0 in range(0, len(sites), step):
        site = torch.tensor(sites[s0:s0 + step], dtype=torch.int64, device=device)[:, None]
        o = philox4x32_10((blk[None, :] & _M32, (blk >> 32)[None, :], site.expand(-1, nb), COUNTER_TAG),
                          (seed & _M32, (seed >> 32) & _M32))
        u = (torch.stack(o, -1) >> 8).to(torch.float32) * (1.0 / 16777216.0)        # (sites, nb, 4): lane-major
        out[s0:s0 + step] = (u >= thr).reshape(u.shape[0], nb * 4).to(torch.uint8)
    return out[:, :n]


def encoder_masks(seed, B, T, device="cpu"):
    """Encoder conv dropout (3, B, 512, T): conv i uses site 1000+i, element (b*T + t)*512 + c, p = 0.5."""
    k = _stream(seed, [1000 + i for i in range(3)], B * T * 512, 0.5, device)
    return k.reshape(3, B, T, 512).permute(0, 1, 3, 2).contiguous()


def postnet_masks(seed, B, T, device="cpu"):
    """Postnet conv dropout [(B, 512, T)] * 4 + [(B, 80, T)]: conv i uses site 2000+i, element (b*T + t)*C + c, p = 0.5."""
    out = []
    for i in range(5):
        C = 80 if i == 4 else 512
        k = _stream(seed, [2000 + i], B * T * C, 0.5, device)
        out.append(k.reshape(B, T, C).permute(0, 2, 1).contiguous())
    return out


def teacher_prenet_masks(seed, T_mel, B, device="cpu"):
    """Teacher-forced prenet (T_mel+1, 2, B, 256): layer 0 / 1 use sites 0xA0 / 0xA1 over the (T_mel+1)*B rows the
    prenet runs on at once, element (t*B + b)*256 + n, p = 0.5."""
    k = _stream(seed, [0xA0, 0xA1], (T_mel + 1) * B * 256, 0.5, device)
    return k.reshape(2, T_mel + 1, B, 256).permute(1, 0, 2, 3).contiguous()


def lstm_masks(seed, T, B, which, p, device="cpu"):
    """Decoder LSTM hidden-state dropout (T, B, 1024): step t uses site t*4+2 (which="att", attention LSTM) or t*4+3
    (which="dec", decoder LSTM), element b*1024 + u, drop probability p."""
    k = {"att": 2, "dec": 3}[which]
    return _stream(seed, [t * 4 + k for t in range(T)], B * 1024, p, device).reshape(T, B, 1024)


def infer_prenet_masks(seed, cap, B, device="cpu"):
    """Free-running prenet (cap, 2, B, 256): step t, layer j uses site t*4+j, element b*256 + c with b the absolute
    batch row (the persistent decoder's second 64-row slice starts at b = 64), p = 0.5."""
    sites = [t * 4 + j for t in range(cap) for j in range(2)]
    return _stream(seed, sites, B * 256, 0.5, device).reshape(cap, 2, B, 256)
