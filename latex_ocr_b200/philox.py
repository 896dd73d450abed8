"""Host mirror (numpy) of the device Philox4x32-10 generator in csrc/lo_common.cuh — used by tests to reproduce the in-kernel
dropout masks and beam-search diversity draws, and documenting the stream layout:

  dropout multiplier of (row b, step t, unit j), call counter n, 64-bit seed s:
      words = philox4x32_10(counter = (j >> 2, t, b, n), key = (s & 0xffffffff, s >> 32));  u = (words[j & 3] >> 8) * 2**-24
      multiplier = 1/(1-p) if u >= p else 0                                   (nn.Dropout semantics, seq2seq_torch.py:316)

  scheduled-sampling coin of (row b, step t) under the same {seed s, call n} (lo_decoder_args.ss_prob without ss_u):
      u = (philox4x32_10(counter = (0xFFFFFFFF, t, b, n), key = (s & 0xffffffff, s >> 32))[0] >> 8) * 2**-24
  a first counter word the dropout stream (j >> 2 < D / 4) never reaches; the model's own argmax is fed where u < p

  Gumbel uniform of (row b, step t, token v) under the same {seed s, call n} (lo_decoder_args.ss_temp without ss_gu):
      words = philox4x32_10(counter = (0x80000000 | (v >> 2), t, b, n), key = (s & 0xffffffff, s >> 32));
      u = ((words[v & 3] >> 8) + 0.5) * 2**-24                     in (0, 1), never 0 or 1
  the first counter word is >= 2**31, which neither the dropout stream (j >> 2 < 2**31) nor the coin (0xFFFFFFFF) uses; a step that
  samples feeds argmax_v (logits[v] / tau - log(-log u_v)), one draw from softmax(logits / tau)
"""
import numpy as np

_M0, _M1, _W0, _W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85


def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """Vectorised over numpy uint32 arrays (broadcast)."""
    c0, c1, c2, c3 = (np.asarray(x, dtype=np.uint64) for x in (c0, c1, c2, c3))
    k0, k1 = np.uint64(k0), np.uint64(k1)
    mask = np.uint64(0xFFFFFFFF)
    for _ in range(10):
        p0 = np.uint64(_M0) * c0
        p1 = np.uint64(_M1) * c2
        hi0, lo0 = p0 >> np.uint64(32), p0 & mask
        hi1, lo1 = p1 >> np.uint64(32), p1 & mask
        c0, c1, c2, c3 = (hi1 ^ c1 ^ k0) & mask, lo1, (hi0 ^ c3 ^ k1) & mask, lo0
        k0 = (k0 + np.uint64(_W0)) & mask
        k1 = (k1 + np.uint64(_W1)) & mask
    return c0, c1, c2, c3


def u01(words):
    return ((np.asarray(words, dtype=np.uint64) >> np.uint64(8)).astype(np.float32) * np.float32(1.0 / 16777216.0)).astype(np.float32)


def dropout_multipliers(seed, call, B, T, D, p):
    """[B, T, D] float32 multipliers exactly as lstm_pw_fwd_kernel draws them."""
    b = np.arange(B, dtype=np.uint64)[:, None, None]
    t = np.arange(T, dtype=np.uint64)[None, :, None]
    j4 = np.arange(D // 4 + (1 if D % 4 else 0), dtype=np.uint64)[None, None, :]
    w = philox4x32_10(j4 + 0 * b + 0 * t, t + 0 * b + 0 * j4, b + 0 * t + 0 * j4, np.uint64(call), seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
    u = np.stack([u01(x) for x in w], axis=-1).reshape(B, T, -1)[:, :, :D]
    return np.where(u >= np.float32(p), np.float32(1.0 / (1.0 - p)), np.float32(0.0)).astype(np.float32)


def sampling_uniforms(seed, call, B, T):
    """[B, T] float32 coins exactly as lstm_pw_fwd_kernel draws them in scheduled-sampling mode (row b, step t)."""
    b = np.arange(B, dtype=np.uint64)[:, None]
    t = np.arange(T, dtype=np.uint64)[None, :]
    w = philox4x32_10(np.uint64(0xFFFFFFFF) + 0 * b + 0 * t, t + 0 * b, b + 0 * t, np.uint64(call), seed & 0xFFFFFFFF,
                      (seed >> 32) & 0xFFFFFFFF)
    return u01(w[0]).reshape(B, T)


def gumbel_uniforms(seed, call, B, T, V):
    """[B, T, V] float64 uniforms exactly as lstm_pw_fwd_gumbel_kernel draws them (row b, step t, token v); float64 holds every
    value exactly (25 significant bits)."""
    b = np.arange(B, dtype=np.uint64)[:, None, None]
    t = np.arange(T, dtype=np.uint64)[None, :, None]
    v4 = np.arange((V + 3) // 4, dtype=np.uint64)[None, None, :]
    w = philox4x32_10(np.uint64(0x80000000) | (v4 + 0 * b + 0 * t), t + 0 * b + 0 * v4, b + 0 * t + 0 * v4, np.uint64(call),
                      seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
    x = np.stack(w, axis=-1).reshape(B, T, -1)[:, :, :V]
    return ((x >> np.uint64(8)).astype(np.float64) + 0.5) * 2.0 ** -24
