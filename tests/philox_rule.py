"""Numpy restatement of the in-kernel dropout and sampling RNG (csrc/common.cuh `philox4` / `dropout_keep8`, csrc/head.cu
`pointer_mix_sample_kernel`) -- test infrastructure.

Every dropout mask the kernels draw is a pure function of (seed + *seed_ctr, stream id, element index), so the float64
oracle can apply exactly the mask a kernel applied:

  * key = (seed + ctr) mod 2^64, split into its low and high 32-bit words;
  * element (r, 8 lane + i) of a [rows, 256] activation is kept iff bit i of dropout_keep8(key, stream, r * 32 + lane, p)
    is set: ONE Philox4x32-7 call with counter (idx8 lo, idx8 hi, stream, 0) gives 16 random bits per element, compared
    with thr = uint32(float32(p) * 65536.0f);
  * a kept element is scaled by 1 / (1 - p32), p32 the fp32 value the kernel receives.

Site table: which stream id and which row index each masking site uses (ops.EncoderFn / DecoderFn, blocks.py and the
`stream_id + 8 i + site` of csrc/decoder_fwd.cu):

  | Block                                  | stream id of layer i            | mask covers     | row index                |
  |----------------------------------------|---------------------------------|-----------------|--------------------------|
  | Encoder Combination gate               | base + 8 i + 0                  | code rows       | b * n_code + i           |
  | Encoder Combination LayerNorm          | base + 8 i + 1                  | code rows       | b * n_code + i           |
  | Encoder GCN LayerNorm                  | base + 8 i + 2                  | all node rows   | segment-major buffer row |
  | Decoder self-attn, cross-attn, FFN     | base + 64 + 8 i + {0, 1, 2}     | decoder rows    | b * T + t                |
  | blocks.py module surface               | BLOCK_SID below                 | the block's rows| flat row of [B, L, D]    |

The segment-major buffer row of a padded batch is: code rows (b * n_code + j), then sub-token rows
(B * n_code + b * n_sub + j), then AST rows (B * (n_code + n_sub) + b * n_ast + j); a packed batch puts commit b's rows
of segment s at off[s][b] + j inside the segment (packed.PackedBatch.off).  The encoder and the decoder draw one seed
each per forward (ops.make_seed); blocks.py draws one per dropout site per call.
"""
import numpy as np

M0, M1, W0, W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85
MASK32 = 0xFFFFFFFF
SAMPLE_STREAM = 0x53414D50
D = 256

ENC_SITE = {"comb_gate": 0, "comb_ln": 1, "gcn_ln": 2}
DEC_SITE = {"self_attn": 0, "cross_attn": 1, "ffn": 2}
DEC_OFFSET = 64
LAYER_STRIDE = 8
BLOCK_SID = {"attention": 0, "feed_forward": 2, "gcn": 2, "comb_gate": 0, "comb_ln": 1, "combination_layer": 0}


def encoder_sid(base, layer, site):
    return base + LAYER_STRIDE * layer + ENC_SITE[site]


def decoder_sid(base, layer, site):
    return base + DEC_OFFSET + LAYER_STRIDE * layer + DEC_SITE[site]


def _u32(x):
    return np.asarray(x, dtype=np.uint64) & np.uint64(MASK32)


def philox4x32_7(c0, c1, c2, c3, k0, k1):
    """Philox4x32-7 of common.cuh, vectorised over broadcastable uint32 arrays -> (x, y, z, w) uint32 arrays."""
    c0, c1, c2, c3 = (_u32(c) for c in np.broadcast_arrays(c0, c1, c2, c3))
    k0, k1 = _u32(k0), _u32(k1)
    m0, m1 = np.uint64(M0), np.uint64(M1)
    sh, m32 = np.uint64(32), np.uint64(MASK32)
    for _ in range(7):
        p0 = m0 * c0                                    # two uint32 factors: the uint64 product is exact
        p1 = m1 * c2
        hi0, lo0 = p0 >> sh, p0 & m32                   # __umulhi / low word
        hi1, lo1 = p1 >> sh, p1 & m32
        n0 = hi1 ^ c1 ^ k0
        n2 = hi0 ^ c3 ^ k1
        c0, c1, c2, c3 = n0, lo1, n2, lo0
        k0 = (k0 + np.uint64(W0)) & m32
        k1 = (k1 + np.uint64(W1)) & m32
    return tuple(c.astype(np.uint32) for c in (c0, c1, c2, c3))


def threshold(p):
    """uint32(p_drop * 65536.0f) with p_drop the fp32 value the kernel receives"""
    return int(np.float32(p) * np.float32(65536.0))


def keep_scale(p):
    """1 / (1 - p32): the factor of a kept element"""
    return 1.0 / (1.0 - float(np.float32(p)))


def key_words(seed, ctr=0):
    key = (int(seed) + int(ctr)) % (1 << 64)
    return key & MASK32, key >> 32


def keep8(seed, ctr, stream_id, idx8, p):
    """dropout_keep8: the 8-bit keep mask of the elements 8 idx8 .. 8 idx8 + 7 (uint32 array shaped like idx8)"""
    k0, k1 = key_words(seed, ctr)
    idx8 = np.asarray(idx8, dtype=np.uint64)
    x, y, z, w = philox4x32_7(idx8 & np.uint64(MASK32), idx8 >> np.uint64(32), np.uint64(stream_id), np.uint64(0), k0, k1)
    thr = np.uint32(threshold(p))
    m = np.zeros(idx8.shape, dtype=np.uint32)
    for j, r in enumerate((x, y, z, w)):
        m |= ((r & np.uint32(0xFFFF)) >= thr).astype(np.uint32) << np.uint32(2 * j)
        m |= ((r >> np.uint32(16)) >= thr).astype(np.uint32) << np.uint32(2 * j + 1)
    return m


def keep_mask(seed, ctr, stream_id, rows, p):
    """bool [len(rows), 256] (rows: a row count or an array of row indices): True where the kernel keeps the element"""
    r = np.arange(rows, dtype=np.int64) if np.isscalar(rows) else np.asarray(rows, dtype=np.int64).reshape(-1)
    idx8 = r[:, None].astype(np.uint64) * np.uint64(32) + np.arange(32, dtype=np.uint64)[None, :]
    m = keep8(seed, ctr, stream_id, idx8, p)                            # [rows, 32]
    bits = (m[:, :, None] >> np.arange(8, dtype=np.uint32)[None, None, :]) & np.uint32(1)
    return bits.reshape(len(r), D).astype(bool)


def sample_uniform(seed, first_index, b, n, pos):
    """the u of fira_pointer_mix_sample without supplied uniforms: Philox keyed by the seed, counter
    (first_index + b, n, 'SAMP', pos), top 24 bits of the first word"""
    k0, k1 = key_words(seed)
    x, _, _, _ = philox4x32_7(np.asarray(first_index, np.int64) + np.asarray(b, np.int64), n, SAMPLE_STREAM, pos, k0, k1)
    return (x >> np.uint32(8)).astype(np.float64) * 2.0 ** -24
