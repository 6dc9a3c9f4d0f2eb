"""Sub-byte IVF-PQ codes (nbits 1-8) for the tests.

Row layout (faiss PQEncoderGeneric): a row is ceil(M * nbits / 8) bytes; code m occupies bits [m*nbits, (m+1)*nbits) of
the row's little-endian bit stream, LSB first within each byte; pad bits are zero.  At nbits = 8: one byte per code.

The oracle's encoder and LUT search take 256 codewords per sub-space.  A [M, 2^nbits, dsub] codebook is run through them
padded to 256 codewords placed 1e15 away from any data: none of them is ever the nearest, so the codes stay below 2^nbits,
and every LUT entry a code can reach is computed from the same codeword in the same order as with 2^nbits codewords.
test_oracle_pq_nbits.py pins both statements against numpy restatements."""
import numpy as np

PAD = np.float32(1e15)


def nbits_of(codebooks):
    ksub = codebooks.shape[1]
    assert ksub >= 2 and ksub <= 256 and ksub & (ksub - 1) == 0, ksub
    return ksub.bit_length() - 1


def code_size(M, nbits):
    return (M * nbits + 7) // 8


def pack(codes, nbits):
    """uint8 codes [n, M] (each < 2^nbits) -> packed rows [n, code_size(M, nbits)]."""
    c = np.ascontiguousarray(codes, np.uint8)
    n, M = c.shape
    bits = np.unpackbits(c[:, :, None], axis=2, bitorder="little")[:, :, :nbits].reshape(n, M * nbits)
    return np.packbits(bits, axis=1, bitorder="little").reshape(n, code_size(M, nbits))


def unpack(packed, M, nbits):
    """packed rows [n, code_size(M, nbits)] -> uint8 codes [n, M]."""
    p = np.ascontiguousarray(packed, np.uint8)
    if nbits == 8:
        return p.copy()
    p = np.concatenate([p, np.zeros((p.shape[0], 1), np.uint8)], axis=1).astype(np.uint16)  # a code may reach into byte b + 1
    out = np.empty((p.shape[0], M), np.uint8)
    for m in range(M):
        b, s = divmod(m * nbits, 8)
        out[:, m] = ((p[:, b] | (p[:, b + 1] << 8)) >> s) & ((1 << nbits) - 1)
    return out


def pad_codebooks(codebooks):
    cb = np.ascontiguousarray(codebooks, np.float32)
    out = np.full((cb.shape[0], 256, cb.shape[2]), PAD, np.float32)
    out[:, :cb.shape[1]] = cb
    return out


def ivfpq_encode(o, codebooks, centroids, x, assign):
    """Packed rows of the oracle's by-residual encoder."""
    codes = o.ivfpq_encode(pad_codebooks(codebooks), centroids, x, assign)
    return pack(codes, nbits_of(codebooks))


def ivfpq_search(o, metric, centroids, codebooks, list_off, packed, ids, xq, k, nprobe, nthreads=1, **filt):
    """The oracle's IVF-PQ search over packed rows."""
    codes = unpack(packed, codebooks.shape[0], nbits_of(codebooks))
    return o.ivfpq_search(metric, centroids, pad_codebooks(codebooks), list_off, codes, ids, xq, k, nprobe, nthreads=nthreads, **filt)
