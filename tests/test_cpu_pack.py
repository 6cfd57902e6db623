"""
Packed decode tiles (engine option ``decode_pack``) restated in numpy: the byte layout launch_pack_scan / launch_pack_tiles
write (launch.h, MegaPack) and the bf16 bits the persistent decode kernel rebuilds from it.

A tile holds 16 rows x 256 k of a layer matrix (or the lm_head) in 6688 bytes: sign | mantissa7 of every value, a 5-bit
exponent code per value split into a nibble plane and a high-bit plane, and a 32-byte header with one exponent base per row and
the tile's escape entry. A value's biased exponent is base_r + code; a tile with a value outside its row's 32-binade window is an
escape tile whose exponent bytes live in a side buffer. The round trip is bit-exact on random bf16, on edge values (signed
zeros, subnormals, the largest finite values, rows spanning more than 31 binades) and at a K that is not a multiple of 256.
The GPU test (test_gpu_pack.py) holds the device packer's bytes to ``pack`` below.
"""
import numpy as np
import pytest

TILE, NIB, HB, HDR, ESC = 6688, 4096, 6144, 6656, 4096
TILE_SEQ, TILE_ROPE, TILE_GLU = 0, 1, 2


def geometry(N, K, mode):
    groups = (N // 2 + 7) // 8 if mode == TILE_GLU else (N + 15) // 16
    return groups, (K + 255) // 256


def tile_row(mode, hd, gi, ar):
    """Source row of A-operand row ar (0..15) of tile group gi (fp8.cuh tile_row), vectorised."""
    gi, ar = np.asarray(gi), np.asarray(ar)
    if mode == TILE_SEQ:
        return gi * 16 + ar
    if mode == TILE_ROPE:
        gph = hd // 16
        return (gi // gph) * hd + ((gi % gph) << 3) + (ar & 7) + (ar >> 3) * (hd // 2)
    return np.where(ar < 8, 2 * (gi * 8 + ar), 2 * (gi * 8 + ar - 8) + 1)


def _value_index(N, K, mode, hd):
    """(row, col, valid) of every value of every tile in [tile][lane][kstep pair p][word k][byte i] order, and the tile row
    (0..15) each value belongs to."""
    groups, tpg = geometry(N, K, mode)
    t = np.arange(groups * tpg)[:, None, None, None, None]
    lane = np.arange(32)[None, :, None, None, None]
    p = np.arange(8)[None, None, :, None, None]
    k = np.arange(4)[None, None, None, :, None]
    i = np.arange(4)[None, None, None, None, :]
    ks, gi = t % tpg, t // tpg
    m = 2 * (k & 1) + (i >> 1)                     # fragment: rows-half m & 1, k-half m >> 1
    ar = (m & 1) * 8 + (lane >> 2)
    row = tile_row(mode, hd, gi, ar)
    col = ks * 256 + (2 * p + (k >> 1)) * 16 + (m >> 1) * 8 + 2 * (lane & 3) + (i & 1)
    shape = (groups * tpg, 32, 8, 4, 4)
    row, col, ar = (np.broadcast_to(x, shape) for x in (row, col, ar))
    return row, col, (row < N) & (col < K), ar


def scan(bits, mode, hd):
    """Row bases [tiles, 16] and escape flags [tiles] (pass 1)."""
    N, K = bits.shape
    groups, tpg = geometry(N, K, mode)
    rows = tile_row(mode, hd, np.arange(groups)[:, None], np.arange(16)[None, :])        # [groups, 16]
    ok_r = rows < N
    w = np.zeros((groups, 16, tpg * 256), np.uint16)
    w[ok_r] = bits[rows[ok_r]][:, :] if K == tpg * 256 else np.pad(bits[rows[ok_r]], ((0, 0), (0, tpg * 256 - K)))
    ok = np.zeros((groups, 16, tpg * 256), bool)
    ok[ok_r] = True
    ok[:, :, K:] = False
    e = ((w >> 7) & 0xFF).astype(np.int32).reshape(groups, 16, tpg, 256)
    ok = ok.reshape(groups, 16, tpg, 256)
    emax = np.where(ok, e, 0).max(-1)
    emin = np.where(ok, e, 255).min(-1)
    base = np.maximum(emax - 31, 0)                                                       # [groups, 16, tpg]
    esc = (emin < base).any(1)                                                            # [groups, tpg]
    base = np.where(esc[:, None, :], 0, base)
    return base.transpose(0, 2, 1).reshape(groups * tpg, 16), esc.reshape(-1)


def escape_tiles(bits, mode, hd):
    return int(scan(bits, mode, hd)[1].sum())


def pack(bits, mode, hd, esc0=0):
    """uint16 [N, K] bf16 bits -> (tiles uint8 [ntiles, 6688], escape planes uint8 [nesc, 4096]); esc0 = first escape entry."""
    N, K = bits.shape
    base, esc = scan(bits, mode, hd)
    T = base.shape[0]
    row, col, ok, ar = _value_index(N, K, mode, hd)
    v = np.where(ok, bits[np.minimum(row, N - 1), np.minimum(col, K - 1)], 0).astype(np.uint32)
    e = (v >> 7) & 0xFF
    byte = (((v >> 8) & 0x80) | (v & 0x7F)).astype(np.uint8)                              # [T, 32, 8, 4, 4]
    b = np.take_along_axis(base, ar.reshape(T, -1), 1).reshape(ar.shape)
    code = np.where(ok & ~esc[:, None, None, None, None], e - b, 0).astype(np.uint32)
    assert code.max(initial=0) < 32
    tiles = np.zeros((T, TILE), np.uint8)
    tiles[:, :NIB] = byte.reshape(T, 32, 8, 16).transpose(0, 2, 1, 3).reshape(T, NIB)     # [p][lane][16 B]
    sh = 8 * np.arange(4)[None, None, None, None, :] + 4 * (np.arange(4) & 1)[None, None, None, :, None]
    nib = ((code & 15) << sh)                                                             # [T, lane, p, k, i]
    nibw = np.stack([(nib[:, :, :, 2 * h:2 * h + 2, :]).reshape(T, 32, 8, 8).sum(-1) for h in range(2)], -1)  # [T, lane, p, 2]
    nibw = nibw.astype(np.uint32).reshape(T, 32, 4, 2, 2).transpose(0, 2, 1, 3, 4)         # [T, load, lane, p & 1, word]
    tiles[:, NIB:HB] = nibw.astype("<u4").view(np.uint8).reshape(T, HB - NIB)
    hsh = (8 * np.arange(4)[None, None, None, None, :] + 4 * (np.arange(8) & 1)[None, None, :, None, None]
           + np.arange(4)[None, None, None, :, None])
    hb = ((code >> 4) << hsh).reshape(T, 32, 4, 2 * 4 * 4).sum(-1).astype(np.uint32)      # [T, lane, word j]
    tiles[:, HB:HDR] = hb.astype("<u4").view(np.uint8).reshape(T, HDR - HB)
    tiles[:, HDR:HDR + 16] = base.astype(np.uint8)
    idx = np.where(esc, esc0 + np.cumsum(esc) - 1, -1).astype("<i4")
    tiles[:, HDR + 16:HDR + 20] = idx.view(np.uint8).reshape(T, 4)
    planes = e.astype(np.uint8).reshape(T, 32, 8, 16).transpose(0, 2, 1, 3).reshape(T, ESC)[esc]
    return tiles, planes


def _prmt_sign(w, sel):
    """prmt.b32 d, w, 0, sel (sign-replicating nibbles), vectorised over uint32 w."""
    src = [(w >> (8 * j)) & 0xFF for j in range(4)] + [np.zeros_like(w)] * 4
    out = np.zeros_like(w)
    for j in range(4):
        n = (sel >> (4 * j)) & 0xF
        byte = src[n & 7]
        if n & 8:
            byte = np.where(byte & 0x80, 0xFF, 0).astype(w.dtype)
        out |= byte << (8 * j)
    return out


def unpack(tiles, planes, N, K, mode, hd):
    """The bf16 bits [N, K] the kernel rebuilds: per pair (prmt(cb) << 7) + ((prmt_sign(w) & 0x807F807F) | base)."""
    T = tiles.shape[0]
    w = tiles[:, :NIB].reshape(T, 8, 32, 4, 4).transpose(0, 2, 1, 3, 4).copy().view("<u4")[..., 0].astype(np.uint32)  # [T, lane, p, k]
    nibw = tiles[:, NIB:HB].copy().view("<u4").reshape(T, 4, 32, 2, 2).transpose(0, 2, 1, 3, 4).reshape(T, 32, 8, 2)
    hbw = tiles[:, HB:HDR].copy().view("<u4").reshape(T, 32, 4).astype(np.uint32)
    base = tiles[:, HDR:HDR + 16].astype(np.uint32)
    idx = tiles[:, HDR + 16:HDR + 20].copy().view("<i4")[:, 0]
    lane = np.arange(32)
    out = np.zeros((N, K), np.uint16)
    row, col, ok, _ = _value_index(N, K, mode, hd)
    vals = np.zeros((T, 32, 8, 4, 4), np.uint16)
    for p in range(8):
        for k in range(4):
            t = 4 * (p & 1) + k
            h = hbw[:, :, p >> 1]
            hs = (h >> (t - 4)) if t >= 4 else ((h << (4 - t)) & 0xFFFFFFFF)
            cb = ((nibw[:, :, p, k >> 1].astype(np.uint32) >> (4 * (k & 1))) & 0x0F0F0F0F) | (hs & 0x10101010)
            esc = idx >= 0
            if esc.any():
                cb[esc] = planes[idx[esc]].reshape(-1, 8, 32, 4, 4)[:, p, :, k, :].copy().view("<u4")[..., 0]
            for u in range(2):
                r = base[:, (lane >> 2) + 8 * u]
                bb = np.where(esc[:, None], 0, r * 0x00800080).astype(np.uint32)
                s = _prmt_sign(w[:, :, p, k], 0x9180 if u == 0 else 0xB3A2)
                ee = _prmt_sign(cb, 0x4140 if u == 0 else 0x4342)
                a = ((ee << 7) + ((s & 0x807F807F) | bb)) & 0xFFFFFFFF
                vals[:, :, p, k, 2 * u] = a & 0xFFFF
                vals[:, :, p, k, 2 * u + 1] = a >> 16
    out[row[ok], col[ok]] = vals[ok]
    return out


def _bf16_bits(x):
    return (np.asarray(x, np.float32).view(np.uint32) >> 16).astype(np.uint16)   # truncation: any bf16 pattern is fine here


@pytest.mark.parametrize("N,K,mode,hd", [(32, 512, TILE_SEQ, 128), (256, 256, TILE_ROPE, 128), (128, 512, TILE_ROPE, 64),
                                         (64, 5504 // 8, TILE_GLU, 128), (48, 5504, TILE_SEQ, 128)])
def test_round_trip_is_bit_exact_on_random_bf16(N, K, mode, hd):
    rng = np.random.default_rng(N * K + mode)
    bits = _bf16_bits(rng.normal(0, 0.02, (N, K)))
    tiles, planes = pack(bits, mode, hd)
    assert tiles.shape == (np.prod(geometry(N, K, mode)), TILE)
    assert np.array_equal(unpack(tiles, planes, N, K, mode, hd), bits)


def test_round_trip_is_bit_exact_on_edge_values():
    rng = np.random.default_rng(7)
    N, K = 64, 1000   # K padding: 24 columns of the last tile lie outside the matrix
    bits = _bf16_bits(rng.normal(0, 0.02, (N, K)))
    bits[0, :8] = [0x0000, 0x8000, 0x0001, 0x807F, 0x7F7F, 0xFF7F, 0x0080, 0x8080]   # +-0, subnormals, +-max, +-min normal
    bits[16, 300] = 0x0000                                                            # a zero in a row with base > 0
    bits[32, 600] = _bf16_bits(1e-12)                                                 # > 31 binades below the row's max
    bits[48] = _bf16_bits(np.float32(2.0) ** rng.integers(-60, 60, K).astype(np.float32))
    bits[49] = _bf16_bits(rng.normal(0, 1e-38, K))                                    # a row of subnormals: base 0, no escape
    tiles, planes = pack(bits, TILE_SEQ, 128)
    base, esc = scan(bits, TILE_SEQ, 128)
    tpg = 4
    assert esc[0 * tpg + 0] and esc[1 * tpg + 1] and esc[2 * tpg + 2] and esc[3 * tpg:3 * tpg + 4].all()
    assert planes.shape == (int(esc.sum()), ESC)
    assert np.array_equal(unpack(tiles, planes, N, K, TILE_SEQ, 128), bits)
    idx = tiles[:, HDR + 16:HDR + 20].copy().view("<i4")[:, 0]
    assert list(idx[esc]) == list(range(int(esc.sum()))) and (idx[~esc] == -1).all()


def test_escapes_are_rare_on_random_init_weights():
    """N(0, 0.02^2) rounded to bf16: a value 31 binades below its row's largest one has probability ~1e-10."""
    rng = np.random.default_rng(0)
    bits = _bf16_bits(rng.normal(0, 0.02, (2048, 5504)))
    assert escape_tiles(bits, TILE_SEQ, 128) == 0
