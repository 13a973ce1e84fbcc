"""bzip2 test corpus: a small bzip2 encoder written for the tests (so that
streams Python's bz2 module never writes can be built: randomised blocks,
chosen Huffman groups and code lengths, extra selectors, chosen origPtr),
the acceptance oracle, and the valid and damaged corpora shared by the host
and GPU tests of dng_scan_feed_bzip2."""

import bz2
import random
import struct

BLOCK_MAGIC = 0x314159265359
EOS_MAGIC = 0x177245385090


def rnums():
    """The randomisation table, from the libbz2 Python's bz2 links."""
    import ctypes
    lib = ctypes.CDLL('libbz2.so.1.0')
    return list((ctypes.c_int32 * 512).in_dll(lib, 'BZ2_rNums'))


def oracle(data):
    """What the decoder must give: bz2.decompress stream by stream, except
    that anything after the last stream must be zero bytes (None: damage)."""
    if data[:3] != b'BZh' or len(data) < 4 or not 0x31 <= data[3] <= 0x39:
        return None
    out = []
    while data:
        if not data.strip(b'\0') and out:
            break
        d = bz2.BZ2Decompressor()
        try:
            out.append(d.decompress(data))
        except (OSError, EOFError, ValueError):
            return None
        if not d.eof:
            return None
        data = d.unused_data
    return b''.join(out)


class Bits(object):
    def __init__(self):
        self.v, self.n = 0, 0

    def put(self, value, n):
        self.v = (self.v << n) | (value & ((1 << n) - 1))
        self.n += n

    def bytes(self):
        pad = -self.n % 8
        return (self.v << pad).to_bytes((self.n + pad) // 8, 'big')


def crc32_msb(data, crc=0xffffffff):
    for b in data:
        crc ^= b << 24
        for _ in range(8):
            crc = ((crc << 1) ^ 0x04c11db7 if crc & 0x80000000
                   else crc << 1) & 0xffffffff
    return crc


def block_crc(data):
    return crc32_msb(data) ^ 0xffffffff


def rle1(data):
    """bzip2's first stage: runs of 4-255 equal bytes as 4 and a count."""
    out, i = bytearray(), 0
    while i < len(data):
        j = i
        while j < len(data) and data[j] == data[i] and j - i < 255:
            j += 1
        n = j - i
        if n >= 4:
            out += bytes([data[i]]) * 4 + bytes([n - 4])
        else:
            out += data[i:j]
        i = j
    return bytes(out)


def unrle1(block):
    """The final run-length stage, as libbz2 undoes it (None: a run of four
    ends the block without its count)."""
    out, i, prev, cnt = bytearray(), 0, None, 0
    for c in block:
        if cnt == 4:
            out += bytes([prev]) * c
            cnt = 0
            continue
        out.append(c)
        cnt = cnt + 1 if cnt and c == prev else 1
        prev = c
    return None if cnt == 4 else bytes(out)


def bwt(block):
    """(last column, origPtr) of the sorted rotations, by prefix doubling."""
    import numpy as np
    n = len(block)
    s = np.frombuffer(block, dtype=np.uint8).astype(np.int64)
    rank = s.copy()
    idx = np.arange(n)
    k = 1
    while True:
        key = rank * (n + 256) + rank[(idx + k) % n]
        order = np.argsort(key, kind='stable')
        sk = key[order]
        newrank = np.empty(n, dtype=np.int64)
        newrank[order] = np.concatenate(([0], np.cumsum(sk[1:] != sk[:-1])))
        rank = newrank
        if k >= n or rank.max() == n - 1:
            break
        k *= 2
    order = np.argsort(rank, kind='stable')
    last = bytes(np.frombuffer(block, dtype=np.uint8)[(order - 1) % n])
    return last, int(np.nonzero(order == 0)[0][0])


def inverse(last, orig, rand=False):
    """libbz2's walk of a BWT block from origPtr, randomisation undone."""
    n = len(last)
    cnt = [0] * 257
    for c in last:
        cnt[c + 1] += 1
    for i in range(256):
        cnt[i + 1] += cnt[i]
    t = [0] * n
    for i, c in enumerate(last):
        t[cnt[c]] = i
        cnt[c] += 1
    out, p = bytearray(), t[orig]
    for _ in range(n):
        out.append(last[p])
        p = t[p]
    if rand:
        r, at, k = rnums(), 0, 0
        while True:
            at += r[k % 512]
            k += 1
            if at - 2 >= n:
                break
            out[at - 2] ^= 1
    return bytes(out)


def mtf_symbols(last, used):
    """RUNA/RUNB and move-to-front symbols of a BWT block, EOB last."""
    seq = {b: i for i, b in enumerate(used)}
    order = list(range(len(used)))
    syms, run = [], 0

    def flush():
        n = run
        while n > 0:
            n -= 1
            syms.append(n & 1)
            n >>= 1
    for c in last:
        v = seq[c]
        j = order.index(v)
        if j == 0:
            run += 1
            continue
        flush()
        run = 0
        order.pop(j)
        order.insert(0, v)
        syms.append(j + 1)
    flush()
    syms.append(len(used) + 1)
    return syms


def lengths_for(freq, limit=17):
    """Huffman code lengths for freq (every symbol gets one), at most
    `limit` bits, by scaling the counts until they fit."""
    import heapq
    freq = [max(f, 1) for f in freq]
    while True:
        heap = [(f, i, [i]) for i, f in enumerate(freq)]
        heapq.heapify(heap)
        lens = [0] * len(freq)
        nxt = len(freq)
        while len(heap) > 1:
            f1, _, a = heapq.heappop(heap)
            f2, _, b = heapq.heappop(heap)
            for s in a + b:
                lens[s] += 1
            heapq.heappush(heap, (f1 + f2, nxt, a + b))
            nxt += 1
        if max(lens) <= limit:
            return lens
        freq = [max(f // 2, 1) for f in freq]


def canonical(lens):
    """bzip2's code assignment (BZ2_hbAssignCodes)."""
    codes, vec = [0] * len(lens), 0
    for n in range(min(lens), max(lens) + 1):
        for i, ln in enumerate(lens):
            if ln == n:
                codes[i] = vec
                vec += 1
        vec <<= 1
    return codes


def block_bits(bits, last, orig, crc, rand=False, ngroups=2, lens=None,
               extra_selectors=0, syms=None):
    """One block into `bits`: the BWT block `last` with `orig`; `lens`
    (ngroups lists) replaces the Huffman lengths; `syms` replaces the
    symbols (the MTF of `last` by default)."""
    used = sorted(set(last))
    if syms is None:
        syms = mtf_symbols(last, used)
    alpha = len(used) + 2
    nsel = (len(syms) + 49) // 50
    groups = [g % ngroups for g in range(nsel)]
    if lens is None:
        lens = []
        for t in range(ngroups):
            f = [0] * alpha
            for g, gi in enumerate(groups):
                if gi == t:
                    for s in syms[g * 50:g * 50 + 50]:
                        f[s] += 1
            lens.append(lengths_for(f))
    bits.put(BLOCK_MAGIC, 48)
    bits.put(crc, 32)
    bits.put(1 if rand else 0, 1)
    bits.put(orig, 24)
    used16 = 0
    for i in range(16):
        if any(b // 16 == i for b in used):
            used16 |= 1 << (15 - i)
    bits.put(used16, 16)
    for i in range(16):
        if used16 >> (15 - i) & 1:
            w = 0
            for b in used:
                if b // 16 == i:
                    w |= 1 << (15 - b % 16)
            bits.put(w, 16)
    bits.put(ngroups, 3)
    allsel = groups + [0] * extra_selectors
    bits.put(len(allsel), 15)
    order = list(range(ngroups))
    for g in allsel:
        j = order.index(g)
        bits.put((1 << (j + 1)) - 2, j + 1)   # j ones, then a zero
        order.pop(j)
        order.insert(0, g)
    for t in range(ngroups):
        curr = lens[t][0]
        bits.put(curr, 5)
        for ln in lens[t]:
            while curr < ln:
                bits.put(2, 2)
                curr += 1
            while curr > ln:
                bits.put(3, 2)
                curr -= 1
            bits.put(0, 1)
    codes = [canonical(ls) for ls in lens]
    for k, s in enumerate(syms):
        t = groups[k // 50]
        bits.put(codes[t][s], lens[t][s])


def stream(blocks, level=9):
    """A stream of the given blocks: each a dict of block_bits() arguments
    plus 'out' (its decoded bytes, for the CRCs)."""
    bits = Bits()
    for c in b'BZh':
        bits.put(c, 8)
    bits.put(0x30 + level, 8)
    scrc = 0
    for b in blocks:
        crc = block_crc(b.pop('out'))
        scrc = ((scrc << 1 | scrc >> 31) & 0xffffffff) ^ crc
        block_bits(bits, crc=crc, **b)
    bits.put(EOS_MAGIC, 48)
    bits.put(scrc, 32)
    return bits.bytes()


def data_block(data, **kw):
    """block_bits() arguments for `data` (at most one block after RLE1)."""
    r = rle1(data)
    rand = kw.get('rand', False)
    if rand:
        # the decoder flips after the walk: flip before the transform
        rn, flip, at, k = rnums(), bytearray(r), 0, 0
        while True:
            at += rn[k % 512]
            k += 1
            if at - 2 >= len(r):
                break
            flip[at - 2] ^= 1
        r = bytes(flip)
    last, orig = bwt(r)
    kw.update(last=last, orig=orig, out=data)
    return kw


def log_lines(n, seed=1):
    rnd = random.Random(seed)
    return b''.join(b'{"req":{"method":"%s","url":"/x/%d"},"res":'
                    b'{"statusCode":%d},"latency":%d}\n' % (
                        rnd.choice([b'GET', b'PUT', b'POST']),
                        rnd.randrange(100), rnd.choice([200, 404, 500]),
                        rnd.randrange(5000)) for _ in range(n))


def hand_built():
    """Streams Python's bz2 module does not write, each a (name, bytes)."""
    out = []
    text = log_lines(300, seed=7)
    out.append(('randomised', stream([data_block(text, rand=True)])))
    out.append(('groups2', stream([data_block(text, ngroups=2)])))
    out.append(('groups6', stream([data_block(text, ngroups=6)])))
    # a complete code of 1, 2, ..., 19, 20 and 20 bits over 19 byte values
    b = data_block(bytes(range(19)) * 6)
    ladder = list(range(1, 20)) + [20, 20]
    assert len(set(b['last'])) + 2 == len(ladder)
    assert sum(2 ** -n for n in ladder) == 1
    b.update(ngroups=2, lens=[ladder, ladder[::-1]])
    out.append(('len20', stream([b])))
    # 20,000 selectors: those past 18,002 are read and ignored
    out.append(('selectors20000', stream([data_block(
        text, extra_selectors=20000 - (len(mtf_symbols(
            bwt(rle1(text))[0], sorted(set(text)))) + 49) // 50)])))
    up = bytes(range(1, 200))
    out.append(('orig0', stream([data_block(up)])))
    out.append(('origlast', stream([data_block(up[::-1])])))
    assert data_block(up)['orig'] == 0
    assert data_block(up[::-1])['orig'] == len(up) - 1
    # exactly level x 100,000 bytes after RLE1, at level 1
    rnd = random.Random(3)
    full = bytes(rnd.randrange(256) for _ in range(100000))
    assert len(rle1(full)) == 100000
    out.append(('full-level1', stream([data_block(full)], level=1)))
    out.append(('false-start', false_start()))
    return out


def false_start():
    """A block whose Huffman-coded symbols hold the block magic: every
    symbol a 9-bit code (an incomplete code libbz2 decodes), its value the
    symbol, the symbols chosen to spell the magic at some alignment."""
    magic = format(BLOCK_MAGIC, '048b')
    for k in range(9):
        bits = '0' * k + magic
        bits += '0' * (-len(bits) % 9)
        vals = [int(bits[i:i + 9], 2) for i in range(0, len(bits), 9)]
        if all(2 <= v <= 256 for v in vals):
            break
    else:
        raise AssertionError('no alignment')
    used = list(range(256))
    syms = [2] * 10 + vals + [2] * 10
    # the BWT block these move-to-front symbols give
    order, last = list(range(256)), bytearray()
    for s in syms:
        j = s - 1
        v = order.pop(j)
        order.insert(0, v)
        last.append(v)
    last += bytes(x for x in range(256) if x not in last)
    syms = mtf_symbols(bytes(last), used)
    assert all(s <= 257 for s in syms)
    out = unrle1(inverse(bytes(last), 0))
    assert out is not None
    lens = [[9] * 258, [9] * 258]
    return stream([dict(last=bytes(last), orig=0, out=out, lens=lens,
                        syms=syms)])


def valid_corpus():
    """(name, bytes) of files the decoder must decode as the oracle does."""
    rnd = random.Random(5)
    text = log_lines(20000)
    c = []
    for lv in range(1, 10):
        c.append(('level%d' % lv, bz2.compress(text[:150000 * lv // 3], lv)))
    c += [('empty', bz2.compress(b'')), ('one', bz2.compress(b'x')),
          ('bytes256', bz2.compress(bytes(range(256))))]
    for n in (3, 4, 5, 259, 260, 10 ** 6):
        c.append(('run%d' % n, bz2.compress(b'q' * n)))
    c.append(('full-run', bz2.compress(b'\0' * 45900000, 9)))
    c.append(('multi-levels', bz2.compress(text[:5000], 1) +
              bz2.compress(b'') + bz2.compress(text[5000:90000], 9) +
              bz2.compress(b'tail without newline', 4)))
    c.append(('zeros-after', bz2.compress(text[:3000]) + b'\0' * 77))
    c.append(('random', bz2.compress(bytes(rnd.randrange(256)
                                           for _ in range(200000)), 2)))
    c.append(('lines', bz2.compress(text)))
    return c


def damaged_corpus(seed=1):
    """(name, bytes) of damaged files: truncations, flipped bits in every
    header field and in the data, CRCs, levels, trailing data."""
    rnd = random.Random(seed)
    base = bz2.compress(log_lines(3000, seed=seed), 1)
    two = bz2.compress(log_lines(200, seed=seed + 1), 2) + \
        bz2.compress(log_lines(100, seed=seed + 2), 3)
    c = []
    for n in (4, 5, 9, 10, 13, 14, 20, 40, 100, len(base) // 2,
              len(base) - 10, len(base) - 5, len(base) - 1):
        c.append(('trunc%d' % n, base[:n]))
    # bits of the stream and block headers, the tables, the data
    for bit in list(range(24, 32)) + list(range(32, 200)) + \
            [rnd.randrange(200, len(base) * 8) for _ in range(150)]:
        d = bytearray(base)
        d[bit // 8] ^= 0x80 >> (bit % 8)
        c.append(('flip%d' % bit, bytes(d)))
    # the block CRC (bits 80-111) and the stream CRC (the last 4-5 bytes)
    d = bytearray(base)
    d[10] ^= 1
    c.append(('bad-block-crc', bytes(d)))
    d = bytearray(two)
    d[-2] ^= 0x10
    c.append(('bad-stream-crc', bytes(d)))
    for lv in b'0:a':
        c.append(('level-%c' % lv, base[:3] + bytes([lv]) + base[4:]))
    end = base.rfind(b'\x17\x72\x45\x38\x50\x90')
    c.append(('no-eos', base[:end] if end > 0 else base[:-10]))
    c.append(('trailing-junk', base + b'junk'))
    c.append(('trailing-zeros-junk', base + b'\0\0\1'))
    c.append(('trailing-bzh', base + b'BZh9'))
    c.append(('second-damaged', base + two[:len(two) // 2]))
    c.append(('bad-second-header', base + b'BZh0' + two[4:]))
    for _ in range(40):
        d = bytearray(two)
        at = rnd.randrange(4, len(d))
        d[at] ^= 1 << rnd.randrange(8)
        c.append(('flip2-%d' % at, bytes(d)))
    return c


def pack_cases(cases):
    """The host driver's input: per case its bytes and extra candidates."""
    out = [struct.pack('<I', len(cases))]
    for data, extra in cases:
        out.append(struct.pack('<Q', len(data)) + data +
                   struct.pack('<I', len(extra)) +
                   b''.join(struct.pack('<Q', b) for b in extra))
    return b''.join(out)
