"""Gzip inputs for the decoder's tests (tests/test_inflate_host.py on the CPU,
tests/test_gpu_gzip.py on the device): zlib's output at every level,
strategy and window size, hand-built streams zlib never writes (a match at
distance 32768, stored blocks of 65535 bytes, every header flag, invalid
codes), multi-member files, and a damaged corpus.  Python's gzip.decompress
is the oracle for all of them."""

import gzip
import random
import struct
import zlib


def oracle(data):
    """gzip.decompress(data), or None where it fails."""
    try:
        return gzip.decompress(data)
    except (OSError, EOFError, zlib.error):
        return None


def raw_deflate(data, level=6, wbits=15, strategy=zlib.Z_DEFAULT_STRATEGY,
                mem_level=8):
    c = zlib.compressobj(level, zlib.DEFLATED, -wbits, mem_level, strategy)
    return c.compress(data) + c.flush()


def member(body, data, flags=0, extra=b'', name=b'', comment=b'', mtime=0):
    """One gzip member around the raw deflate stream `body` of `data`."""
    h = bytearray(b'\x1f\x8b\x08') + bytes([flags]) + \
        struct.pack('<I', mtime) + b'\x00\xff'
    if flags & 4:
        h += struct.pack('<H', len(extra)) + extra
    if flags & 8:
        h += name + b'\x00'
    if flags & 16:
        h += comment + b'\x00'
    if flags & 2:
        h += struct.pack('<H', zlib.crc32(bytes(h)) & 0xffff)
    return bytes(h) + body + struct.pack('<II', zlib.crc32(data),
                                         len(data) & 0xffffffff)


def gz(data, level=6, wbits=15, strategy=zlib.Z_DEFAULT_STRATEGY, **hdr):
    return member(raw_deflate(data, level, wbits, strategy), data, **hdr)


class Bits:
    """An LSB-first bit writer, as DEFLATE packs its bits."""

    def __init__(self):
        self.acc = 0
        self.n = 0
        self.out = bytearray()

    def put(self, v, k):
        self.acc |= v << self.n
        self.n += k
        while self.n >= 8:
            self.out.append(self.acc & 255)
            self.acc >>= 8
            self.n -= 8

    def huff(self, code, k):
        """a Huffman code: its bits go most significant first"""
        self.put(int(format(code, '0%db' % k)[::-1], 2), k)

    def done(self):
        if self.n:
            self.out.append(self.acc & 255)
        return bytes(self.out)


LBASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51,
         59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
LEXT = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
DBASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385,
         513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385,
         24577]
DEXT = [0, 0, 0, 0] + [i // 2 for i in range(2, 28)]


def fixed_lit(b, sym):
    if sym < 144:
        b.huff(0x30 + sym, 8)
    elif sym < 256:
        b.huff(0x190 + sym - 144, 9)
    elif sym < 280:
        b.huff(sym - 256, 7)
    else:
        b.huff(0xc0 + sym - 280, 8)


def fixed_block(tokens, final=True, b=None):
    """One fixed-Huffman block of tokens: an int is a literal, (len, dist) a
    match, ('sym', s) / ('dsym', s) a raw (possibly invalid) code."""
    b = b or Bits()
    b.put(1 if final else 0, 1)
    b.put(1, 2)
    for t in tokens:
        if isinstance(t, int):
            fixed_lit(b, t)
        elif t[0] == 'sym':
            fixed_lit(b, t[1])
        elif t[0] == 'dsym':
            fixed_lit(b, 257)
            b.huff(t[1], 5)
        else:
            ln, d = t
            i = max(k for k in range(29) if LBASE[k] <= ln)
            if ln == 258:
                i = 28
            fixed_lit(b, 257 + i)
            b.put(ln - LBASE[i], LEXT[i])
            j = max(k for k in range(30) if DBASE[k] <= d)
            b.huff(j, 5)
            b.put(d - DBASE[j], DEXT[j])
    fixed_lit(b, 256)
    return b


def expand(tokens):
    out = bytearray()
    for t in tokens:
        if isinstance(t, int):
            out.append(t)
        else:
            ln, d = t
            for _ in range(ln):
                out.append(out[-d])
    return bytes(out)


def stored(data, final=True):
    """Stored blocks of at most 65535 bytes each."""
    out = bytearray()
    chunks = [data[i:i + 65535] for i in range(0, len(data), 65535)] or [b'']
    for k, c in enumerate(chunks):
        last = final and k == len(chunks) - 1
        out += bytes([1 if last else 0]) + struct.pack('<HH', len(c),
                                                        len(c) ^ 0xffff) + c
    return bytes(out)


def ndjson(n, seed=0):
    """Log-like records, as the scan reads them."""
    rng = random.Random(seed)
    methods = ['GET', 'PUT', 'POST', 'DELETE', 'HEAD']
    lines = []
    for i in range(n):
        lines.append(
            '{"time":"2014-05-%02dT%02d:%02d:%02d.%03dZ","req":{"method":"%s",'
            '"url":"/v1/obj/%d"},"res":{"statusCode":%d},"latency":%d,'
            '"host":"ra%03d"}' % (
                1 + i % 28, rng.randrange(24), rng.randrange(60),
                rng.randrange(60), rng.randrange(1000), rng.choice(methods),
                rng.randrange(5000), rng.choice([200, 204, 404, 500]),
                rng.randrange(3000), rng.randrange(40)))
    return ('\n'.join(lines) + '\n').encode()


def valid_corpus():
    """(name, gzip bytes): every form the decoder must accept."""
    rng = random.Random(1)
    text = ndjson(3000, 1)
    noise = bytes(rng.randrange(256) for _ in range(70000))
    mixed = text[:40000] + noise[:20000] + b'a' * 5000 + text[40000:80000]
    cases = []
    for level in range(10):
        cases.append(('level%d' % level, gz(mixed, level)))
    for sname in ('Z_DEFAULT_STRATEGY', 'Z_FILTERED', 'Z_HUFFMAN_ONLY',
                  'Z_RLE', 'Z_FIXED'):
        cases.append((sname, gz(mixed, 6, strategy=getattr(zlib, sname))))
    for w in range(9, 16):
        cases.append(('wbits%d' % w, gz(text, 9, wbits=w)))
    cases.append(('empty', gz(b'')))
    cases.append(('one-byte', gz(b'x')))
    cases.append(('nothing', b''))
    # a match 32768 back, of length 258, and overlapping matches
    head = noise[:32768]
    toks = list(head) + [(258, 32768), (258, 1), (100, 3), (3, 32768)]
    body = fixed_block(toks).done()
    cases.append(('dist32768-len258', member(body, expand(toks))))
    # stored blocks of 65535 bytes, and an empty stored block
    cases.append(('stored65535', member(stored(noise[:65535 * 2 + 7]),
                                        noise[:65535 * 2 + 7])))
    cases.append(('stored-empty', member(stored(b''), b'')))
    for flags in range(32):
        cases.append(('flags%d' % flags,
                      gz(text[:3000], flags=flags, extra=b'ab\x00cd',
                         name=b'access.log', comment=b'rotated')))
    m1, m2, m3 = gz(text[:5000]), gz(b''), gz(text[5000:9000], 1)
    cases.append(('members', m1 + m2 + m3))
    cases.append(('members-zeros', m1 + b'\x00' * 5 + m3 + b'\x00' * 9))
    cases.append(('member-zeros-only', m1 + b'\x00'))
    cases.append(('ndjson', gz(ndjson(20000, 7))))
    return cases


def damaged_corpus(seed=2):
    """(name, bytes): truncations, flips, bad trailers and invalid codes;
    most fail, some (a flipped mtime) still decode."""
    rng = random.Random(seed)
    small = gz(ndjson(6, 3), 9)
    dyn = gz(ndjson(40, 4), 9)
    cases = []
    for i in range(len(small)):
        cases.append(('trunc%d' % i, small[:i]))
    for i in range(len(dyn)):
        b = bytearray(dyn)
        b[i] ^= 1 << rng.randrange(8)
        cases.append(('flip%d' % i, bytes(b)))
        b = bytearray(dyn)
        b[i] = rng.randrange(256)
        cases.append(('set%d' % i, bytes(b)))
    fixed = gz(ndjson(10, 5), 6, strategy=zlib.Z_FIXED)
    for i in range(10, len(fixed) - 8):
        b = bytearray(fixed)
        b[i] ^= 1 << rng.randrange(8)
        cases.append(('fixedflip%d' % i, bytes(b)))
    st = member(stored(b'abc' * 50), b'abc' * 50)
    for i in range(10, 15):
        b = bytearray(st)
        b[i] ^= 0x10
        cases.append(('storedflip%d' % i, bytes(b)))
    crc = bytearray(small)
    crc[-8] ^= 1
    isz = bytearray(small)
    isz[-4] ^= 1
    cases += [('bad-crc', bytes(crc)), ('bad-isize', bytes(isz)),
              ('trailing-garbage', small + b'x'),
              ('trailing-zeros-garbage', small + b'\x00\x00\x01'),
              ('trailing-magic', small + b'\x1f\x8b'),
              ('trailing-partial-member', small + small[:20]),
              ('trailing-byte-1f', small + b'\x1f'),
              ('bad-method', small[:2] + b'\x07' + small[3:]),
              ('bad-magic', b'\x1f\x8c' + small[2:])]
    # invalid codes and distances, in fixed blocks
    for name, toks in (('lit286', [65, ('sym', 286)]),
                       ('lit287', [65, ('sym', 287)]),
                       ('dist30', [65, 66, ('dsym', 30)]),
                       ('dist31', [65, 66, ('dsym', 31)]),
                       ('too-far', [65, 66, (3, 3)]),
                       ('too-far-first', [(3, 1)])):
        body = fixed_block(toks).done() if name not in ('lit286', 'lit287',
                                                        'dist30', 'dist31') \
            else _raw_fixed(toks)
        cases.append((name, member(body, b'')))
    b = Bits()
    b.put(1, 1)
    b.put(3, 2)
    cases.append(('btype3', member(b.done() + b'\x00' * 8, b'')))
    cases += _bad_dynamic()
    return cases


def _raw_fixed(toks):
    b = Bits()
    b.put(1, 1)
    b.put(1, 2)
    for t in toks:
        if isinstance(t, int):
            fixed_lit(b, t)
        elif t[0] == 'sym':
            fixed_lit(b, t[1])
            b.put(0, 5)
        else:
            fixed_lit(b, 257)
            b.huff(t[1], 5)
    fixed_lit(b, 256)
    return b.done() + b'\x00' * 4


def _dynamic_header(hlit, hdist, clens, lens, bits=None):
    """A dynamic block header: HLIT/HDIST/HCLEN as given, the code-length
    code `clens` (19 lengths in symbol order) and `lens` coded with it."""
    order = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1,
             15]
    b = bits or Bits()
    b.put(1, 1)
    b.put(2, 2)
    b.put(hlit - 257, 5)
    b.put(hdist - 1, 5)
    b.put(15, 4)
    for s in order:
        b.put(clens[s], 3)
    codes = _canonical(clens)
    for v in lens:
        if isinstance(v, tuple):
            sym, extra, k = v
            b.huff(*codes[sym])
            b.put(extra, k)
        else:
            b.huff(*codes[v])
    return b


def _canonical(lens):
    code, nxt, out = 0, {}, {}
    for ln in range(1, 16):
        code = (code + sum(1 for x in lens if x == ln - 1 and ln > 1)) << 1 \
            if ln > 1 else 0
        nxt[ln] = code
    for s, ln in enumerate(lens):
        if ln:
            out[s] = (nxt[ln], ln)
            nxt[ln] += 1
    return out


def _bad_dynamic():
    """Code sets at and around zlib's limits: complete, over-subscribed,
    incomplete, one code of length 1, a repeat with nothing before it, a
    repeat past the end, no end-of-block code, too many symbols."""
    cl = [0] * 19
    cl[0] = cl[8] = 2                  # a complete code-lengths code
    cl[1] = cl[16] = cl[17] = cl[18] = 3
    z256 = [(18, 127, 7), (18, 107, 7)]
    out = []
    for name, hlit, hdist, lens in (
            ('dyn-over', 257, 1, [8] * 257 + [8]),
            ('dyn-repeat-first', 257, 1, [(16, 0, 2)] + [0] * 257),
            ('dyn-repeat-past', 257, 1, [(18, 127, 7)] * 3),
            ('dyn-no-eob', 257, 1, z256 + [0, 1]),
            ('dyn-one-code', 257, 1, z256 + [1, 1]),
            ('dyn-no-dist', 257, 1, z256 + [1, 0]),
            ('dyn-incomplete', 258, 1, z256 + [8, 8, 1]),
            ('dyn-too-many', 287, 1, [0] * 10)):
        b = _dynamic_header(hlit, hdist, cl, lens)
        b.put(0, 16)
        out.append((name, member(b.done() + b'\x00' * 8, b'')))
    return out
