"""Edge-case inputs and query plans shared by the CPU (hostcheck) and GPU
parity tests.  Everything here is checked oracle-vs-implementation, so the
cases may go beyond what the reference's own tests exercise (those are in
tests/golden)."""

import decimal
import json
import math
import random
import struct

from hostmirror import dn as mod_dn
from dragnet_b200 import query as mod_query

# ---------------------------------------------------------------------------
# handcrafted lines: JSON grammar corners, duplicates, nesting, types
# ---------------------------------------------------------------------------
EDGE_LINES = [
    b'{"a":1}', b'{"a":1} ', b' {"a":1}', b'\t{"a" : 1 }\r', b'{"a":1}x',
    b'{"a":1,}', b'{,"a":1}', b'{"a" 1}', b'{"a":}', b'{"a"}', b'{a:1}',
    b"{'a':1}", b'', b' ', b'{}', b'[]', b'[1,2', b'{"a":[1,2}', b'{"a":{]}',
    b'123', b'"str"', b'null', b'true', b'false', b'nul', b'tru', b'True',
    b'-', b'-0', b'01', b'1.', b'.5', b'1e', b'1e+', b'1.5e3', b'1E5', b'0e0',
    b'-0.0', b'1.0', b'{"a":01}', b'{"a":1.}', b'{"a":+1}', b'{"a":0x10}',
    b'{"a":NaN}', b'{"a":Infinity}', b'{"a":-Infinity}', b'{"a":1e999}',
    b'{"a":-1e999}', b'{"a":1e-999}',
    b'{"a":"\\u0041"}', b'{"a":"\\u004"}', b'{"a":"\\uZZZZ"}', b'{"a":"\\x41"}',
    b'{"a":"\\"}', b'{"a":"\\\\"}', b'{"a":"\\/"}', b'{"a":"a\\nb"}',
    b'{"a":"tab\there"}', b'{"a":"nul\x00"}', b'{"a":"del\x7f"}',
    b'{"a":"\xc3\xa9"}', b'{"a":"\\u00e9"}', b'{"a":"\xe2\x82\xac"}',
    b'{"a":"\\ud83d\\ude00"}', b'{"a":"\xf0\x9f\x98\x80"}',
    b'{"\\u0061":5}', b'{"\\u0061":5,"a":6}', b'{"a":5,"\\u0061":6}',
    b'{"a":1,"a":2}', b'{"a":{"b":1},"a":{"c":2}}', b'{"a":{"b":1},"a":3}',
    b'{"a.b":1,"a":{"b":2}}', b'{"a":{"b":2},"a.b":1}', b'{"a":{"b.c":3}}',
    b'{"a":{"b":{"c":4}}}', b'{"a":{"b.c":3,"b":{"c":4}}}',
    b'{"a.b.c":5,"a":{"b.c":3,"b":{"c":4}}}', b'{"a":{"b":5}}',
    b'{"a":{"b":null}}', b'{"a":{"b":true}}', b'{"a":{"b":false}}',
    b'{"a":{"b":"x"}}', b'{"a":{"b":[1,2]}}', b'{"a":{"b":{}}}',
    b'{"a":{"b":[]}}', b'{"a":{"b":[[1,2],[3]]}}', b'{"a":{"b":[null,1]}}',
    b'{"a":{"b":[{"x":1},"s",true,false,null,1.50,"q\\"r"]}}',
    b'{"a":{"b":[" 7 "]}}', b'{"a":[{"b":1}]}', b'{"a":"str","b":2}',
    b'{"a":5,"b":"5"}', b'{"a":"5","b":5}', b'{"a":"05"}', b'{"a":" 5 "}',
    b'{"a":"5e0"}', b'{"a":"0x5"}', b'{"a":""}', b'{"a":"abc"}', b'{"a":"ABC"}',
    b'{"a":200}', b'{"a":200.0}', b'{"a":2e2}', b'{"a":2.0e2}', b'{"a":"200"}',
    b'{"a":1e21}', b'{"a":1e-7}', b'{"a":123456789012345678901234567890}',
    b'{"a":0.1}', b'{"a":0.30000000000000004}', b'{"a":-5}', b'{"a":-0}',
    b'{"a":4.35}', b'{"a":9007199254740993}', b'{"a":1.7976931348623157e308}',
    b'{"a":5e-324}', b'{"a":0.000001}', b'{"a":1234.5678}', b'{"a":100000000000000000000}',
    b'{"b":1}', b'{"x":{"a":1}}', b'[{"a":1}]', b'{"a":1,"b":{"a":2}}',
    b'{"t":"2014-05-01T00:00:00.000Z","a":1}', b'{"t":"2014-05-01","a":1}',
    b'{"t":"2014-05-01T10:20","a":1}', b'{"t":"2014-05-01T10:20:30+02:00","a":1}',
    b'{"t":1398902400,"a":1}', b'{"t":1398902400.5,"a":1}', b'{"t":"nope","a":1}',
    b'{"t":null,"a":1}', b'{"t":true,"a":1}', b'{"t":{},"a":1}',
    b'{"t":["2014-05-01"],"a":1}', b'{"t":"\\u0032014-05-01","a":1}',
    b'{"t":"2014-02-30","a":1}', b'{"a":1,"t":"1969-12-31T23:59:59.500Z"}',
    b'{"fields":{"a":1},"value":3}', b'{"fields":{"a":1},"value":0}',
    b'{"fields":{"a":"x","b":2},"value":7}', b'{"fields":{},"value":1}',
    b'{"fields":{"a":1},"value":-1}', b'{"fields":{"a":1},"value":1.5}',
    b'{"fields":{"a":1},"value":"3"}', b'{"fields":[1],"value":3}',
    b'{"fields":{"a":1}}', b'{"value":3}', b'{"fields":{"a.b":9,"a":{"b":8}},"value":2}',
    b'{"a":' + b'[' * 40 + b']' * 40 + b'}',
    b'{"a":"' + b'x' * 300 + b'"}', b'{"k' + b'y' * 100 + b'":1,"a":2}',
    b'{"a":1,"pad":"' + b'p' * 5000 + b'"}',
    b'{"pad":"' + b'p' * 9000 + b'","a":"late"}',
    b'{"a":"\xff\xfe"}', b'{"a":"\xc3"}',
    b'{"a": [ 1 , 2 , { "b" : [ ] } ] , "b" : { } }',
    b'{"a":"x"}{"a":"y"}', b'{"a":"x"} {"a":"y"}', b'[1,2,3]', b'[[[]]]',
    b'{"":1}', b'{"":{"":2}}', b'{"a":{"":3}}', b'{"a.":4}', b'{".a":5}',
    b'{"a..b":6}', b'{"a":{"":{"b":7}}}',
]

SKINNER_LINES = [l for l in EDGE_LINES if b'"value"' in l or b'fields' in l] + [
    b'{"fields":{"req.method":"GET","x":1},"value":5}',
    b'{"fields":{"req":{"method":"PUT"}},"value":2}',
    b'not json', b'', b'{"fields":{"req.method":"GET"},"value":1}',
]


def rand_json(rng, depth=0):
    r = rng.random()
    if depth > 3 or r < 0.35:
        c = rng.randrange(9)
        if c == 0:
            return None
        if c == 1:
            return rng.random() < 0.5
        if c == 2:
            return rng.randrange(-50, 5000)
        if c == 3:
            return rng.choice([0.5, 1.25, 1e21, 1e-7, 123.456, -0.0, 2e2,
                               1.5e300, 4.35, 0.1])
        if c == 4:
            return rng.choice(['GET', 'PUT', 'a b', '', '200', ' 12 ', '1e3',
                               'x"y', 'tab\t', 'é', '€uro', '\U0001F600',
                               'null', 'true', '2014-05-01T00:00:00Z', '0x1f',
                               'Infinity', '-5', '5.0'])
        return rng.choice(['GET', 'HEAD', 'PUT', 'DELETE', 'x', 'y'])
    if r < 0.7:
        n = rng.randrange(0, 5)
        keys = ['a', 'b', 'c', 'a.b', 'b.c', 'req', 'method', 'x', '', 'length',
                '0', 't']
        return {rng.choice(keys): rand_json(rng, depth + 1) for _ in range(n)}
    return [rand_json(rng, depth + 1) for _ in range(rng.randrange(0, 4))]


def _dumps(rng, v):
    """JSON text with random (legal) formatting: whitespace, escapes,
    exponent spellings, duplicate keys."""
    if isinstance(v, dict):
        parts = []
        for k, x in v.items():
            ks = json.dumps(k)
            if k and rng.random() < 0.15:
                ks = '"' + ''.join('\\u%04x' % ord(ch) for ch in k) + '"'
            parts.append(ks + rng.choice([':', ' : ', ': ']) + _dumps(rng, x))
            if rng.random() < 0.08:       # duplicate key, later wins
                parts.append(ks + ':' + _dumps(rng, rand_json(rng, 3)))
        return '{' + rng.choice([',', ' , ', ', ']).join(parts) + '}'
    if isinstance(v, list):
        return '[' + rng.choice([',', ' ,']).join(_dumps(rng, x) for x in v) + ']'
    if isinstance(v, float) and rng.random() < 0.3 and v == int(v) and abs(v) < 1e15:
        return rng.choice(['%d.0', '%de0', '%d.00E+0']) % int(v)
    s = json.dumps(v, ensure_ascii=rng.random() < 0.5)
    return s


def random_lines(seed, n):
    rng = random.Random(seed)
    out = []
    for _ in range(n):
        v = rand_json(rng)
        if rng.random() < 0.8 and not isinstance(v, dict):
            v = {'a': v, 'b': rand_json(rng), 'req': {'method': rand_json(rng, 3)}}
        text = _dumps(rng, v)
        r = rng.random()
        if r < 0.04:
            text = text[:rng.randrange(0, max(1, len(text)))]   # truncated
        elif r < 0.06:
            text += rng.choice(['x', ',', '}', ' 1'])
        out.append(text.encode('utf-8'))
    return out


# ---------------------------------------------------------------------------
# query plans
# ---------------------------------------------------------------------------

class DroppedBreakdown(ValueError):
    pass


def written_breakdowns(argv):
    """The field names written after each -b of argv: the text split at
    commas outside [...], each piece without its [...] attributes."""
    names = []
    for i in range(1, len(argv)):
        if argv[i - 1] not in ('-b', '--breakdowns'):
            continue
        depth, piece = 0, ''
        for ch in argv[i] + ',':
            if ch == '[':
                depth += 1
            elif ch == ']':
                depth -= 1
            elif ch == ',' and depth == 0:
                if piece:
                    names.append(piece)
                piece = ''
            elif depth == 0:
                piece += ch
    return names


def make_plan(argv, ds=None, allow_dropped=False):
    """`dn scan ARGV` against datasource properties ds -> plan dict.

    dn's breakdown parser drops a trailing bare name of one character (`-b a`
    groups by nothing, `-b a,b` by a alone; lib/attr-parser.js:73 tests
    `j < str.length - 1`).  A query that means to group by such a name must
    end it with a comma (`-b a,`); one that loses a name raises
    DroppedBreakdown unless allow_dropped is set."""
    ds = ds or {}
    options = mod_dn.dnParseArgs(list(argv))
    q = mod_dn.dnQueryConfig(options)['query']
    plan = mod_query.scan_plan(q, ds_filter=ds.get('filter'),
                               time_field=ds.get('timeField'),
                               data_format=ds.get('dataFormat', 'json'))
    got = [b['name'] for b in plan['breakdowns']]
    want = written_breakdowns(argv)
    if got != want and not allow_dropped:
        raise DroppedBreakdown('%r groups by %r, not by %r' % (argv, got, want))
    return plan


EDGE_QUERIES = [
    ([], None),
    (['-b', 'a,'], None),
    (['-b', 'a.b'], None),
    (['-b', 'a.b.c'], None),
    (['-b', 'a,b,'], None),
    (['-b', 'a[aggr=quantize]'], None),
    (['-b', 'a[aggr=lquantize,step=100]'], None),
    (['-b', 'b[aggr=lquantize,step=7],a,'], None),
    (['-b', 'a.b[aggr=quantize],req.method'], None),
    (['-f', '{"eq":["a",200]}'], None),
    (['-f', '{"eq":["a","200"]}', '-b', 'a,'], None),
    (['-f', '{"ne":["a",5]}', '-b', 'a,'], None),
    (['-f', '{"lt":["a",100]}', '-b', 'a,'], None),
    (['-f', '{"ge":["a","abc"]}', '-b', 'a,'], None),
    (['-f', '{"le":["a","5"]}', '-b', 'a,'], None),
    (['-f', '{"gt":["a.b",1]}', '-b', 'a.b'], None),
    (['-f', '{"eq":["a",true]}', '-b', 'a,'], None),
    (['-f', '{"eq":["a.b","1,2"]}', '-b', 'a.b'], None),
    (['-f', '{"eq":["a","[object Object]"]}'], None),
    (['-f', '{"and":[{"ge":["a",1]},{"lt":["a",300]}]}', '-b', 'a,'], None),
    (['-f', '{"or":[{"eq":["a","x"]},{"eq":["b",2]}]}', '-b', 'a,b,'], None),
    (['-f', '{"or":[{"and":[{"eq":["a",1]},{"eq":["b",1]}]},{"gt":["a",100]}]}'],
     None),
    (['-f', '{"eq":["req.method","GET"]}', '-b', 'req.method'],
     {'filter': {'ne': ['a', 1]}}),
    (['-b', 'ts[date,field=t,aggr=lquantize,step=86400]'], None),
    (['-b', 'ts[date,field=t],a,'], None),
    (['-b', 'a,', '--after', '2014-04-30', '--before', '2014-05-02'],
     {'timeField': 't'}),
    (['-b', 't[date],a,'], None),
    (['-b', 'a[date,field=t]'], None),
    (['-b', 'x,'], None),
    (['-b', ''], None) if False else (['-b', 'length'], None),
    (['-b', 'a.0'], None),
    (['-b', 'a.b.1,a.b.length'], None),
    (['-b', '0.a,a.length'], None),
    (['-b', 'a.b.0.1'], None),
    (['-f', '{"eq":["a.b.length",2]}', '-b', 'a.b'], None),
    (['-b', 'a.b.0.x'], None),
]

SKINNER_QUERIES = [
    ([], {'dataFormat': 'json-skinner'}),
    (['-b', 'a,'], {'dataFormat': 'json-skinner'}),
    (['-b', 'req.method'], {'dataFormat': 'json-skinner'}),
    (['-b', 'a.b,b,'], {'dataFormat': 'json-skinner'}),
    (['-f', '{"eq":["a",1]}', '-b', 'a,'], {'dataFormat': 'json-skinner'}),
]

BASELINE_QUERIES = {
    'C2': (['-b', 'req.method'], None),
    'C3': (['-b', 'req.method,res.statusCode', '-f',
            '{"eq":["req.method","GET"]}'], None),
    'C4': (['-b', 'latency[aggr=quantize]'], None),
    'C5': (['-b', 'operation,req.method,host'], None),
    'count': ([], None),
    'date': (['-b', 'ts[date,field=time,aggr=lquantize,step=3600],'
              'req.method'], None),
    'bounds': (['-b', 'host', '--after', '2014-05-31T22:00:00Z', '--before',
                '2014-05-31T23:00:00Z'], {'timeField': 'time'}),
    'caller': (['-b', 'req.caller,res.statusCode', '-f',
                '{"ne":["req.caller","admin"]}'], None),
    'lq': (['-b', 'dataLatency[aggr=lquantize,step=100],host'], None),
    'url': (['-b', 'req.url'], None),
    'urlhost': (['-b', 'req.url,host'], None),
}


# scalar forms behind one skeleton ({"a":<bare>,"s":"<string>"}): what the
# template matcher's wildcard scans must accept, reject or hand to the automaton
BARE_FORMS = [b'0', b'-0', b'1', b'12', b'123', b'1234', b'12345', b'123456',
              b'1234567', b'12345678', b'123456789', b'123456789012345',
              b'1234567890123456', b'12345678901234567890', b'-1', b'-12',
              b'-123', b'-1234', b'-12345', b'-123456789012345',
              b'-1234567890123456', b'0.5', b'-0.5', b'1e5', b'1E+5', b'1e-5',
              b'1.5e3', b'1.0', b'100.000', b'0e0', b'0.0', b'-0.0', b'1e400',
              b'-1e400', b'1e-400', b'01', b'-01', b'00', b'1.', b'.5', b'1e',
              b'1e+', b'-', b'+1', b'0x10', b'1a', b'1 ', b' 1', b'true',
              b'false', b'null', b'tru', b'nul', b'falsy', b'truee', b'nulll',
              b'True', b'NaN', b'Infinity', b'-Infinity', b'1,', b'1}',
              b'"x"', b'{}', b'[]', b'[1]', b'{"b":1}', b'']
STR_FORMS = [b'', b'a', b'ab', b'abc', b'abcd', b'abcde', b'abcdefgh',
             b'abcdefghi', b'x' * 63, b'x' * 64, b'x' * 65, b'\\n', b'a\\"b',
             b'\\\\', b'a\\u0041', b'\x01', b'a\tb', b'\x7f', b'\xc3\xa9',
             b'\xf0\x9f\x98\x80', b'\xff\xfe', b'a"', b'"', b'a\\']


def scalar_lines():
    out = []
    for i, f in enumerate(BARE_FORMS):
        out.append(b'{"a":' + f + b',"s":"k%d"}' % (i % 5))
    for i, f in enumerate(STR_FORMS):
        out.append(b'{"a":%d,"s":"' % (i % 7) + f + b'"}')
    return out


# ---------------------------------------------------------------------------
# template fuzz: a few record shapes, every line one of them with re-rolled
# scalar values (nasty strings, every number form, bare-scalar type flips) and
# a sprinkle of damage -- what the template matcher sees in the field
# ---------------------------------------------------------------------------

def _reroll(rng, v):
    if isinstance(v, dict):
        return {k: _reroll(rng, x) for k, x in v.items()}
    if isinstance(v, list):
        return [_reroll(rng, x) for x in v]
    if isinstance(v, str):
        return rng.choice(['GET', 'PUT', 'x', '', 'a b', '\u00e9', 'x"y', 'tab\t',
                           '\U0001F600', '2014-05-01T00:00:00Z', '200', ' 12 ',
                           '\\', '/', '\u20acuro' * 3, 'long' * 9])
    return rng.choice([None, True, False, 0, -0.0, 7, -12, 123456789012345,
                       1234567890123456, 0.5, 1e21, 1e-7, 1.5e300, 2e2, 4.35,
                       100])


def _dumps_shape(v, fmt, rng):
    """Formatting (separators) is a property of the shape, not of the line."""
    if isinstance(v, dict):
        sep, col = fmt.choice([',', ', ']), fmt.choice([':', ': '])
        return '{' + sep.join(json.dumps(k) + col + _dumps_shape(x, fmt, rng)
                              for k, x in v.items()) + '}'
    if isinstance(v, list):
        return '[' + ','.join(_dumps_shape(x, fmt, rng) for x in v) + ']'
    if isinstance(v, float) and rng.random() < 0.3 and v == int(v) and \
            abs(v) < 1e15:
        return rng.choice(['%d.0', '%de0', '%d.00E+0']) % int(v)
    return json.dumps(v, ensure_ascii=rng.random() < 0.5)


def template_fuzz_lines(seed, n, nshapes=6):
    rng = random.Random(seed)
    shapes = []
    while len(shapes) < nshapes:
        v = rand_json(rng)
        if isinstance(v, dict) and len(v) >= 1:
            shapes.append((v, rng.randrange(1 << 30)))
    out = []
    for _ in range(n):
        v, fmt = rng.choice(shapes)
        text = _dumps_shape(_reroll(rng, v), random.Random(fmt), rng)
        r = rng.random()
        if r < 0.03:
            text = text[:rng.randrange(0, max(1, len(text)))]
        elif r < 0.05:
            text += rng.choice(['x', ',', '}', ' 1', ' '])
        elif r < 0.07:
            text = text.replace(':', ' :', 1)
        out.append(text.encode('utf-8'))
    return out


# ---------------------------------------------------------------------------
# group-by corpora (tests/test_aggregation_host.py, test_gpu_aggregation.py):
# many distinct keys, keys whose hashes collide on purpose, key lengths at the
# tally tiers' edges, weights.  Everything is a function of its arguments.
# ---------------------------------------------------------------------------

M64 = (1 << 64) - 1
M32 = (1 << 32) - 1
KEY_MAX = 512           # plan.h: longest encoded group key
SKEY = 40               # scan_kernel.cuh DNG_SKEY: key bytes inline in tier 1
F_MAXKEY = 256          # fast.h: longest key the F path tallies itself
# printable ASCII that needs no escape in a JSON string
_PLAIN = bytes(c for c in range(0x20, 0x7f) if c not in b'"\\')
_PLAIN_SET = frozenset(_PLAIN)


def encode_key(*cols):
    """The encoded group key of discrete columns (DESIGN §2): per column a
    little-endian u16 length, then the bytes of String(value)."""
    return b''.join(len(c).to_bytes(2, 'little') + c for c in cols)


def _g_step(h, w):
    h ^= w
    h = (h * 0xff51afd7ed558ccd) & M64
    return h ^ (h >> 32)


def _g_words(key):
    key = key + b'\0' * (-len(key) % 8)
    return [int.from_bytes(key[i:i + 8], 'little')
            for i in range(0, len(key), 8)]


def key_hash(key):
    """record.cuh key_hash: the general kernels' 64-bit hash of a key."""
    h = 0x9E3779B97F4A7C15 ^ ((len(key) * 0xff51afd7ed558ccd) & M64)
    for w in _g_words(key):
        h = _g_step(h, w)
    h ^= h >> 29
    h = (h * 0xc4ceb9fe1a85ec53) & M64
    return h ^ (h >> 32)


def _fmix(h, w):
    h = ((h ^ w) * 0x9E3779B1) & M32
    return h ^ (h >> 15)


def _f_state(s, nwords=None):
    """fast.cuh fkey_hash of one discrete column s, before its finaliser,
    after the first nwords 4-byte words of s (all of them by default)."""
    h = _fmix(0x2545F491, len(s))
    p = s + b'\0' * (-len(s) % 4)
    words = [int.from_bytes(p[i:i + 4], 'little') for i in range(0, len(p), 4)]
    for w in words[:nwords]:
        h = _fmix(h, w)
    return h


def fkey_hash(s):
    """fast.cuh fkey_hash of a plan with one discrete column, value s."""
    h = _f_state(s)
    h ^= h >> 16
    h = (h * 0x85ebca6b) & M32
    return h ^ (h >> 13)


def _rand_plain(rng, n):
    return bytes(rng.choice(_PLAIN) for _ in range(n))


def g_collisions(slen, count, seed):
    """count strings of slen bytes (slen + 2 a multiple of 8, >= 22) whose
    one-column keys have the same 64-bit general hash: equal first word, the
    second-to-last word drawn at random, the last one solved for (the hash
    is invertible word by word) until it is printable."""
    klen = slen + 2
    assert klen % 8 == 0 and klen >= 24
    rng = random.Random(seed)
    base = _rand_plain(rng, slen)
    key = encode_key(base)
    words = _g_words(key)
    h = 0x9E3779B97F4A7C15 ^ ((klen * 0xff51afd7ed558ccd) & M64)
    for w in words[:-2]:
        h = _g_step(h, w)
    target = _g_step(h, words[-2]) ^ words[-1]
    out = {base}
    while len(out) < count:
        w1 = _rand_plain(rng, 8)
        w2 = (target ^ _g_step(h, int.from_bytes(w1, 'little'))).to_bytes(
            8, 'little')
        if _PLAIN_SET.issuperset(w2):
            out.add(base[:slen - 16] + w1 + w2)
    out = sorted(out)
    assert len({key_hash(encode_key(s)) for s in out}) == 1
    return out


def f_collisions(slen, count, seed):
    """count strings of slen bytes (a multiple of 4, >= 8) with the same F
    hash (fkey_hash, one discrete column): the last word solved for."""
    assert slen % 4 == 0 and slen >= 8
    rng = random.Random(seed)
    base = _rand_plain(rng, slen)
    nw = slen // 4
    h = _f_state(base, nw - 2)
    target = _f_state(base)
    out = {base}
    while len(out) < count:
        w1 = _rand_plain(rng, 4)
        hs = _fmix(h, int.from_bytes(w1, 'little'))
        # _fmix(hs, w) == target  <=>  (hs ^ w) * K == unmix(target)
        x = target
        x ^= x >> 15
        x ^= x >> 30
        x = (x * pow(0x9E3779B1, -1, 1 << 32)) & M32
        w2 = (x ^ hs).to_bytes(4, 'little')
        if _PLAIN_SET.issuperset(w2):
            out.add(base[:slen - 8] + w1 + w2)
    out = sorted(out)
    assert len({fkey_hash(s) for s in out}) == 1
    return out


GLOBAL_SLOT = 1020


def index_collisions(slen, count, hashfn, shift, bits, seed, pool=60000,
                     slot=None):
    """count distinct strings of slen bytes whose hashfn(string) agree in
    bits [shift, shift + bits) (they probe from the same slot of a table of
    up to 2^bits entries) but not in the whole hash: the largest such group
    of a seeded pool, or the group of that slot."""
    rng = random.Random(seed)
    groups = {}
    mask = (1 << bits) - 1
    for _ in range(pool):
        s = _rand_plain(rng, slen)
        groups.setdefault((hashfn(s) >> shift) & mask, set()).add(s)
    best = max(groups.values(), key=len) if slot is None else groups[slot]
    assert len(best) >= count, (len(best), count)
    return sorted(best)[:count]


def gkey_hash(s):
    return key_hash(encode_key(s))


def collision_groups(seed=0):
    """name -> strings that meet in one slot of one tally tier (see
    test_aggregation_host.py for what each one has to reach)."""
    return {
        # F inline tier: index (h >> 7) & mask1, mask1 <= 1023, 8 probes
        'f_index': index_collisions(28, 40, fkey_hash, 7, 10, seed + 1),
        # F inline tier: equal claims, fkey_equal decides
        'f_full': f_collisions(24, 40, seed + 2),
        # general tier 1 (keys <= 40 B): bits 40-49, 8 probes
        'g1_index': index_collisions(30, 40, gkey_hash, 40, 10, seed + 3),
        # general tier 1, equal tags: the inline word compare decides
        'g1_full': g_collisions(22, 40, seed + 4),
        # general tier 2 (keys > 40 B): bits 28-39, 24 probes
        'g2_index': index_collisions(46, 40, gkey_hash, 28, 12, seed + 5,
                                     pool=160000),
        # tier 2 and the global table, equal tags: the arena bytes decide
        'g2_full': g_collisions(46, 40, seed + 6),
        # global table of DNG_TABLE_CAP=1024: bits 17-26
        # global table of DNG_TABLE_CAP=1024: bits 17-26, home slot 1020,
        # so that the chain wraps around the table's end
        'global_index': index_collisions(20, 40, gkey_hash, 17, 10,
                                         seed + 7, slot=GLOBAL_SLOT),
    }


def kv_line(key, v, pad):
    return b'{"key":' + json.dumps(key.decode('latin-1')).encode() + \
        b',"val":%d,"pad":"%s"}' % (v, pad)


def kv_lines(keys, n, seed, pad=40):
    """n records {"key":key,"val":..,"pad":..} cycling through keys in a seeded
    order, so that every chunk (and CTA) sees keys of every group."""
    rng = random.Random(seed)
    padb = b'p' * pad
    order = list(keys)
    out = []
    while len(out) < n:
        rng.shuffle(order)
        out.extend(kv_line(k, i % 7, padb) for i, k in
                   enumerate(order[:n - len(out)]))
    return out


def sweep_lines(k, n, seed=0):
    """n records over k distinct keys k%d (lengths 2-8: tier 1 everywhere)."""
    rng = random.Random(seed)
    return [b'{"key":"k%d","val":%d,"pad":"%s"}' %
            (rng.randrange(k), i % 7, b'p' * (30 + i % 11)) for i in range(n)]


def skew_lines(n, seed=0, hot=16, tail=100000):
    """Half the records on hot keys, the rest over a long tail: the hot keys
    are in every CTA's tier 1 while the tail fills tier 2 and the table."""
    rng = random.Random(seed)
    out = []
    for i in range(n):
        key = b'hot%d' % rng.randrange(hot) if i % 2 else \
            b'tail-%d' % rng.randrange(tail)
        out.append(b'{"key":"%s","val":%d,"pad":"%s"}' % (key, i % 5,
                                                      b'q' * (24 + i % 13)))
    return out


# encoded key lengths (one column: 2 + len): both sides of the inline tier
# (40), of 8-byte word edges, of the F path's 256 and of KEY_MAX (512; the
# longest accepted one-column key is 512 bytes: a 510-byte string)
KEY_LENGTHS = [38, 39, 40, 41, 42, 47, 48, 49, 254, 255, 256, 257, 258, 511,
               512]


def key_length_lines(two=False, seed=0, reps=40):
    """Records whose keys (-b key, or with two=True -b key,key2) are KEY_LENGTHS
    long, a few variants of each, repeated so that every key is tallied from
    many CTAs."""
    rng = random.Random(seed)
    recs = []
    for kl in KEY_LENGTHS:
        for var in range(4):
            s = (b'%d-%d-' % (kl, var) + _rand_plain(rng, kl))[:kl - 2]
            if not two:
                recs.append(b'{"key":"%s","pad":"x"}' % s)
                continue
            # two columns: 2 + a + 2 + b == kl, a <= 500
            a = min(len(s) - 2, 500) if var % 2 else (len(s) - 2) // 2
            recs.append(b'{"key":"%s","key2":"%s","pad":"y"}' % (s[:a],
                                                             s[a:len(s) - 2]))
    out = []
    for r in range(reps):
        rng.shuffle(recs)
        out.extend(recs)
    return out


def merge_apart_lines(reps=50):
    """Keys that must stay apart although their bytes nearly agree, and
    spellings of one value that must merge into one key."""
    apart = []
    for n in (5, 6, 7, 13, 14, 15, 21, 22, 23, 37, 38, 39, 45, 46, 47):
        stem = b'w' * (n - 1)
        # differ only in the last byte (the last, zero padded key word)
        apart += [stem + b'a', stem + b'b', stem + b'\x7e']
    recs = [b'{"key":"%s","key2":"z","pad":"mmmmmmmm"}' % s for s in apart]
    recs += [
        b'{"key":"a","key2":"z","pad":"mmmmmmmm"}',
        b'{"key":"a\\u0000","key2":"z","pad":"mmmmmmmm"}',
        b'{"key":"xy","key2":"","pad":"mmmmmmmm"}',
        b'{"key":"x","key2":"y","pad":"mmmmmmmm"}',
        b'{"key":"","key2":"xy","pad":"mmmmmmmm"}',
        b'{"key":"ab","key2":"","pad":"mmmmmmmm"}',
        b'{"key":"a","key2":"\\u0000","pad":"mmmmmmmm"}',
        # String(value) of numbers: one key
        b'{"key":1,"key2":"z","pad":"mmmmmmmm"}',
        b'{"key":1.0,"key2":"z","pad":"mmmmmmmm"}',
        b'{"key":1e0,"key2":"z","pad":"mmmmmmmm"}',
        b'{"key":"1","key2":"z","pad":"mmmmmmmm"}',
        b'{"key":10e-1,"key2":"z","pad":"mmmmmmmm"}',
        b'{"key":1,"key2":1.0,"pad":"mmmmmmmm"}',
        b'{"key":"1","key2":"1","pad":"mmmmmmmm"}',
    ]
    out = []
    for r in range(reps):
        out.extend(recs[r % len(recs):] + recs[:r % len(recs)])
    return out


# bucketized merges (-0 and 0, spellings of one number)
BUCKET_LINES = [b'{"num":%s,"pad":"mmmmmmmmmmmm"}' % v for v in
                (b'0', b'-0', b'0.0', b'-0.0', b'0e5', b'1', b'1.0', b'1e0',
                 b'"1"', b'2', b'3', b'-1', b'255', b'256')] * 30


# json-skinner weights: the tally's w <= 255 inline route and w > 255 route
WEIGHTS = [b'0', b'1', b'254', b'255', b'256', b'257', b'2147483648',
           b'4294967295', b'4294967296', b'1099511627776', b'9007199254740992',
           b'2.5e2', b'256.0', b'9007199254740993', b'9007199254740994']


def weight_lines(seed=0, nkeys=20000, n=200000):
    """Skinner points: every weight on three shared keys (each key takes the
    whole list in turn; the weights of 2^40 and more only in the first eight
    rounds per key), weights <= 255 and > 255 mixed over a high-cardinality
    set, and keys all of whose points weigh 0.  Every sum stays below 2^63
    (weight_sums)."""
    rng = random.Random(seed)
    nw = len(WEIGHTS)
    out = []
    for i in range(n):
        if i % 4 == 0:
            j = i // 4
            k = b'shared%d' % (j // nw % 3)
            w = WEIGHTS[j % nw] if j < nw * 3 * 8 else WEIGHTS[j % 8]
        elif i % 50 == 1:
            # keys all of whose points weigh 0: points of value 0
            k = b'zero%d' % (i % 7)
            w = rng.choice([b'0', b'0.0', b'-0'])
        else:
            k = b'key%d' % rng.randrange(nkeys)
            w = rng.choice(WEIGHTS[:11] + [b'2.5e2', b'256.0'])
        out.append(b'{"fields":{"key":"%s"},"value":%s}' % (k, w))
    return out


def weight_sums(lines):
    """key -> exact sum of the weight_lines records' values, as Python
    integers: a value counts when it is a whole number from 0 to 2^53 as a
    double (9007199254740993 reads as 2^53; 9007199254740994 does not
    count)."""
    sums = {}
    for ln in lines:
        doc = json.loads(ln)
        v = float(doc['value'])
        if v != int(v) or not 0 <= v <= 1 << 53:
            continue
        k = doc['fields']['key'].encode()
        sums[k] = sums.get(k, 0) + int(v)
    return sums


# ---------------------------------------------------------------------------
# value sweep (tests/test_value_sweep_host.py, test_gpu_value_sweep.py): a few
# record shapes, each field a value where JS semantics are easy to get wrong.
# Lines are 120-200 bytes, so that the F kernel keeps its chunks (at most 128
# lines) and learns the shapes as templates.
# ---------------------------------------------------------------------------

TWO53 = 1 << 53
# steps of the lquantize queries: every m * step and its neighbouring doubles
# are numbers of the sweep
SWEEP_STEPS = [1, 7, 100, 2147483647, -3, 3600, 86400]
# a number of the sweep the relational filters compare with (with its two
# neighbours, also numbers of the sweep)
SWEEP_CONST = 1234.5678
# code points at the UTF-8 (1/2/3/4 bytes) and UTF-16 (surrogates) edges
SWEEP_CPS = [0x41, 0x7a, 0x7f, 0x80, 0xe9, 0x7ff, 0x800, 0xd7ff, 0xe000,
             0xff61, 0xfffd, 0xffff, 0x10000, 0x1f600, 0x10ffff]
SWEEP_NSTR = ['26', ' 26 ', '\u00a026\ufeff', '\ufeff26', '\u300026', '-0',
              '0', '', ' ', '1e3', '1E+3', '.5', '5.', '+5', '-5', '0x1F',
              '0X1f', '0o17', '0b101', '0x', '0b2', 'Infinity', '-Infinity',
              '+Infinity', 'infinity', 'NaN', 'abc', '12abc', '1_000', '--5',
              '9007199254740993', '1e309', '-1e309', '5e-324',
              '00026', '2.6e1', '26.000', '0.1', '\u00a0', '\u2028-7\u2029']


def _f64(u):
    return struct.unpack('<d', struct.pack('<Q', u))[0]


def sweep_number(rng):
    """The text of a bare JSON number."""
    c = rng.randrange(10)
    if c == 0:
        nd = rng.randint(1, 20)
        v = rng.randrange(10 ** (nd - 1) if nd > 1 else 0, 10 ** nd)
        return ('-' if rng.random() < 0.3 else '') + str(v)
    if c == 1:
        # 16-digit integers above 2^53: their key is JS String(value), not
        # their own digits
        return str(rng.randrange(TWO53 + 1, 10 ** 16))
    if c == 2:
        return rng.choice([str(TWO53 - 1), str(TWO53), str(TWO53 + 1),
                           str(TWO53 + 2), str(TWO53 + 3), '-' + str(TWO53 + 1),
                           '-' + str(TWO53 - 1), '-0', '0', '0.0', '-0.0',
                           '0e0', '-0e-0', '1.7976931348623157e308',
                           '1.7976931348623158e308', '1e309', '-1e309',
                           '5e-324', '2.5e-324', '2.4703282292062328e-324',
                           '2.2250738585072014e-308', '2.225073858507201e-308',
                           '123456789012345', '-123456789012345',
                           '999999999999999', '1000000000000000',
                           '1e21', '1e-7', '100000000000000000000'])
    if c == 3:
        # a random binary64: shortest repr, or 17-25 significant digits
        while True:
            x = _f64(rng.getrandbits(64))
            if math.isfinite(x):
                break
        if rng.random() < 0.5:
            return repr(x)
        return '%.*e' % (rng.randint(16, 24), x)
    if c == 4:
        # exponent spellings: E+, e-, trailing zeros, leading fraction zeros
        m = rng.randrange(1, 10 ** rng.randint(1, 6))
        e = rng.randint(-30, 30)
        return rng.choice(['%dE+%d', '%de-%d', '%d.000e%d', '%d00E-%d',
                           '0.000%de%d']) % (m, abs(e))
    if c == 5:
        # halfway between two neighbouring doubles, written out exactly
        k = rng.randint(40, 75)
        a = _f64(rng.randrange(1 << 52) | (1023 + k) << 52)
        mid = (decimal.Decimal(a) + decimal.Decimal(math.nextafter(a, math.inf))) / 2
        return format(mid, 'f')
    if c == 6:
        # subnormals
        x = _f64(rng.randrange(1, 1 << 52))
        return repr(x) if rng.random() < 0.5 else '%.*e' % (rng.randint(16, 22), x)
    if c == 7:
        # 2^k, k = -3..70, and its neighbours
        x = math.ldexp(1.0, rng.randint(-3, 70))
        x = rng.choice([x, x, math.nextafter(x, 0), math.nextafter(x, math.inf)])
        if x == int(x) and rng.random() < 0.5:
            return str(int(x))
        return repr(-x if rng.random() < 0.2 else x)
    if c == 8:
        # m * step, with its neighbouring doubles
        s = rng.choice(SWEEP_STEPS)
        x = float(rng.randint(-3000, 3000) * s)
        x = rng.choice([x, x, math.nextafter(x, -math.inf),
                        math.nextafter(x, math.inf)])
        return str(int(x)) if x == int(x) and rng.random() < 0.5 else repr(x)
    # the filters' constant and its neighbours
    return repr(rng.choice([SWEEP_CONST, math.nextafter(SWEEP_CONST, 0),
                            math.nextafter(SWEEP_CONST, math.inf), 26.0,
                            float(TWO53)]))


def sweep_string(rng):
    """(the JSON text of a string body, whether it holds a \\u escape)."""
    cps = [rng.choice(SWEEP_CPS) for _ in range(rng.randint(0, 4))]
    if rng.random() < 0.04:
        # escaped: the F path hands these to the general parser
        out = []
        for cp in cps or [0x41]:
            if cp < 0x10000:
                out.append('\\u%04x' % cp)
            else:
                v = cp - 0x10000
                out.append('\\u%04X\\u%04X' % (0xd800 + (v >> 10),
                                                0xdc00 + (v & 0x3ff)))
        return ''.join(out), True
    return ''.join(chr(cp) for cp in cps), False


def sweep_date(rng):
    """(a date string, its (y, mo, d, h, mi, s, ms, offset minutes) or None
    for one that is not a date).  Only ISO forms: nothing V8's legacy parser
    would read."""
    y = rng.randint(0, 9999)
    mo = rng.randint(1, 12)
    d = rng.choice([rng.randint(1, 28), 29, 30, 31])
    h, mi, s, ms = (rng.randint(0, 23), rng.randint(0, 59), rng.randint(0, 59),
                    rng.randint(0, 999))
    r = rng.random()
    if r < 0.1:
        h, mi, s, ms = 23, 59, 59, 999
    elif r < 0.15:
        h, mi, s, ms = 0, 0, 0, 0
    ymd = '%04d-%02d-%02d' % (y, mo, d)
    c = rng.random()
    if c < 0.85:
        return ymd + 'T%02d:%02d:%02d.%03dZ' % (h, mi, s, ms), \
            (y, mo, d, h, mi, s, ms, 0)
    if c < 0.89:
        return ymd + 'T%02d:%02d:%02dZ' % (h, mi, s), (y, mo, d, h, mi, s, 0, 0)
    if c < 0.93:
        off = rng.choice([-1, 1]) * rng.randint(0, 23 * 60 + 59)
        return ymd + 'T%02d:%02d:%02d.%03d%s%02d:%02d' % (
            h, mi, s, ms, '-' if off < 0 else '+', abs(off) // 60,
            abs(off) % 60), (y, mo, d, h, mi, s, ms, off)
    if c < 0.96:
        return ymd, (y, mo, d, 0, 0, 0, 0, 0)
    if c < 0.98:
        return ymd + rng.choice(['T24:00:00Z', 'T24:00:00.000Z', 'T24:00']), \
            (y, mo, d, 24, 0, 0, 0, 0)
    return rng.choice(['', 'x', 'never']), None


def value_sweep_records(seed, n):
    """n records as dicts of field -> text: num (a bare number), nstr (a
    numeric string's body), str (a string's body), str_esc (it holds a \\u
    escape), ts (a date string), date (ts's parts), shape (0-2)."""
    rng = random.Random(seed)
    out = []
    for _ in range(n):
        s, esc = sweep_string(rng)
        ts, date = sweep_date(rng)
        out.append({'num': sweep_number(rng), 'nstr': rng.choice(SWEEP_NSTR)
                    if rng.random() < 0.7 else sweep_number(rng),
                    'str': s, 'str_esc': esc, 'ts': ts, 'date': date,
                    'shape': rng.randrange(3), 'len': rng.randint(130, 195)})
    return out


_SWEEP_SHAPES = [
    '{"num":%(num)s,"nstr":"%(nstr)s","str":"%(str)s","ts":"%(ts)s",'
    '"pad":"%(pad)s"}',
    '{"ts":"%(ts)s","host":"%(pad)s","num":%(num)s,"str":"%(str)s",'
    '"nstr":"%(nstr)s"}',
    '{"kind":"sweep","str":"%(str)s","req":{"ts":"%(ts)s"},'
    '"nstr":"%(nstr)s","num":%(num)s,"ts":"%(ts)s","pad":"%(pad)s"}',
]


def value_sweep_line(rec):
    d = dict(rec, pad='')
    text = _SWEEP_SHAPES[rec['shape']] % d
    d['pad'] = 'p' * max(4, rec['len'] - len(text.encode('utf-8')))
    return (_SWEEP_SHAPES[rec['shape']] % d).encode('utf-8')


def value_sweep_lines(seed, n):
    return [value_sweep_line(r) for r in value_sweep_records(seed, n)]


def _iso_ms(ms):
    from dragnet_b200 import jsdate
    return jsdate.to_iso_string(ms)


SWEEP_STR_CONSTS = ['｡', '\U0001f600']     # U+FF61 sorts above U+1F600


def sweep_queries(records):
    """name -> (argv, datasource properties, kind, arg) for a sweep corpus;
    kind and arg say what sweep_reference derives (None: nothing)."""
    q = {
        'num': (['-b', 'num,'], None, 'discrete', None),
        'str': (['-b', 'str,'], None, None, None),
        'nstr': (['-b', 'nstr,'], None, None, None),
        'num_p2': (['-b', 'num[aggr=quantize]'], None, 'p2', None),
        'nstr_p2': (['-b', 'nstr[aggr=quantize]'], None, None, None),
    }
    for s in (1, 7, 100, 2147483647, 0, -3):
        q['num_lq%d' % s] = (['-b', 'num[aggr=lquantize,step=%d]' % s],
                             None, 'linear', s)
    for s in (1, 3600, 86400):
        q['ts_lq%d' % s] = (['-b', 'ts[date,field=ts,aggr=lquantize,step=%d]'
                             % s], None, 'date', s)
    # --after/--before on two records' seconds, and a millisecond either side
    secs = sorted({_date_ms(r['date']) // 1000 * 1000 for r in records[:50]
                   if r['date'] and r['date'][3] < 24})
    lo, hi = secs[len(secs) // 4], secs[3 * len(secs) // 4]
    for d in (-1, 0, 1):
        q['bounds%+d' % d] = (['-b', 'nstr,', '--after', _iso_ms(lo + d),
                               '--before', _iso_ms(hi - d)],
                              {'timeField': 'ts'}, None, None)
    consts = [('c', repr(SWEEP_CONST)),
              ('c-', repr(math.nextafter(SWEEP_CONST, 0))),
              ('c+', repr(math.nextafter(SWEEP_CONST, math.inf))),
              ('2^53', str(TWO53)), ('"26"', '"26"')]
    for op in ('eq', 'ne', 'lt', 'le', 'gt', 'ge'):
        for cname, c in consts:
            q['%s_num_%s' % (op, cname)] = (
                ['-f', '{"%s":["num",%s]}' % (op, c), '-b', 'nstr,'], None,
                'filter', (op, 'num', json.loads(c)))
        # a numeric string against a number: StringToNumber, then numbers
        q['%s_nstr_26' % op] = (['-f', '{"%s":["nstr",26]}' % op, '-b',
                                 'nstr,'], None, None, None)
        for i, c in enumerate(SWEEP_STR_CONSTS):
            q['%s_str_%d' % (op, i)] = (
                ['-f', json.dumps({op: ['str', c]}), '-b', 'str,'], None,
                'filter', (op, 'str', c))
    return q


def sweep_f_decided(records, argv):
    """How many records the F path decides itself for a sweep query: all but
    those with an escaped string where the query reads str, and those whose
    num is a discrete key but not a plain integer of at most 15 digits (its
    key is Number::toString)."""
    reads_str = any('str' in a.replace('nstr', '') for a in argv)
    num_key = 'num,' in argv
    n = 0
    for r in records:
        if reads_str and r['str_esc']:
            continue
        if num_key and not _simple_int(r['num']):
            continue
        n += 1
    return n


def _simple_int(t):
    d = t[1:] if t.startswith('-') else t
    return d.isdigit() and len(d) <= 15 and t != '-0'


# the second reference: from the generated values, with Python's own binary64
# (float() is correctly rounded), frexp, floor, a civil-calendar day count and
# UTF-16 code unit order -- not the oracle's code

def _days(y, m, d):
    """Days from 1970-01-01 to y-m-d (proleptic Gregorian, any d >= 1 carries
    into the next months)."""
    def before_year(y):     # days from 0000-01-01 to y-01-01, y >= 0
        return 365 * y + (y + 3) // 4 - (y + 99) // 100 + (y + 399) // 400
    leap = y % 4 == 0 and (y % 100 != 0 or y % 400 == 0)
    mdays = [31, 29 if leap else 28, 31, 30, 31, 30, 31, 31, 30, 31, 30, 31]
    return before_year(y) + sum(mdays[:m - 1]) + d - 1 - before_year(1970)


def _date_ms(p):
    y, mo, d, h, mi, s, ms, off = p
    return _days(y, mo, d) * 86400000 + ((h * 60 + mi) * 60 + s) * 1000 + \
        ms - off * 60000


def _js_string(x):
    """Number::toString (ECMA-262 7.1.12.1) from repr's shortest digits."""
    if x != x:
        return 'NaN'
    if x == 0:
        return '0'
    if x < 0:
        return '-' + _js_string(-x)
    if math.isinf(x):
        return 'Infinity'
    t = decimal.Decimal(repr(x)).normalize().as_tuple()
    ds = ''.join(map(str, t.digits))
    k, n = len(ds), t.exponent + len(ds)
    if k <= n <= 21:
        return ds + '0' * (n - k)
    if 0 < n <= 21:
        return ds[:n] + '.' + ds[n:]
    if -6 < n <= 0:
        return '0.' + '0' * -n + ds
    e = '%s%d' % ('+' if n > 0 else '-', abs(n - 1))
    return ds[0] + ('.' + ds[1:] if k > 1 else '') + 'e' + e


def _str_value(r):
    return json.loads('"%s"' % r['str'])


def _ordinal_min(kind, x, step=None):
    if kind == 'p2':
        if x < 1:
            return 0.0
        if math.isinf(x):
            return x
        return math.ldexp(1.0, math.frexp(x)[1] - 1)
    q = x / step
    if math.isinf(q):
        return q * step
    return (math.floor(q) + 0.0) * step


def _compare(op, a, b):
    return {'eq': a == b, 'ne': a != b, 'lt': a < b, 'le': a <= b,
            'gt': a > b, 'ge': a >= b}[op]


def sweep_reference(records, kind, arg):
    """{key: count} a sweep query must give (keys as sweep_points makes
    them), or for lquantize with step 0 the sorted counts of its NaN
    buckets."""
    out = {}

    def bump(k):
        out[k] = out.get(k, 0) + 1
    for r in records:
        if kind == 'discrete':
            bump(_js_string(float(r['num'])).encode())
        elif kind == 'p2':
            bump(_ordinal_min('p2', float(r['num'])))
        elif kind == 'linear':
            x = float(r['num'])
            if arg == 0:
                bump('+inf' if x > 0 else '-inf' if x < 0 else 'nan')
            else:
                bump(_ordinal_min('linear', x, arg))
        elif kind == 'date':
            if r['date'] is not None:
                sec = _date_ms(r['date']) // 1000
                bump((sec // arg) * arg + 0.0)
        elif kind == 'filter':
            op, field, c = arg
            if field == 'num':
                x, y = float(r['num']), float(c)
                key = r['nstr'].encode()
            else:
                s = _str_value(r)
                x, y = s.encode('utf-16-be'), c.encode('utf-16-be')
                key = s.encode()
            if _compare(op, x, y):
                bump(key)
    if kind == 'linear' and arg == 0:
        return sorted(out.values())
    return out


def sweep_points(points, kind, arg):
    """A scan's points in sweep_reference's form."""
    d = {}
    for fields, v in points:
        x = fields[0][1]
        k = x if isinstance(x, bytes) else ('nan' if x != x else x + 0.0)
        d[k] = d.get(k, 0) + v
    if kind == 'linear' and arg == 0:
        assert set(d) <= {'nan'} and len(points) <= 3, points
        return sorted(v for _, v in points)
    return d


# ---------------------------------------------------------------------------
# krill filters: records whose `v` takes every value form a JSON field can
# have, the constants a filter compares it with, seeded predicate trees, and a
# second reference for them written from ECMA-262 (not the oracle's code)
# ---------------------------------------------------------------------------

MISSING = object()      # a field the record does not have

# (tag, JSON text, value as krill_reference sees it) of every form `v` takes;
# numbers are floats, strings str, containers dict / list
V_FORMS = [
    ('missing', None, MISSING),
    ('null', 'null', None), ('true', 'true', True), ('false', 'false', False),
    ('zero', '0', 0.0), ('negzero', '-0', -0.0), ('int', None, None),
    ('tenth', '0.1', 0.1), ('e21', '1e21', 1e21),
    ('two53p1', '9007199254740993', float(TWO53)),
    ('s_empty', '""', ''), ('s_0', '"0"', '0'), ('s_26', '"26"', '26'),
    ('s_sp26', '" 26 "', ' 26 '), ('s_hex', '"0x1a"', '0x1a'),
    ('s_abc', '"abc"', 'abc'), ('s_get', '"GET"', 'GET'),
    ('s_kana', '"ｶﾀ"', 'ｶﾀ'),
    ('s_emoji', '"\U0001f600"', '\U0001f600'),
    ('s_quote', '"x\\"y"', 'x"y'), ('s_escA', '"\\u0041"', 'A'),
    ('obj', '{}', {}), ('arr', '[1,2]', [1.0, 2.0]), ('arr0', '[]', []),
]
V_INTS = [1, 2, 25, 26, 27, -1, 100]

# the constants of the filters: numbers around the forms above, strings
# equal to some of them, a prefix of none, and the two booleans
KRILL_CONSTS = [0, -0.0, 1, 26, 0.1, TWO53, 1e21, '', '0', '26', ' 26 ',
                '0x1a', 'abc', 'GET', 'x"y', 'A', 'ｶﾀ', True, False]

S_VALUES = ['GET', 'GEX', 'G', 'GF', 'GETS', 'GETSA', 'GETSAB', 'GETSABC',
            'GETSABCD', 'PUT', 'abc', '26', '', ' 26 ', '0x1a']
OPT_VALUES = [('0', 0.0), ('26', 26.0), ('"26"', '26'), ('"abc"', 'abc'),
              ('true', True), ('null', None)]

# field orders of the four record shapes; only shapes 0 and 2 have `opt`,
# shape 3 has a literal key "a.b" (pluck reads it before a.b)
_FILTER_SHAPES = [
    ['tag', 'v', 'n', 's', 'b', 'opt', 'a', 't', 'pad'],
    ['t', 'tag', 'a', 'n', 'v', 's', 'b', 'pad'],
    ['tag', 's', 'v', 'opt', 'b', 'n', 't', 'a', 'pad'],
    ['tag', 'a.b', 'v', 'n', 'a', 's', 'b', 't', 'pad'],
]
FILTER_DAY_MS = 1398902400000       # 2014-05-01T00:00:00.000Z


def filter_records(seed, n):
    """n records as dicts: tag, v_text/v (the form of `v`), n, s, b, opt
    (MISSING in shapes 1 and 3), ab (what pluck(rec, "a.b") gives), t_ms,
    shape, len (the line's length in bytes) and damage (None, 'cut' or a
    junk suffix)."""
    rng = random.Random(seed)
    out = []
    for _ in range(n):
        tag, text, val = rng.choice(V_FORMS)
        if tag == 'int':
            k = rng.choice(V_INTS)
            text, val = str(k), float(k)
        shape = rng.randrange(4)
        nv = rng.choice([rng.randint(-5, 300), 26, 0])
        ot, ov = rng.choice(OPT_VALUES)
        ab = rng.randint(0, 40)
        r = rng.random()
        damage = 'cut' if r < 0.005 else \
            rng.choice(['x', ',', '}', ' 1', '{}']) if r < 0.01 else None
        out.append({'tag': tag, 'v_text': text, 'v': val,
                    'n': float(nv), 'n_text': str(nv),
                    's': rng.choice(S_VALUES), 'b': rng.random() < 0.5,
                    'opt_text': ot if shape in (0, 2) else None,
                    'opt': ov if shape in (0, 2) else MISSING,
                    'ab': float(ab), 'ab2': ab + 1,
                    't_ms': FILTER_DAY_MS + rng.randrange(86400000),
                    'shape': shape, 'len': rng.randint(120, 215),
                    'damage': damage})
    return out


def _iso_z(ms):
    s, ms = divmod(ms - FILTER_DAY_MS, 1000)
    return '2014-05-01T%02d:%02d:%02d.%03dZ' % (s // 3600, s // 60 % 60,
                                                 s % 60, ms)


def filter_line(rec):
    def render(pad):
        parts = []
        for f in _FILTER_SHAPES[rec['shape']]:
            if f == 'tag':
                parts.append('"tag":"%s"' % rec['tag'])
            elif f == 'v' and rec['v'] is not MISSING:
                parts.append('"v":' + rec['v_text'])
            elif f == 'n':
                parts.append('"n":' + rec['n_text'])
            elif f == 's':
                parts.append('"s":' + json.dumps(rec['s']))
            elif f == 'b':
                parts.append('"b":' + ('true' if rec['b'] else 'false'))
            elif f == 'opt' and rec['opt'] is not MISSING:
                parts.append('"opt":' + rec['opt_text'])
            elif f == 'a':
                parts.append('"a":{"b":%d}' % (rec['ab2'] if rec['shape'] == 3
                                               else int(rec['ab'])))
            elif f == 'a.b':
                parts.append('"a.b":%d' % int(rec['ab']))
            elif f == 't':
                parts.append('"t":"%s"' % _iso_z(rec['t_ms']))
            elif f == 'pad':
                parts.append('"pad":"%s"' % pad)
        return ('{' + ','.join(parts) + '}').encode('utf-8')
    line = render('')
    line = render('p' * max(8, rec['len'] - len(line)))
    if rec['damage'] == 'cut':          # after every field a filter reads
        return line[:-4]
    if rec['damage']:
        return line + rec['damage'].encode()
    return line


def filter_lines(seed, n):
    return [filter_line(r) for r in filter_records(seed, n)]


FILTER_FIELDS = ['v', 'v', 'v', 'n', 's', 'b', 'opt', 'a.b', 'nope']
OPS = ['eq', 'ne', 'lt', 'le', 'gt', 'ge']


def random_predicate(rng, nleaves, fields=FILTER_FIELDS, depth=0):
    """A krill tree of `nleaves` leaves (counting each `{}` child, which
    compiles to a leaf too): and/or nodes of 1-5 children nested at most 5
    deep, leaves of every operator over `fields` with constants of
    KRILL_CONSTS."""
    if nleaves == 1:
        if depth and rng.random() < 0.08:
            return {}
        return {rng.choice(OPS): [rng.choice(fields),
                                  rng.choice(KRILL_CONSTS)]}
    cap = 5 ** (4 - depth)          # leaves a child at depth + 1 can hold
    lo = max(1, -(-nleaves // cap))
    k = rng.randint(lo, max(lo, min(5, nleaves)))
    # nleaves split into k parts, each 1..cap
    parts = [1] * k
    for _ in range(nleaves - k):
        i = rng.choice([j for j in range(k) if parts[j] < cap])
        parts[i] += 1
    return {rng.choice(['and', 'or']): [
        random_predicate(rng, p, fields, depth + 1) for p in parts]}


def predicate_leaves(pred):
    """Leaves the plan compiler emits for pred ({} children count)."""
    if not pred:
        return 1
    key = next(iter(pred))
    if key in ('and', 'or'):
        return sum(predicate_leaves(p) for p in pred[key])
    return 1


# --- the second reference: ECMA-262 7.2.13 / 7.2.14 on the values above ---

# WhiteSpace and LineTerminator (ECMA-262 12.2, 12.3)
_JS_WS = ('\t\n\v\f\r \u00a0\u1680\u2000\u2001\u2002\u2003\u2004'
          '\u2005\u2006\u2007\u2008\u2009\u200a\u2028\u2029\u202f'
          '\u205f\u3000\ufeff')


class FieldMissing(Exception):
    pass


def _js_type(x):
    if x is None:
        return 'null'
    if isinstance(x, bool):
        return 'boolean'
    if isinstance(x, float):
        return 'number'
    if isinstance(x, str):
        return 'string'
    return 'object'


def _string_to_number(s):
    """StringToNumber (ECMA-262 7.1.4.1.1)."""
    s = s.strip(_JS_WS)
    if s == '':
        return 0.0
    for pre, base, digits in (('0x', 16, '0123456789abcdef'),
                              ('0o', 8, '01234567'), ('0b', 2, '01')):
        if s[:2].lower() == pre:
            body = s[2:]
            if body and all(c in digits for c in body.lower()):
                return float(int(body, base))
            return math.nan
    sign, body = 1.0, s
    if body[:1] in '+-':
        sign, body = (-1.0 if body[0] == '-' else 1.0), body[1:]
    if body == 'Infinity':
        return sign * math.inf
    mant, _, exp = body.partition('e') if 'e' in body else \
        body.partition('E')
    if exp[:1] in '+-':
        exp = exp[1:]
    if ('e' in body or 'E' in body) and not (exp and exp.isdigit()):
        return math.nan
    ip, dot, fp = mant.partition('.')
    if not (ip or fp) or not all(c.isdigit() and c.isascii()
                                 for c in ip + fp):
        return math.nan
    return sign * float(body)


def _to_primitive(x):
    """ToPrimitive(x, hint number) of a JSON value: objects give
    "[object Object]", arrays Array.prototype.join."""
    if isinstance(x, dict):
        return '[object Object]'
    if isinstance(x, list):
        return ','.join('' if e is None else _to_string(e) for e in x)
    return x


def _to_string(x):
    if isinstance(x, float):
        return _js_string(x)
    if isinstance(x, bool):
        return 'true' if x else 'false'
    if x is None:
        return 'null'
    if isinstance(x, str):
        return x
    return _to_primitive(x)


def _to_number(x):
    x = _to_primitive(x)
    if x is None:
        return 0.0
    if isinstance(x, bool):
        return 1.0 if x else 0.0
    if isinstance(x, str):
        return _string_to_number(x)
    return x


def loose_equals(x, y):
    """x == y (IsLooselyEqual, ECMA-262 7.2.14)."""
    tx, ty = _js_type(x), _js_type(y)
    if tx == ty:
        return x is y if tx == 'object' else x == y
    if 'null' in (tx, ty):
        return False            # (no undefined here: it raised before)
    if tx == 'number' and ty == 'string':
        return x == _string_to_number(y)
    if tx == 'string' and ty == 'number':
        return _string_to_number(x) == y
    if tx == 'boolean':
        return loose_equals(1.0 if x else 0.0, y)
    if ty == 'boolean':
        return loose_equals(x, 1.0 if y else 0.0)
    if tx == 'object':
        return loose_equals(_to_primitive(x), y)
    return False


def _less_than(x, y):
    """IsLessThan (ECMA-262 7.2.13): True, False or None (undefined)."""
    px, py = _to_primitive(x), _to_primitive(y)
    if isinstance(px, str) and isinstance(py, str):
        # UTF-16 code units: big-endian UTF-16 bytes order the same way
        return px.encode('utf-16-be') < py.encode('utf-16-be')
    nx, ny = _to_number(px), _to_number(py)
    if nx != nx or ny != ny:
        return None
    return nx < ny


def js_compare(op, x, y):
    if op == 'eq':
        return loose_equals(x, y)
    if op == 'ne':
        return not loose_equals(x, y)
    if op == 'lt':
        return _less_than(x, y) is True
    if op == 'gt':
        return _less_than(y, x) is True
    if op == 'le':
        return _less_than(y, x) is False
    return _less_than(x, y) is False


def _field(rec, name):
    v = {'v': rec['v'], 'n': rec['n'], 's': rec['s'], 'b': rec['b'],
         'opt': rec['opt'], 'a.b': rec['ab'], 'tag': rec['tag']}.get(
             name, MISSING)
    if v is MISSING:
        raise FieldMissing(name)
    return v


def krill_test(pred, rec):
    """krill's evaluation of pred on rec: left to right, short-circuit; a
    leaf on a field the record does not have raises FieldMissing."""
    if not pred:
        return True
    key = next(iter(pred))
    if key == 'and':
        return all(krill_test(p, rec) for p in pred[key])
    if key == 'or':
        return any(krill_test(p, rec) for p in pred[key])
    field, c = pred[key]
    if isinstance(c, int) and not isinstance(c, bool):
        c = float(c)
    return js_compare(key, _field(rec, field), c)


def krill_reference(records, pred, ds=None, bounds=None):
    """What `-f pred -b tag,` over records gives, with an optional
    datasource filter ds and time bounds (ge_ms, lt_ms) on t:
    ({tag: count}, {stage: (noutputs, nfilteredout, nfailedeval)})."""
    tally = {}
    stages = [(name, p) for name, p in (('Datasource filter', ds),
                                        ('User filter', pred)) if p]
    split = {name: [0, 0, 0] for name, _ in stages}
    if bounds:
        split['Time filter'] = [0, 0, 0]
    for r in records:
        if r['damage']:
            continue
        passed = True
        for name, p in stages:
            try:
                ok = krill_test(p, r)
            except FieldMissing:
                split[name][2] += 1
                passed = False
                break
            if not ok:
                split[name][1] += 1
                passed = False
                break
            split[name][0] += 1
        if passed and bounds:
            if not bounds[0] <= r['t_ms'] < bounds[1]:
                split['Time filter'][1] += 1
                passed = False
            else:
                split['Time filter'][0] += 1
        if passed:
            tally[r['tag'].encode()] = tally.get(r['tag'].encode(), 0) + 1
    return tally, {k: tuple(v) for k, v in split.items()}


def filter_split(counters, stage):
    """(noutputs, nfilteredout, nfailedeval) of a stage of a scan's
    counters."""
    c = counters.get(stage, {})
    return (c.get('noutputs', 0), c.get('nfilteredout', 0),
            c.get('nfailedeval', 0))


def tag_points(points):
    """{tag: count} of the points of a `-b tag,` scan."""
    out = {}
    for fields, v in points:
        out[fields[0][1]] = out.get(fields[0][1], 0) + v
    return out


# --- the queries of the filter tests ---

FILTER_AFTER, FILTER_BEFORE = '2014-05-01T06:00:00.000Z', \
    '2014-05-01T18:30:00.000Z'
FILTER_BOUNDS = (FILTER_DAY_MS + 6 * 3600000,
                 FILTER_DAY_MS + 18 * 3600000 + 1800000)
# sizes of the random trees: every size up to the plan's 48 leaves, most
# around the F path's 16
TREE_SIZES = [1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13] + \
    list(range(14, 19)) * 4 + [19, 20, 21, 22, 23, 24, 25, 26, 27, 28, 30,
                               32, 33, 35, 36, 38, 40, 42, 44, 45, 46, 47,
                               48]


def filter_queries():
    """name -> (argv, datasource properties, user predicate, datasource
    predicate, time bounds) of every filter query: the comparison matrix
    (op_<const>), the random trees (tree<i>_<leaves>: the odd ones read only
    v and opt, so that with tag they need three capture rows) and the
    combined programs (comb16, comb17: leaves of the datasource filter, the
    user filter and the two time-bound leaves together)."""
    q = {}
    for op in OPS:
        for c in KRILL_CONSTS:
            pred = {op: ['v', c]}
            q['%s_%s' % (op, json.dumps(c, ensure_ascii=False))] = (
                ['-f', json.dumps(pred), '-b', 'tag,'], None, pred, None,
                None)
    rng = random.Random(4242)
    for i, n in enumerate(TREE_SIZES):
        pred = random_predicate(rng, n, FILTER_FIELDS if i % 2 == 0 else
                                ('v', 'v', 'opt'))
        q['tree%02d_%d' % (i, n)] = (['-f', json.dumps(pred), '-b', 'tag,'],
                                     None, pred, None, None)
    for total in (16, 17):
        ds = random_predicate(rng, 6, ('v',))
        pred = random_predicate(rng, total - 8, ('v',))
        q['comb%d' % total] = (
            ['-f', json.dumps(pred), '-b', 'tag,', '--after', FILTER_AFTER,
             '--before', FILTER_BEFORE], {'filter': ds, 'timeField': 't'},
            pred, ds, FILTER_BOUNDS)
    return q


def filter_jit_names(names):
    """The filter queries a run-time compiled F kernel is built for (each
    distinct plan costs a link): one constant of each type per operator,
    the trees of 14-18 leaves and the combined programs."""
    return sorted(
        [n for n in names if n.split('_', 1)[0] in OPS and
         n.split('_', 1)[1] in ('26', '"26"', 'true')] +
        [n for n in names if n.startswith('tree') and
         14 <= int(n.rsplit('_', 1)[1]) <= 18] +
        [n for n in names if n.startswith('comb')])


def query_leaves(query):
    """Leaves of a filter query's whole plan."""
    _, _, pred, ds, bounds = query
    return (predicate_leaves(pred) if pred else 0) + \
        (predicate_leaves(ds) if ds else 0) + (2 if bounds else 0)


def _pred_fields(pred):
    if not pred:
        return set()
    key = next(iter(pred))
    if key in ('and', 'or'):
        return set().union(*(_pred_fields(p) for p in pred[key]))
    return {pred[key][0]}


def query_capture_rows(query):
    """Capture rows the F kernel needs for a filter query (fast.cpp
    fplan_build): one per distinct field, here the filters' fields, tag and
    the time field; its only column, tag, is not bucketized."""
    _, _, pred, ds, bounds = query
    return len(_pred_fields(pred) | _pred_fields(ds) | {'tag'} |
               ({'t'} if bounds else set()))


def _or_eq(fields_consts):
    return json.dumps({'or': [{'eq': [f, c]} for f, c in fields_consts]})


# the plan compiler's limits (plan.cpp), each as (argv at the limit, argv one
# past it, the DNG_ELIMIT message of the second)
_COMPONENTS_30 = ['a.b.c.d.e.f.g.h', 'a.b.c.d.e.f.g.i', 'a.b.c.d.e.f.g.j',
                  'a.b.c.x']          # + tag + v: 30 path components
PLAN_LIMITS = {
    'leaves_48': (
        ['-f', json.dumps(random_predicate(random.Random(48), 48, ('v',))),
         '-b', 'tag,'],
        ['-f', json.dumps(random_predicate(random.Random(48), 49, ('v',))),
         '-b', 'tag,'],
        'filter too large'),
    # the pool holds the string constants and the candidate key names ("s"
    # and "tag" here)
    'pool_2048': (
        ['-f', _or_eq([('s', 'x' * (2048 - 4))]), '-b', 'tag,'],
        ['-f', _or_eq([('s', 'x' * (2048 - 3))]), '-b', 'tag,'],
        'plan constant pool exhausted'),
    'fields_24': (
        ['-f', _or_eq([(f, 1) for f in ['v'] + ['f%02d' % i
                                                for i in range(22)]]),
         '-b', 'tag,'],
        ['-f', _or_eq([(f, 1) for f in ['v'] + ['f%02d' % i
                                                for i in range(23)]]),
         '-b', 'tag,'],
        'too many distinct fields'),
    'components_30': (
        ['-f', _or_eq([(f, 1) for f in ['v'] + _COMPONENTS_30]),
         '-b', 'tag,'],
        ['-f', _or_eq([(f, 1) for f in ['v'] + _COMPONENTS_30 +
                       ['a.b.c.d.y']]), '-b', 'tag,'],
        'too many distinct fields in one scan'),
    'levels_8': (
        ['-f', _or_eq([('v', 1), ('a.b.c.d.e.f.g.h', 1)]), '-b', 'tag,'],
        ['-f', _or_eq([('v', 1), ('a.b.c.d.e.f.g.h.i', 1)]), '-b', 'tag,'],
        'field "a.b.c.d.e.f.g.h.i" has too many dot-separated components'),
    'breakdowns_12': (
        ['-b', 'tag,n,s,b,v,opt,a.b,t,c1,c2,c3,c4,'],
        ['-b', 'tag,n,s,b,v,opt,a.b,t,c1,c2,c3,c4,c5,'],
        'too many breakdowns'),
}

# constants of 1-8 bytes beside values of `s` of the same length that share
# all but their last byte with them (G GF GET GETS GETSA GETSAB GETSABC
# GETSABCD), then long ones: 48 + 7 * 56 + 44 = 484 bytes padded to words
_F_SHORT = ['G', 'GE', 'GET', 'GETT', 'GETSA', 'GETSAC', 'GETSABC',
            'GETSABCE']
_F_LONG = ['%02d' % i + 'L' * 54 for i in range(7)]

# the F plan's limits (fast.cpp fplan_build), each as (argv at the limit,
# argv one past it)
F_LIMITS = {
    'leaves_16': (
        ['-f', json.dumps(random_predicate(random.Random(16), 16, ('v',))),
         '-b', 'tag,'],
        ['-f', json.dumps(random_predicate(random.Random(16), 17, ('v',))),
         '-b', 'tag,']),
    'pool_484': (
        ['-f', _or_eq([('s', c) for c in _F_SHORT + _F_LONG + ['y' * 44]]),
         '-b', 'tag,'],
        ['-f', _or_eq([('s', c) for c in _F_SHORT + _F_LONG + ['y' * 45]]),
         '-b', 'tag,']),
    'paths_8': (
        ['-f', _or_eq([(f, 26) for f in ('v', 'n', 's', 'b', 'opt', 'a.b',
                                         'nope')]), '-b', 'tag,'],
        ['-f', _or_eq([(f, 26) for f in ('v', 'n', 's', 'b', 'opt', 'a.b',
                                         'nope', 't')]), '-b', 'tag,']),
    'columns_6': (['-b', 'tag,n,s,b,opt,a.b'],
                  ['-b', 'tag,n,s,b,opt,a.b,v,']),
    'synthetic_2': (
        ['-b', 'd1[date,field=t,aggr=lquantize,step=3600],'
         'd2[date,field=t,aggr=lquantize,step=60]'],
        ['-b', 'd1[date,field=t,aggr=lquantize,step=3600],'
         'd2[date,field=t,aggr=lquantize,step=60],'
         'd3[date,field=t,aggr=lquantize,step=1]']),
}

# plans the key automaton (plan.cpp FastBuilder) cannot take
_LONG_KEYS = ['k' + chr(ord('a') + i) + 'z' * 26 for i in range(10)]
AUTOMATON_LIMITS = {
    # ten 28-byte keys: more than FAST_MAXSTATES (200) trie states
    'states': ['-f', _or_eq([('v', 26)] + [(k, 1) for k in _LONG_KEYS]),
               '-b', 'tag,'],
    # 13 field contexts (the root, a .. a.b.c.d.e.f.g, x .. x.y.z.w.q), more
    # than FAST_MAXCTX (12)
    'contexts': ['-f', _or_eq([('v', 26), ('a.b.c.d.e.f.g.h', 1),
                               ('x.y.z.w.q.r', 1)]), '-b', 'tag,'],
    # (no case for FAST_MAXKEYS (48): each path component adds one key name
    # and each context at most one more, so a plan of at most 30 components
    # and 12 contexts has at most 41 keys, and the key limit is never the
    # one a plan exceeds; DESIGN §4)
}
