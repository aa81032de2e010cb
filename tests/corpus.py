"""Input corpus shared by the CPU and GPU suites, and a plain-Python walker of Lizard streams.

The families are built to reach the edges of the format where a codec goes wrong: matches 65536 or more bytes back (the
24-bit-offset codewords and the LIZv1 parsers' far-candidate rule), literal runs and matches of exact lengths at every
boundary between the length-extension widths, Huffman-hostile literal alphabets, and periodic data whose periods straddle
the decoder's wide-copy threshold.  `walk` decodes streams without a Huffman stage and counts the codeword classes it
met, so the tests can prove that the corpus really reaches what it claims to."""
import random
from collections import Counter

import numpy as np

import lizard_b200 as lz

BS = lz.BLOCK_SIZE
MINMATCH = 4
MM_LONGOFF = 16                 # LIZv1: a 24-bit-offset match is at least this long
LAST_LONG_OFF = 31              # LIZv1 token 31: 24-bit offset, match length 47 + extension
MAX_16BIT_OFFSET = 1 << 16

# literal run / match lengths at the boundaries between the 0-, 1-, 3- and 4-byte extension forms
#   LZ4 codewords: token field 15, then one byte, 254 + LE16 from 15 + 254, 255 + LE24 from 15 + 65536
#   LIZv1 codewords: literals 7 / 7 + 254 / 7 + 65536, matches 15 / 15 + 254 / 15 + 65536
LZ4_LITERALS = (14, 15, 16, 268, 269, 270, 65550, 65551)
LZ4_MATCHES = tuple(MINMATCH + n for n in (14, 15, 16, 268, 269, 270, 65550, 65551))
LIZ_LITERALS = (6, 7, 8, 260, 261, 65542, 65543)
LIZ_MATCHES = (14, 15, 16, 268, 269, 65550, 65551)
# 24-bit-offset matches: shorter than MM_LONGOFF + MINMATCH (refused by the far-candidate rule), token 0-30 (16-46),
# token 31 with a zero / one-byte / 254 + LE16 extension (47, 48, 300, 301)
FAR_LENGTHS = (15, 16, 17, 19, 20, 46, 47, 48, 300, 301)
PERIODS = (8, 9, 15, 16, 17, 31, 32, 33, 64, 100, 255, 256, 257, 511, 512, 543, 544, 545, 600)


# ---------------------------------------------------------------------------------------------------------------------
# families kept from the first CPU suite (same seeds, same bytes)
# ---------------------------------------------------------------------------------------------------------------------
def far_match_input(seed=3, n=BS):
    """Matches 65536 or more bytes back, short and long: exercises the LIZv1 parsers' rule that a far candidate is only taken
    when the match is at least MM_LONGOFF + MINMATCH long (lizard_parser_fastbig.h:99,142; lizard_parser_pricefast.h:69) and
    the 24-bit-offset codewords."""
    rnd = random.Random(seed)
    head = bytes(rnd.randrange(256) for _ in range(70000))
    out = bytearray(head)
    while len(out) < n:
        k = rnd.choice([5, 8, 12, 17, 19, 20, 21, 24, 40, 100])
        at = rnd.randrange(0, 4000)                      # source near the start: offsets >= 65536
        out += head[at:at + k]
        out += bytes(rnd.randrange(256) for _ in range(rnd.randrange(1, 30)))
    return bytes(out[:n])


def inputs(seed, count):
    """Mixed sizes (0 to 200000 bytes) and kinds: datagen, zeros, uniform random, 4-letter alphabet, a repeated 8-byte
    pattern, a skewed 4-symbol alphabet, Dirichlet(0.05) bytes."""
    rnd = random.Random(seed)
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(count):
        kind = rnd.randrange(7)
        n = rnd.choice([0, 1, 5, 19, 20, 21, 22, 40, 100, 1000, 1025, 2000, 4096, 30000, 65536, 131071, 131072,
                        131073, 200000])
        if kind == 0:
            out.append(lz.datagen(n, rnd.choice([10, 30, 50, 70, 90, 100]), rnd.randrange(1000)))
        elif kind == 1:
            out.append(bytes(n))
        elif kind == 2:
            out.append(rng.integers(0, 256, n, dtype=np.uint8).tobytes())
        elif kind == 3:
            out.append(rng.integers(0, 4, n, dtype=np.uint8).tobytes())
        elif kind == 4:
            out.append((b"abcdefgh" * (n // 8 + 1))[:n])
        elif kind == 5:
            out.append(rng.choice(np.array([65, 66, 67, 200], dtype=np.uint8), size=n, p=[0.9, 0.05, 0.04, 0.01]).tobytes())
        else:
            p = rng.dirichlet(np.ones(256) * 0.05)
            out.append(rng.choice(256, size=n, p=p).astype(np.uint8).tobytes())
    return out


def skewed(rnd, n, nrare, tail):
    """Three common symbols (97 %) and `nrare` rare ones; the last `tail` share of the block is mostly rare symbols, so the
    Huffman codes of its literals are long (10/11 bits) where the stream ends."""
    common = [rnd.randrange(256) for _ in range(3)]
    rare = rnd.sample(range(256), nrare)
    out = bytearray()
    cut = int(n * (1 - tail))
    while len(out) < cut:
        out.append(rnd.choice(common) if rnd.random() < 0.97 else rnd.choice(rare))
    while len(out) < n:
        out.append(rnd.choice(rare) if rnd.random() < 0.9 else rnd.choice(common))
    return bytes(out)


# ---------------------------------------------------------------------------------------------------------------------
# new families
# ---------------------------------------------------------------------------------------------------------------------
def _random(rng, n):
    return rng.integers(0, 256, n, dtype=np.uint8).tobytes()


def far_unit(seed, n=BS, head=70000):
    """`head` fresh random bytes, then copies of FAR_LENGTHS bytes from the head, each at least 65536 bytes back, with and
    without literals before them.  Every copy takes its own part of the head, and the bytes around a copy differ from the
    bytes around its source, so each copy is one match of exactly its length (or literals, when the parser refuses it)."""
    rnd = random.Random(seed)
    rng = np.random.default_rng(seed)
    src = _random(rng, head)
    out = bytearray(src)
    cur = 1                                             # next unused byte of the head
    cont = None                                         # the byte that would continue the previous copy's match
    lengths = FAR_LENGTHS + ((2000, 65583, 65584) if n > 2 * head else ())     # 65583 = 47 + 65536: 4-byte extension
    while True:
        k = rnd.choice(lengths)
        gap = rnd.choice([0, 0, 1, 2, 5, 7, 8, 30])
        at = cur + 1
        if gap == 0:                                    # neither end may continue the previous copy
            while at + k < head and (src[at] == cont or src[at - 1] == out[-1]):
                at += 1
        if len(out) + gap + k + 64 > n or at + k + 1 > head:
            break
        assert len(out) + gap - at >= MAX_16BIT_OFFSET
        if gap:
            lit = bytearray(_random(rng, gap))
            while lit[0] == cont or lit[-1] == src[at - 1]:
                lit[0], lit[-1] = rnd.randrange(256), rnd.randrange(256)
            out += lit
        out += src[at:at + k]
        cont = src[at + k]
        cur = at + k + 1
    tail = bytearray(_random(rng, n - len(out)))
    if tail and tail[0] == cont:
        tail[0] ^= 0x5A
    return bytes(out + tail)


def far_units(seed=40):
    """Single-block units (128 KiB) and multi-inner-block units (1.5 and 3 MiB) whose copies reach more than 1 MiB back."""
    return [far_unit(seed, BS), far_unit(seed + 1, BS), far_unit(seed + 2, BS - 777),
            far_unit(seed + 3, 3 * (1 << 19), head=1100000), far_unit(seed + 4, 3 << 20, head=1200000)]


def threshold_unit(seed, literals, matches, n=BS, head=16384):
    """Fresh random literal runs and copied matches of exactly the given lengths, (literals, match) pairs taken in turn
    until the unit is full.  A match copies from inside its own literal run (off <= run; off < length makes the match
    periodic) or, behind runs shorter than 8 bytes and for the long matches, from an unused part of a random head.  The
    last literal and the byte behind the match differ from the bytes around the source, so a match cannot grow."""
    rnd = random.Random(seed)
    rng = np.random.default_rng(seed)
    out = bytearray(_random(rng, head))
    hcur = 1                                            # next unused byte of the head
    cont = None
    pairs = [(a, b) for a in literals for b in matches]
    rnd.shuffle(pairs)
    misses = 0
    for lit, ml in (pairs[i % len(pairs)] for i in range(1 << 30)):
        if misses > len(pairs):
            break
        pos = len(out) + lit
        if pos + ml + 64 > n:
            misses += 1
            continue
        if ml > 2000:
            off = rnd.choice([1000, 4096, 9999])
            if pos - off < hcur or len(out) != head:        # the only pair of its unit: the source is the head's end
                misses += 1
                continue
        elif lit >= 8:
            off = rnd.randrange(8, lit + 1)
        else:
            off = pos - hcur
            if off >= 60000 or hcur + ml + 1 > head:
                misses += 1
                continue
            hcur += ml + 2
        misses = 0
        run = bytearray(_random(rng, lit))
        if lit:
            while run[0] == cont or run[-1] == (out[pos - 1 - off] if pos - 1 - off < len(out) else run[pos - 1 - off - len(out)]):
                run[0], run[-1] = rnd.randrange(256), rnd.randrange(256)
        out += run
        for _ in range(ml):
            out.append(out[-off])
        cont = out[-off]
    tail = bytearray(_random(rng, n - len(out)))
    if tail and tail[0] == cont:
        tail[0] ^= 0x5A
    return bytes(out + tail)


def threshold_units(seed=50):
    """Per flavour: one block of the short boundaries, and blocks that hold one 64 KiB+ literal run or match followed by a
    copy, so that the block still compresses."""
    short = lambda xs: tuple(x for x in xs if x < 1000)
    long_ = lambda xs: tuple(x for x in xs if x > 60000)
    out = []
    for k, (lits, mls) in enumerate(((LZ4_LITERALS, LZ4_MATCHES), (LIZ_LITERALS, LIZ_MATCHES))):
        s = seed + 10 * k
        out.append(threshold_unit(s, short(lits), short(mls)))
        for j, ll in enumerate(long_(lits)):        # a 64 KiB+ run, then a long copy of part of it
            out.append(threshold_unit(s + 1 + j, (ll,), (40000,), head=0))
        for j, ml in enumerate(long_(mls)):         # a 64 KiB+ match (periodic) behind a short literal run
            out.append(threshold_unit(s + 5 + j, short(lits)[:1], (ml,)))
    return out


def hostile_units(seed=60):
    """Literal alphabets the Huffman stage finds hard: many rare symbols (code lengths at the 11-bit limit), a skewed
    block whose stream ends in rare symbols, one symbol (RLE streams) and two symbols (nearly incompressible literals or a
    stored stream)."""
    rnd = random.Random(seed)
    rng = np.random.default_rng(seed)
    p = np.concatenate([np.full(4, 0.24), rng.dirichlet(np.ones(252) * 0.3) * 0.04])
    rare = rng.choice(256, size=BS, p=p).astype(np.uint8).tobytes()
    dirichlet = rng.choice(256, size=BS - 5, p=rng.dirichlet(np.ones(256) * 0.02)).astype(np.uint8).tobytes()
    two = rng.choice(np.array([0x31, 0xC7], dtype=np.uint8), size=70000, p=[0.5, 0.5]).tobytes()
    two_skew = rng.choice(np.array([0x00, 0xFF], dtype=np.uint8), size=BS, p=[0.995, 0.005]).tobytes()
    return [rare, dirichlet, skewed(rnd, BS, 200, 0.1), bytes([0x41]) * BS, two, two_skew]


def periodic_units(seed=70, n=20000):
    """A random period of PERIODS bytes repeated, with a byte changed every few thousand bytes: long overlapping matches at
    offsets on both sides of the decoder's wide-copy threshold, and (LIZv1) repeat offsets after each change."""
    rng = np.random.default_rng(seed)
    out = []
    for p in PERIODS:
        base = bytearray((_random(rng, p) * (n // p + 1))[:n])
        for at in rng.integers(100, n, size=n // 3000):
            base[int(at)] ^= 0xA5
        out.append(bytes(base))
    return out


def corpus():
    """family -> list of units (about 6 MiB in all)."""
    return {"far": far_units(), "threshold": threshold_units(), "hostile": hostile_units(), "periodic": periodic_units()}


# ---------------------------------------------------------------------------------------------------------------------
# collide: inputs built against the lowestPrice map (csrc/encode_lp.cuh, LpMap)
# ---------------------------------------------------------------------------------------------------------------------
# The lowestPrice levels hash a position's 4 bytes (Lizard_hashPtr, searchLength 4: level 25/45) or 5 bytes (Lizard_hash5:
# 23/24/43/44) to a bucket of hashLog bits.  A unit of one inner block keeps (bucket, position) pairs in a map of 2^18
# slots whose home slot is the bucket's top 18 bits, probed linearly, so at hashLog 23 (24/25/44/45) 32 buckets share a
# home slot.  Both hashes are invertible (odd multipliers), so keys of any chosen bucket can be written down.
MAP_LOG = 18
HASH4_PRIME, HASH5_PRIME = 2654435761, 889523592379
_INV4, _INV5 = pow(HASH4_PRIME, -1, 1 << 32), pow(HASH5_PRIME, -1, 1 << 40)


def bucket(window: bytes, hash_log: int) -> int:
    """hc_hash of a 4-byte (searchLength 4) or 5-byte window."""
    if len(window) == 4:
        return (int.from_bytes(window, "little") * HASH4_PRIME % (1 << 32)) >> (32 - hash_log)
    return (int.from_bytes(window, "little") * HASH5_PRIME % (1 << 40)) >> (40 - hash_log)


def key(b: int, mls: int, rnd, hash_log=23) -> bytes:
    """`mls` bytes (4 or 5) whose bucket at `hash_log` is b; the low bits of the product are random."""
    bits = 32 if mls == 4 else 40
    low = bits - hash_log
    x = (b << low) | rnd.getrandbits(low)
    v = x * (_INV4 if mls == 4 else _INV5) % (1 << bits)
    return v.to_bytes(mls, "little")


def collide_unit(seed, mls, first, keys=2048, n=BS, background="random", repeat=False):
    """A unit of `n` bytes with `keys` planted keys of consecutive hashLog-23 buckets first, first + 1, ..., one at the start
    of each 8-byte record from n // 8 on.  The keys are inserted in bucket order, so each one probes past the slots of the
    keys before it that share or precede its home slot: long probe runs, and with `first` near 2^23 runs that wrap past the
    map's last slot.  repeat=True follows every record with a copy of an earlier record (key and 3 bytes), so the parser
    finds matches of 7 bytes through the runs."""
    rnd = random.Random(seed)
    rng = np.random.default_rng(seed)
    out = bytearray(_random(rng, n) if background == "random" else lz.datagen(n, 50, seed))
    step = 16 if repeat else 8
    at = max(0, min(n // 8, n - keys * step - 64))
    assert at + keys * step + 64 <= n
    recs = []
    for i in range(keys):
        r = key(first + i, mls, rnd) + bytes(rnd.getrandbits(8) for _ in range(8 - mls))
        out[at + step * i:at + step * i + 8] = r
        recs.append(r)
        if repeat:
            j = rnd.randrange(i + 1)
            out[at + step * i + 8:at + step * i + 16] = recs[j][:7] + bytes([recs[j][7] ^ 0x5A])
    return bytes(out[:n])


def race_unit(seed, mls, n=BS, pairs=48):
    """Pairs of new buckets that share a home slot and are inserted by one 32-position insert step, so that two lanes claim
    the same empty slot at once (on the device, one loses the atomic compare-and-swap and must go on probing).

    A literal-only parse inserts one position per step; only the positions behind a match are inserted many at a time, and
    of those only the last mls - 1 have windows that did not occur before.  So each pair is a 32-byte match ending at E whose
    last bytes and the two bytes behind it are chosen: the windows at E - mls + 1 and E - mls + 2 have the same home slot.
    Copies of each of the two windows alone appear later, each a match of exactly one window, found only if its position
    was inserted.  A map that drops the insert of the lane that lost the race changes the stream."""
    rnd = random.Random(seed)
    rng = np.random.default_rng(seed)
    hl, bits = 23, 8 * mls
    prime, mask = (HASH4_PRIME, 0xFFFFFFFF) if mls == 4 else (HASH5_PRIME, (1 << 40) - 1)
    found = []
    while len(found) < pairs:
        # w0 random; w1 = w0's last mls - 1 bytes + one byte t: all 256 t at once
        w0 = rng.integers(0, 1 << 62, 1 << 14, dtype=np.uint64) & np.uint64(mask)
        home0 = ((w0 * np.uint64(prime)) & np.uint64(mask)) >> np.uint64(bits - MAP_LOG)
        w1 = (w0[:, None] >> np.uint64(8)) | (np.arange(256, dtype=np.uint64)[None, :] << np.uint64(bits - 8))
        home1 = ((w1 * np.uint64(prime)) & np.uint64(mask)) >> np.uint64(bits - MAP_LOG)
        for r, t in zip(*np.nonzero(home1 == home0[:, None])):
            a, b = int(w0[r]).to_bytes(mls, "little"), int(w1[r, t]).to_bytes(mls, "little")
            if bucket(a, hl) != bucket(b, hl):
                found.append((a, b))
    found = found[:pairs]
    # zeros around 8-byte random guards: the block compresses well, so it is not stored raw and its parse shows in the output
    out = bytearray(n)
    src_at, copy_at, probe_at = 256, n // 3, 2 * n // 3
    spans = []
    for j in range(pairs):
        spans += [(src_at + 64 * j, 33), (copy_at + 64 * j, 34)]
        spans += [(probe_at + 64 * j + 24 * k, mls) for k in range(2)]
    for at, length in spans:
        out[at - 8:at + length + 8] = _random(rng, length + 16)
    for j, (a, b) in enumerate(found):
        body = bytes(_random(rng, 32 - (mls - 1))) + a[:mls - 1]       # the match: 32 bytes ending in w0's first mls - 1
        s = src_at + 64 * j
        out[s:s + 32] = body
        out[s + 32] = a[mls - 1] ^ 0x5A                                 # the source's match ends here
        c = copy_at + 64 * j
        out[c - 1] = out[s - 1] ^ 0x33                                  # ... and cannot grow backwards
        out[c:c + 32] = body
        out[c + 32:c + 34] = b[mls - 2:]                                # t0, t1
        e = c + 32                                                      # w0 at e - mls + 1, w1 at e - mls + 2
        for k, w in enumerate((a, b)):
            p = probe_at + 64 * j + 24 * k
            pos = e - mls + 1 + k
            out[p:p + mls] = w
            out[p - 1] = out[pos - 1] ^ 0x77
            out[p + mls] = out[pos + mls] ^ 0x77
    return bytes(out)


def collide_units(seed=80):
    """The `collide` family, for both key widths: a 2048-key cluster in the middle of the map on random background (a block
    the encoder stores raw), one straddling the map's end and one whose keys repeat, both on datagen background (their
    parse shows in the stream), and the insert-race units."""
    top = (1 << 23) - 2048                              # the last 2048 buckets: the runs of the last home slots wrap
    out = []
    for k, mls in enumerate((5, 4)):
        s = seed + 10 * k
        out.append(collide_unit(s, mls, 3 << 20))
        out.append(collide_unit(s + 1, mls, top, background="datagen"))
        out.append(collide_unit(s + 2, mls, top - 4096, background="datagen", repeat=True))
        out.append(race_unit(s + 3, mls))
    return out


def corpus_units():
    return [u for units in corpus().values() for u in units]


def edge_capacities(rnd, units, bound):
    """Destination capacities drawn like the GPU edge-input test: the bound twice, one byte short of the input, half of it
    plus one, anything from 1 to the bound."""
    return [rnd.choice([bound(len(u)), bound(len(u)), max(len(u) - 1, 1), len(u) // 2 + 1, rnd.randrange(1, bound(len(u)) + 1)])
            for u in units]


# ---------------------------------------------------------------------------------------------------------------------
# walker
# ---------------------------------------------------------------------------------------------------------------------
def _le(b, at, n):
    if at + n > len(b):
        raise ValueError("stream ends inside a field")
    return int.from_bytes(b[at:at + n], "little")


def is_lizv1(level):
    return 20 <= level <= 29 or 40 <= level <= 49


class _Stream:
    def __init__(self, data):
        self.b, self.p = data, 0

    def byte(self):
        if self.p >= len(self.b):
            raise ValueError("stream exhausted")
        self.p += 1
        return self.b[self.p - 1]

    def take(self, n):
        if self.p + n > len(self.b):
            raise ValueError("stream exhausted")
        self.p += n
        return self.b[self.p - n:self.p]

    def ext(self, classes, kind):
        """One length extension: a byte, 254 + LE16 or 255 + LE24 (lizard_decompress_lz4.h:48-64)."""
        v = self.byte()
        if v == 254:
            classes[kind + "_ext3"] += 1
            return _le(self.take(2), 0, 2)
        if v == 255:
            classes[kind + "_ext4"] += 1
            return _le(self.take(3), 0, 3)
        classes[kind + "_ext1"] += 1
        return v


def _copy(out, off, n):
    if off < 1 or off > len(out):
        raise ValueError("offset %d outside the output (%d bytes)" % (off, len(out)))
    if off >= n:
        out += out[len(out) - off:len(out) - off + n]
    else:                                               # overlapping: the last `off` bytes repeat
        out += (out[-off:] * (n // off + 1))[:n]


def max_dist(level):
    """The farthest offset a level's parser takes: 2^windowLog - 1 (64 KiB - 1 for the LZ4 codewords, 4 MiB - 1 for LIZv1
    below level 29, whose window is 16 MiB)."""
    if not is_lizv1(level):
        return (1 << 16) - 1
    return (1 << 24) - 1 if level in (29, 49) else (1 << 22) - 1


class _DictCopy:
    """Counts where a match's source lies when the output starts with a dictionary of `base` bytes."""

    def __init__(self, out, classes, base, level):
        self.out, self.classes, self.base, self.edge = out, classes, base, max_dist(level)

    def __call__(self, off, n, kind):
        src = len(self.out) - off
        if self.base and 0 <= src < self.base:
            kind_in = "dict_match" if src + n <= self.base else "dict_straddle"
            self.classes[kind_in] += 1
            self.classes[(kind_in, n)] += 1
            if off == self.edge:
                self.classes["dict_edge"] += 1
            if kind:
                self.classes["dict_" + kind] += 1
        _copy(self.out, off, n)


def walk(comp, rep_short_at=None, dictionary=b""):
    """Decode a Lizard stream whose inner blocks carry no Huffman-coded stream (levels 10-29, or blocks of the higher levels
    the encoder stored plain), following Lizard_decompress_generic (lib/lizard_decompress.c:115-264; streams as read by
    Lizard_readStream, :72-112).  Returns (decoded bytes, Counter of codeword classes):
      lit_ext0/1/3/4, match_ext0/1/3/4   width in bytes of a length's extension (0: the length fits the token)
      off16, off24, off_repeat           how a match's offset was coded
      far_short, far_long                LIZv1 24-bit-offset tokens 0-30 and 31
      far_after_literals                 a far token behind a literal-only token (literals before a far match)
      rep_short                          a repeat-offset match of 2-3 bytes (LIZv1)
      raw_block, block                   stored and coded inner blocks
      ("lit", n), ("match", n), ("far", n)   lengths of literal runs, of 16-bit/repeat matches and of far matches.
    With a `dictionary` (a stream of Lizard_loadDict + Lizard_compress_continue) the output starts as the dictionary, matches
    may reach into it, and the dictionary is stripped from the result.  Matches whose source starts in it also count as
      dict_match, dict_straddle          the source lies wholly in the dictionary / runs on into the unit (also counted
                                         by length: ("dict_match", n), ("dict_straddle", n))
      dict_edge                          ... at offset max_dist(level), the farthest the window reaches
      dict_far, dict_repeat              ... coded with a 24-bit offset / as a repeat offset (LIZv1).
    If `rep_short_at` is a list, the unit offset of every rep_short match is appended to it.
    Raises ValueError on a stream the reference would refuse (as far as a valid-stream walker needs to tell)."""
    if not comp:
        raise ValueError("empty input")
    level = comp[0]
    if not 10 <= level <= 49:
        raise ValueError("level %d" % level)
    lizv1 = is_lizv1(level)
    out = bytearray(dictionary)
    classes = Counter()
    copy = _DictCopy(out, classes, len(dictionary), level)
    ip = 1
    while ip < len(comp):
        flag = comp[ip]
        ip += 1
        if flag == 0x80:
            n = _le(comp, ip, 3)
            ip += 3
            if ip + n > len(comp):
                raise ValueError("raw block past the end")
            out += comp[ip:ip + n]
            ip += n
            classes["raw_block"] += 1
            continue
        if flag & 16:
            raise ValueError("flag 0x%x" % flag)
        if flag & 15:
            raise NotImplementedError("Huffman-coded stream (flag 0x%x)" % flag)
        streams = []
        for _ in range(5):                              # lengths (unused by the decoder), off16, off24, flags, literals
            n = _le(comp, ip, 3)
            if ip + 3 + n > len(comp):
                raise ValueError("stream past the end")
            streams.append(comp[ip + 3:ip + 3 + n])
            ip += 3 + n
        classes["block"] += 1
        _, off16, off24, flags, lits = (_Stream(s) for s in streams)
        if lizv1:
            _block_liz(out, flags, lits, off16, off24, classes, rep_short_at, copy)
        else:
            _block_lz4(out, flags, lits, off16, off24, classes, copy)
        if lits.p != len(lits.b):                       # last literals: the rest of the stream
            n = len(lits.b) - lits.p
            out += lits.take(n)
    return bytes(out[len(dictionary):]), classes


def _block_lz4(out, flags, lits, off16, off24, classes, copy):
    while flags.p < len(flags.b):
        token = flags.byte()
        n = token & 15
        if n == 15:
            n = 15 + lits.ext(classes, "lit")
        else:
            classes["lit_ext0"] += 1
        classes[("lit", n)] += 1
        out += lits.take(n)
        off = _le(lits.take(2), 0, 2)
        classes["off16"] += 1
        ml = token >> 4
        if ml == 15:
            ml = 15 + lits.ext(classes, "match")
        else:
            classes["match_ext0"] += 1
        ml += MINMATCH
        classes[("match", ml)] += 1
        copy(off, ml, None)


def _block_liz(out, flags, lits, off16, off24, classes, rep_short_at, copy):
    last_off = 0                                        # LIZARD_INIT_LAST_OFFSET, per inner block
    lit_only = False
    while flags.p < len(flags.b):
        token = flags.byte()
        if token >= 32:
            n = token & 7
            if n == 7:
                n = 7 + lits.ext(classes, "lit")
            else:
                classes["lit_ext0"] += 1
            classes[("lit", n)] += 1
            out += lits.take(n)
            if token >> 7:
                if (token >> 3) & 15:
                    classes["off_repeat"] += 1
            else:
                last_off = _le(off16.take(2), 0, 2)
                classes["off16"] += 1
            ml = (token >> 3) & 15
            if ml == 15:
                ml = 15 + lits.ext(classes, "match")
            else:
                classes["match_ext0"] += 1
            lit_only = ml == 0
            if ml and token >> 7 and ml < MINMATCH:       # only lowestPrice writes these: a 2-3 byte repeat-offset match
                classes["rep_short"] += 1
                if rep_short_at is not None:
                    rep_short_at.append(len(out) - copy.base)
            if ml:
                classes[("match", ml)] += 1
                copy(last_off, ml, "repeat" if token >> 7 else None)
            continue
        if token < LAST_LONG_OFF:
            ml = token + MM_LONGOFF
            classes["far_short"] += 1
        else:
            ml = lits.ext(classes, "match") + LAST_LONG_OFF + MM_LONGOFF
            classes["far_long"] += 1
        if lit_only:
            classes["far_after_literals"] += 1
        lit_only = False
        last_off = _le(off24.take(3), 0, 3)
        classes["off24"] += 1
        classes[("far", ml)] += 1
        copy(last_off, ml, "far")


# ---------------------------------------------------------------------------------------------------------------------
# what the corpus must reach
# ---------------------------------------------------------------------------------------------------------------------
ENCODE_LEVELS = [10, 11, 13, 14, 15, 16, 17, 20, 21, 22, 30, 31, 34, 35, 36, 37, 38, 40, 41, 42]     # implemented on the GPU
WALKED_ENCODE_LEVELS = [lv for lv in ENCODE_LEVELS if lv < 30]                                     # no Huffman stage
# lowestPrice, in a kernel of its own that has one launch shape (LIZARDB200_ENC_SHAPE does not apply)
LP_ENCODE_LEVELS = [23, 24, 25, 43, 44, 45]
LP_WALKED_LEVELS = [23, 24, 25]


def lp_corpus():
    """family -> units for the lowestPrice levels: the shared corpus and `collide`."""
    return dict(corpus(), collide=collide_units())


def lp_targets():
    """Codeword classes the lowestPrice streams of lp_corpus() must contain, summed over its families and LP_WALKED_LEVELS:
    short repeat matches, 24-bit offsets of both token forms, and every extension width of literal runs and matches."""
    return ({"rep_short", "off_repeat", "off16", "off24", "far_short", "far_long", "far_after_literals", "raw_block"}
            | {k + "_ext" + w for k in ("lit", "match") for w in "0134"})


def targets(family, lizv1):
    """Codeword classes (walk's names) that a family's streams must contain, summed over the walked encode levels of one
    codeword flavour."""
    if family == "threshold":
        lits, mls = (LIZ_LITERALS, LIZ_MATCHES) if lizv1 else (LZ4_LITERALS, LZ4_MATCHES)
        return ({k + "_ext" + w for k in ("lit", "match") for w in "0134"} | {"off16"}
                | {("lit", n) for n in lits} | {("match", n) for n in mls})
    if family == "far":
        if not lizv1:                                   # 64 KiB window: the far copies stay literals, the heads raw blocks
            return {"raw_block"}
        return ({"raw_block", "off24", "off_repeat", "far_short", "far_long", "far_after_literals", "match_ext1", "match_ext3",
                 "match_ext4"} | {("far", n) for n in (20, 46, 47, 48, 300, 301, 65583, 65584)})
    if family == "periodic":
        return {"off16", "match_ext3"} | ({"off_repeat"} if lizv1 else set())
    if family == "hostile":
        return {"off16", "match_ext4"}
    raise KeyError(family)


def missing(family, lizv1, classes):
    """The targets of a family that `classes` lacks, by name."""
    return sorted((t for t in targets(family, lizv1) if classes[t] == 0), key=str)


# ---------------------------------------------------------------------------------------------------------------------
# dictionaries: inputs for Lizard_loadDict + Lizard_compress_continue (hashChain 13-17 / 34-38, priceFast 21, 22, 41, 42)
# ---------------------------------------------------------------------------------------------------------------------
DICT_ENCODE_LEVELS = [13, 14, 15, 16, 17, 21, 22, 34, 35, 36, 37, 38, 41, 42]
DICT_WALKED_LEVELS = [lv for lv in DICT_ENCODE_LEVELS if lv < 30]
HC_WINDOW, PF_WINDOW = (1 << 16) - 1, (1 << 22) - 1          # max_dist of hashChain and of priceFast


class DictCase:
    """One unit and its dictionary.  prefix: the dictionary lies directly in front of the unit (otherwise it is external).
    before_dict / after_dict / before_unit: bytes a layout must put right around the dictionary and the unit (empty: any
    filler).  A poisoned case chooses them so that reading past the dictionary's end or extending a match below the start of
    the dictionary or of the unit finds a longer match than the reference does.
    expect: per codeword flavour ("lz4", "lizv1"), the walk classes (with their least counts) that the case's streams must
    hold, summed over the DICT_WALKED_LEVELS of that flavour (dict_missing)."""

    def __init__(self, family, dictionary, unit, prefix, before_dict=b"", after_dict=b"", before_unit=b"", lz4=(), lizv1=()):
        self.family, self.dictionary, self.unit, self.prefix = family, dictionary, unit, prefix
        self.before_dict, self.after_dict, self.before_unit = before_dict, after_dict, before_unit
        self.expect = {"lz4": Counter(dict(lz4)), "lizv1": Counter(dict(lizv1))}

    def __repr__(self):
        return "DictCase(%s, dict %d, unit %d, %s)" % (self.family, len(self.dictionary), len(self.unit),
                                                       "prefix" if self.prefix else "external")


def _fresh(rng, n, avoid=None):
    """n random bytes whose first byte differs from `avoid` (so a match in front of them cannot grow into them)."""
    b = bytearray(_random(rng, n))
    if n and avoid is not None and b[0] == avoid:
        b[0] ^= 0x5A
    return bytes(b)


def _nonzero(rng, n):
    """n random bytes, none of them 0: pieces that a match cannot grow into the zero filler around them."""
    return rng.integers(1, 256, n, dtype=np.uint8).tobytes()


def _far_cases(rng, window):
    """A dictionary of window + 64 bytes, random in its first 8 KiB and zero behind them (so no later position takes the
    random positions' buckets), and units holding 64-byte pieces of it at offsets window - 1, window and window + 1 (the
    last out of reach) from where they are copied, each between 24 fresh bytes (so the block compresses)."""
    d = _random(rng, 8192) + bytes(window + 64 - 8192)
    out = []
    for prefix in (False, True):
        u = bytearray(_random(rng, 200))
        for k in range(8):
            for off in (window - 1, window, window + 1):
                p = len(u)
                q = len(d) + p - off                    # the piece's place in the dictionary
                piece = d[q:q + 64]
                if u[-1] == d[q - 1]:
                    u[-1] ^= 0x77
                u += piece
                u += _fresh(rng, 24, d[q + 64])
        if window == HC_WINDOW:                         # LIZv1 codes the pieces at 65536 - 1 and 65536 with 16 / 24 bits
            expect = dict(lz4={"dict_match": 16, "dict_edge": 8}, lizv1={"dict_match": 24, "dict_far": 8})
        else:                                           # out of the LZ4 window
            expect = dict(lizv1={"dict_match": 16, "dict_far": 16, "dict_edge": 8})
        out.append(DictCase("far", d, bytes(u), prefix, **expect))
    return out


def _straddle_cases(rng):
    """One match per unit that starts k bytes before the dictionary's end and runs L - k bytes into the unit: the unit
    begins with those L - k bytes, zeros follow, then the copy, then 1000 zeros (so the block gains the 512 bytes
    Lizard_writeBlock asks of a coded block, lib/lizard_compress.c:228, and the copy is exactly one
    match of L bytes; the dictionary and the copied bytes hold no zero).
      * every match length of the codeword thresholds below 64 KiB (LZ4_MATCHES, LIZ_MATCHES, the LZ4 token's 15 and 19),
        300 bytes behind the unit's start: a 16-bit offset in both flavours;
      * FAR_LENGTHS, 66000 bytes behind it: a 24-bit offset, which LIZv1 takes from 20 bytes on (MM_LONGOFF + MINMATCH);
        the shorter ones must stay literals;
      * LIZ_MATCHES' 65550 and 65551, nearly all in the dictionary, more than 64 KiB back: LIZv1 only.
    The LZ4 lengths of 64 KiB and more cannot straddle: such a match would reach further back than the 64 KiB window."""
    d = _nonzero(rng, 70000)
    near = sorted(L for L in set(LZ4_MATCHES + LIZ_MATCHES + (15, 19)) if L < 60000)
    jobs = [(L, 300, "both") for L in near] + [(L, 66000, "lizv1" if L >= MM_LONGOFF + MINMATCH else "none")
                                                for L in FAR_LENGTHS] + [(L, 100, "lizv1") for L in (65550, 65551)]
    out = []
    for j, (L, gap, flavours) in enumerate(jobs):
        k = L - 40 if L > 60000 else (8, 12, 9, 33)[j % 4] if L > 33 else 8
        head = _nonzero(rng, L - k + 1)                 # the match runs over head[:L - k]; head[L - k] ends the source
        u = head + bytes(gap) + d[-k:] + head[:L - k] + bytes(1000)
        want = {("dict_straddle", L): 1}
        expect = {"both": dict(lz4=want, lizv1=want), "lizv1": dict(lizv1=want), "none": {}}[flavours]
        out.append(DictCase("straddle", d, u, j % 2 == 1, **expect))
    return out


def _periodic_cases(rng):
    """Dictionaries that repeat a period of 1-8, 16 or 33 bytes (same-bucket runs inside one 32-position load step), with a
    changed byte now and then, and units made of pieces of them and fresh bytes."""
    out = []
    for i, p in enumerate((1, 2, 3, 4, 5, 6, 7, 8, 16, 33)):
        base = bytearray((_random(rng, p) * (6000 // p + 1))[:6000])
        for at in rng.integers(100, len(base), size=3):
            base[int(at)] ^= 0xA5
        d = _random(rng, 700) + bytes(base) + _random(rng, 300)
        u = d[900:2500] + _random(rng, 500) + d[-400:] + bytes(base[:300]) + _random(rng, 100)
        out.append(DictCase("periodic", d, u, i % 2 == 0, lz4={"dict_match": 1}, lizv1={"dict_match": 1}))
    return out


def _tiny_cases(rng):
    """Dictionaries of 0 to 8 bytes, both layouts: the unit repeats the dictionary's bytes between zero runs, so its block
    is coded (its zeros pay for the 512 bytes a coded block must gain)."""
    out = []
    for n in range(9):
        d = _random(rng, n)
        u = d + bytes(30) + d * 3 + _random(rng, 50) + bytes(1200) + (d + b"xyz") * 4
        out += [DictCase("tiny", d, u, prefix, lz4={"block": 1}, lizv1={"block": 1}) for prefix in (False, True)]
    return out


def _repeat_cases(rng):
    """Pieces of the dictionary with one byte changed every 40: each piece after the first continues at the previous
    match's offset (a LIZv1 repeat offset into the dictionary)."""
    d = _random(rng, 30000)
    out = []
    for prefix in (False, True):
        piece = bytearray(d[20000:26000])
        for k in range(0, len(piece), 40):
            piece[k] ^= 0x55
        u = _random(rng, 500) + bytes(piece) + _random(rng, 2000) + d[-300:] + b"#" + d[-200:]
        out.append(DictCase("repeat", d, u, prefix, lz4={"dict_match": 100}, lizv1={"dict_match": 100, "dict_repeat": 100}))
    return out


def _corpus_cases():
    """Every corpus unit, cut to 64 KiB, against a dictionary of 32 KiB of another corpus unit and the unit's own last
    32 KiB (for a unit of more than 64 KiB, bytes that follow the cut, of the same kind)."""
    units = corpus_units()
    out = []
    for i, u in enumerate(units):
        d = units[(i + 7) % len(units)][-32768:] + u[-32768:]
        out.append(DictCase("corpus", d, u[:65536], i % 3 == 0))
    return out


def _poisoned_cases(rng):
    """A dictionary A + M + B (A, B of 24 bytes) and a unit C 0... Y A 0... B X 0... whose first 24 bytes C are a piece of
    M; between them zero runs, so the block is coded and A, B and C are dictionary matches of exactly 24 bytes (the
    pieces hold no zero).  The bytes after the dictionary are X (what follows B in the unit), the bytes in front of the
    dictionary are Y (what precedes A in the unit) and the bytes in front of the unit are those in front of C in M.  A
    kernel that counts on in the dictionary's buffer past its end instead of at the unit's first byte, or extends a match
    below the dictionary's or the unit's start, finds longer matches than the reference."""
    out = []
    for j in range(4):
        A, B, M = _nonzero(rng, 24), _nonzero(rng, 24), _nonzero(rng, 3000)
        d = A + M + B
        c_at = 1000 + 100 * j
        C = M[c_at:c_at + 24]
        X, Y = bytearray(_nonzero(rng, 40)), _nonzero(rng, 32)
        if X[0] == C[0]:                                # B's match continues at the unit's first byte, and stops there
            X[0] ^= 0x5A
        u = C + bytes(400) + Y + A + bytes(300) + B + bytes(X) + bytes(300)
        prefix = j == 3
        want = {("dict_match", 24): 2}                  # A and B; C's match starts behind the unit's first byte, a literal
        out.append(DictCase("poisoned", d, u, prefix, before_dict=Y, after_dict=b"" if prefix else bytes(X),
                            before_unit=b"" if prefix else M[c_at - 32:c_at], lz4=want, lizv1=want))
    return out


def dict_corpus(seed=90):
    """The dictionary cases, family by family (far, straddle, periodic, tiny, repeat, corpus, poisoned); seeded, about
    12 MiB of dictionaries (the two 4 MiB ones twice) and 2.6 MiB of units."""
    rng = np.random.default_rng(seed)
    return (_far_cases(rng, HC_WINDOW) + _far_cases(rng, PF_WINDOW) + _straddle_cases(rng) + _periodic_cases(rng)
            + _tiny_cases(rng) + _repeat_cases(rng) + _corpus_cases() + _poisoned_cases(rng))


def dict_targets():
    """Codeword classes the streams of dict_corpus() reach, summed over DICT_WALKED_LEVELS: matches from the dictionary, into
    the unit, at the window's last offset, and (LIZv1) with 24-bit and repeat offsets into the dictionary."""
    return {"dict_match", "dict_straddle", "dict_edge", "dict_far", "dict_repeat"}


def poisoned_parse_ok(classes):
    """A poisoned unit's stream at one level: three dictionary matches (C, A, B) of 23 or 24 bytes and none longer, which a
    kernel that read the poisoned surroundings would have found."""
    lengths = Counter({k[1]: v for k, v in classes.items() if isinstance(k, tuple) and k[0] == "dict_match"})
    return sum(lengths.values()) == 3 and set(lengths) <= {23, 24}


def dict_missing(case, lizv1, classes):
    """What `classes` (summed over the case's walked levels of one flavour) lacks of case.expect: (class, have, want)."""
    want = case.expect["lizv1" if lizv1 else "lz4"]
    return sorted(((k, classes[k], n) for k, n in want.items() if classes[k] < n), key=str)


CORPUS_DICT_SHARE = 0.5         # the least share of the corpus family's cases whose streams hold a dictionary match


def dict_shortfalls(cases, walked):
    """walked: level -> the walk classes of every case at that level (DICT_WALKED_LEVELS).  Returns what falls short, case
    by case and flavour by flavour: the expectations of dict_missing, and for the corpus family the share of cases with a
    dictionary match (CORPUS_DICT_SHARE).  Empty when every family reaches what it is built for."""
    out = []
    for lizv1 in (False, True):
        seen = [Counter() for _ in cases]
        for level, per_case in walked.items():
            if is_lizv1(level) == lizv1:
                for acc, classes in zip(seen, per_case):
                    acc.update(classes)
        for i, (c, acc) in enumerate(zip(cases, seen)):
            m = dict_missing(c, lizv1, acc)
            if m:
                out.append((i, c, "lizv1" if lizv1 else "lz4", m))
        corp = [acc for c, acc in zip(cases, seen) if c.family == "corpus"]
        share = sum(1 for acc in corp if acc["dict_match"]) / max(len(corp), 1)
        if share < CORPUS_DICT_SHARE:
            out.append(("corpus", "lizv1" if lizv1 else "lz4", share))
    return out
