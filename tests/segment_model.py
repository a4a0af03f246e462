"""The candidate pool's segment encoding, restated in plain Python (kernels.cu: SegOut::push encodes, cand_at and
seg_record decode).

K2 (k_candidates) writes one 8-byte segment per candidate source of a start position: a trie hit's postings list or
an unknown-word span of unk.def entries, in the order Tokenizer::add_lattice_edges inserts them.
  x = kind | index   kind USER / UNK / 0 (system); index: a postings list's header (record j at index + 1 + j) or
                     the first unk.def entry (record j at index + j)
  y = delta << 16 | count   delta (signed 16 bits) moves the run's end slot from the previous segment's end (from
                     the position's own slot for the first one)
A move of more than 32 767 goes through count-0 segments of +-32 767; a source of 2^16 candidates or more becomes
several segments of at most 65 535, the index advanced by the candidates before (`v += c`).

A position's candidate trace (BoundedOracle.lattice(trace=...)) is grouped into sources: consecutive candidates of
the same lexicon type and end.  The records of each source are laid out in an image of the position's own, a
postings list behind a header entry as in the dictionary image, so that decoding goes through the same index
arithmetic as the kernels.  Test infrastructure."""
MAX_DELTA = 32767
MAX_COUNT = 0xFFFF
USER, UNK, INDEX = 0x80000000, 0x40000000, 0x3FFFFFFF
HEADER = None  # the header entry of a postings list in the image


def pack_y(delta, count):
    assert -MAX_DELTA <= delta <= MAX_DELTA and 0 <= count <= MAX_COUNT
    return ((delta & 0xFFFF) << 16) | count


def unpack_y(y):
    """int32_t(y) >> 16 (sign-extending) and y & 0xFFFF"""
    d = y >> 16
    return (d - 0x10000 if d & 0x8000 else d), y & 0xFFFF


def lex_type(x):
    """0 system, 1 user, 2 unknown: the lexicon type of a segment's candidates (word_idx >> 30)."""
    return 1 if x & USER else 2 if x & UNK else 0


def follows(prev, widx):
    """Does word_idx `widx` come right after `prev` in its postings list (word ids are consecutive there: see
    test_span_limits_model) or in unk.def (the 16-bit entry index, mod 2^16)?"""
    if widx >> 30 == 2:
        return widx & 0xFFFF == (prev + 1) & 0xFFFF
    return widx == prev + 1


def sources(cands, spans=False):
    """cands: [(end, word_idx)] of one position in insertion order -> [(lex type, end, [word_idx...])].  spans: a
    source also breaks where a record is skipped (span_postings and count_span push one segment per run of records
    that match a span's pattern)."""
    out = []
    for end, widx in cands:
        lt = widx >> 30
        if out and out[-1][0] == lt and out[-1][1] == end and (not spans or follows(out[-1][2][-1], widx)):
            out[-1][2].append(widx)
        else:
            out.append((lt, end, [widx]))
    return out


def encode(slot, cands, spans=False):
    """SegOut::push over the sources of the position at `slot` -> (segments [(x, y)], image)."""
    segs, image, last = [], [], slot
    for lt, end, words in sources(cands, spans):
        if lt == 2:
            v = UNK | len(image)
        else:
            image.append(HEADER)
            v = (USER if lt == 1 else 0) | (len(image) - 1)
        image += words
        count, delta = len(words), end - last
        while delta > MAX_DELTA or delta < -MAX_DELTA:
            step = MAX_DELTA if delta > 0 else -MAX_DELTA
            segs.append((v, pack_y(step, 0)))
            delta -= step
        last = end
        while True:
            c = min(count, MAX_COUNT)
            segs.append((v, pack_y(delta, c)))
            count -= c
            if count == 0:
                break
            v += c  # the next run starts c records further; for postings the index stays one before the run
            delta = 0
    assert len(image) <= INDEX
    return segs, image


def seg_record(seg, image, j):
    x = seg[0]
    rec = image[(x & INDEX) + j] if x & UNK else image[(x & INDEX) + 1 + j]
    assert rec is not HEADER and rec >> 30 == lex_type(x)
    return rec


def cand_at(slot, enc, j):
    """Candidate j of the position: (end, word_idx), found by walking its segments as cand_at does."""
    segs, image = enc
    h, end = 0, slot
    while True:
        delta, c = unpack_y(segs[h][1])
        end += delta
        if j < c:
            return end, seg_record(segs[h], image, j)
        j -= c
        h += 1


def walk(slot, enc):
    """[(lex type, end, count)] of every segment, move segments (count 0) included."""
    out, end = [], slot
    for x, y in enc[0]:
        delta, c = unpack_y(y)
        end += delta
        out.append((lex_type(x), end, c))
    return out


def deltas(enc):
    return [unpack_y(y)[0] for _, y in enc[0]]


def moves(enc):
    return sum(1 for _, y in enc[0] if unpack_y(y)[1] == 0)


def n_segments(enc):
    return len(enc[0])


def positions(bo, sent, bounds=(), slot0=0):
    """{slot: [(end slot, word_idx)]} of the positions BoundedOracle visits in one sentence (bytes), whose first slot
    is slot0 (a sentence of n characters takes n + 1 slots).  Positions the reference never reaches (no path into
    them) are missing; K2 encodes those too."""
    trace = []
    bo.lattice(sent, bounds, trace=trace)
    out = {}
    for start_node, _, end, widx in trace:
        out.setdefault(slot0 + start_node, []).append((slot0 + end, widx))
    return out


def unknown_cands(sw, g, length, words, mgl=0):
    """Closed form of UnkHandler::gen_unk_words (unknown.rs:69-116) at a start word with no lexicon match in an
    INVOKE 1, GROUP 1 category of LENGTH `length`, whose run has g characters from sw: [(end, word_idx)] with the
    category's unk.def entries `words`.  The CPU tests check it against BoundedOracle on short runs."""
    ends = []
    if mgl == 0 or g - 1 <= mgl:
        ends.append(sw + g)
    ends += [sw + i for i in range(1, min(length, g) + 1) if i != g]
    if not ends:
        ends = [sw + 1]
    return [(e, w) for e in ends for w in words]


def run_positions(n, length, words, mgl=0, slot0=0):
    """{slot: cands} of every position of a sentence that is one run of n characters of such a category."""
    return {slot0 + p: unknown_cands(slot0 + p, n - p, length, words, mgl) for p in range(n)}


def totals(pos):
    """(segments, candidates) over the positions of `pos`."""
    return sum(n_segments(encode(s, c)) for s, c in pos.items()), sum(len(c) for c in pos.values())
