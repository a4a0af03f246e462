"""Required tokens (vbt_tokenize_batch_spans) over the oracle's dictionary: the lattice of tests/bounded_oracle.py with
the span rules of README "Required tokens", restated in Python.

For a span [a, b) (byte offsets; character positions below) with an optional pattern:
  1. a and b are required boundaries, with the bounded oracle's lim(sw) rules;
  2. no node ends strictly inside the span: the loop skips every interior start position (its ends row is empty);
  3. where a word starts at a, the candidates are the user-, then the system-lexicon words of surface [a, b) whose
     feature matches the pattern, in lattice order; without any, one unknown word [a, b) per unk.def entry of the
     category of character a that matches (every entry of the category when none does);
  4. a pattern is split into csv fields like a feature; each field that is not exactly "*" must equal the word's field
     of the same index; a field the word lacks never matches; an empty pattern matches every word;
  5. the ignore_space skip is unchanged;  6. nothing else changes.

SpanOracle.lattice(sent, bounds) takes `bounds` as a plain boundary list (the bounded oracle) or as a Constraints
(boundaries and spans), so lattice_oracle, marginal_oracle and sampling_oracle run over the span lattice unchanged.
Test infrastructure."""
from typing import NamedTuple

from bounded_oracle import BoundedOracle

MAX_FIELDS, MAX_FIELD_INDEX = 16, 255
SPAN_ANY = 0xFFFFFFFF


class Constraints(NamedTuple):
    bounds: tuple = ()
    spans: tuple = ()  # (start_byte, end_byte) or (start_byte, end_byte, pattern str / bytes / None)


class PatternError(ValueError):
    def __init__(self, pos, why):
        super().__init__(f"byte {pos}: {why}")
        self.pos = pos


def csv_fields(b):
    """The unquoted fields of a feature string, split as csv_fields in kernels.cu, with each field's first byte."""
    fields, cur, start = [], bytearray(), 0
    quoted, at_start, i = False, True, 0
    while i < len(b):
        c = b[i]
        if quoted:
            if c != 0x22:
                cur.append(c)
            elif i + 1 < len(b) and b[i + 1] == 0x22:
                cur.append(c)
                i += 1
            else:
                quoted = False
        elif c == 0x22 and at_start:
            quoted = True
        elif c == 0x2C:
            fields.append((bytes(cur), start))
            cur, start, at_start = bytearray(), i + 1, True
            i += 1
            continue
        else:
            cur.append(c)
        at_start = False
        i += 1
    fields.append((bytes(cur), start))
    return fields


def compile_pattern(p):
    """bytes or str -> [(field index, bytes)] of the constrained fields; PatternError past the limits."""
    if p is None:
        return []
    p = p.encode("utf-8") if isinstance(p, str) else bytes(p)
    if not p:
        return []
    out = []
    for i, (f, start) in enumerate(csv_fields(p)):
        if f == b"*":
            continue
        if i > MAX_FIELD_INDEX:
            raise PatternError(start, "field index above 255")
        if len(out) == MAX_FIELDS:
            raise PatternError(start, "more than 16 constrained fields")
        out.append((i, f))
    return out


def matches(feature, compiled):
    fields = [f for f, _ in csv_fields(feature.encode("utf-8") if isinstance(feature, str) else feature)]
    return all(i < len(fields) and fields[i] == v for i, v in compiled)


class SpanOracle(BoundedOracle):
    def __init__(self, od, char_def, unk_def, ignore_space=False, max_grouping_len=0):
        super().__init__(od, char_def, unk_def, ignore_space, max_grouping_len)
        self._feat = {}

    def feature(self, widx):
        f = self._feat.get(widx)
        if f is None:
            f = self._feat[widx] = self.od.feature(widx)
        return f

    def lattice(self, sent, bounds, trace=None):
        if not isinstance(bounds, Constraints):
            return super().lattice(sent, bounds, trace)
        text = sent.decode("utf-8")
        n = len(text)
        c2b = [0] * (n + 1)
        for i, ch in enumerate(text):
            c2b[i + 1] = c2b[i] + len(ch.encode("utf-8"))
        b2c = {b: i for i, b in enumerate(c2b)}
        ci = [self.od.char_info(ord(ch)) for ch in text]
        start_of, inside = {}, set()
        brk = {b2c[b] for b in bounds.bounds if 0 < b < len(sent)}
        prev_end = 0
        for sp in bounds.spans:
            a, b = sp[0], sp[1]
            if not (prev_end <= a < b <= len(sent)) or a not in b2c or b not in b2c:
                raise ValueError(f"invalid span {sp}")
            ca, cb = b2c[a], b2c[b]
            if self.space_mask and ci[ca] & self.space_mask:
                raise ValueError(f"span {sp} starts at a skipped space")
            if any(ca < c < cb for c in brk):
                raise ValueError(f"explicit boundary inside span {sp}")
            start_of[ca] = (cb, compile_pattern(sp[2] if len(sp) > 2 else None))
            inside.update(range(ca + 1, cb))
            brk.update(c for c in (ca, cb) if 0 < c < n)
            prev_end = b
        brk = sorted(brk)
        grp = [0] * n
        for i in range(n - 1, -1, -1):
            grp[i] = 1 if i == n - 1 or (ci[i] & ci[i + 1] & 0x3FFFF) == 0 else grp[i + 1] + 1
        for p in range(n):  # rule 5: a space skip may not land strictly inside a span
            if p not in inside and self.space_mask and ci[p] & self.space_mask and p + grp[p] in inside:
                raise ValueError(f"the space skip from character {p} lands inside a span")
        ends = [[] for _ in range(n + 1)]
        ends[0].append([0, 0, 0xFFFFFFFF, 0, 0, 0, 0, 0])  # BOS

        def lim(sw):
            for c in brk:
                if c > sw:
                    return c
            return n

        def insert(start_node, sw, ew, widx, left, right, cost):
            best, bi = None, 0
            for i, l in enumerate(ends[start_node]):
                v = self._wrap(l[6] + self.conn(l[4], left))
                if best is None or v <= best:
                    best, bi = v, i
            ends[ew].append([start_node, sw, widx, left, right, bi, self._wrap(best + cost), cost])
            if trace is not None:
                trace.append((start_node, sw, ew, widx))

        lex_types = (1, 0) if self.has_user else (0,)
        start_node = start_word = 0
        while start_word < n:
            if not ends[start_node]:
                start_word += 1
                start_node = start_word
                continue
            assert start_node not in inside  # rule 2: no node ends there
            if self.space_mask and (ci[start_node] & self.space_mask):
                start_word += grp[start_node]
            if start_word == n:
                break
            sw = start_word
            c = ci[sw]
            base = (c >> 18) & 0xFF
            if sw in start_of:  # rule 3
                cb, pat = start_of[sw]
                matched = False
                for lt in lex_types:
                    for wid, end_char in self.od.common_prefix(text[sw:cb], lt):
                        widx = (lt << 30) | wid
                        if sw + end_char == cb and matches(self.feature(widx), pat):
                            insert(start_node, sw, cb, widx, *self.param(widx))
                            matched = True
                if not matched:
                    ents = range(self.unk_off[base], self.unk_off[base + 1])
                    ok = [w for w in ents if matches(self.feature((2 << 30) | w), pat)]
                    for w in ok or ents:
                        insert(start_node, sw, cb, (2 << 30) | (w & 0xFFFF), *self.unk[w])
                start_word += 1
                start_node = start_word
                continue
            limit = lim(sw)
            matched = False
            for lt in lex_types:
                for wid, end_char in self.od.common_prefix(text[sw:limit], lt):
                    widx = (lt << 30) | wid
                    insert(start_node, sw, sw + end_char, widx, *self.param(widx))
                    matched = True
            if not (matched and not (c >> 26) & 1):
                g = min(grp[sw], limit - sw)

                def span(ew):
                    for w in range(self.unk_off[base], self.unk_off[base + 1]):
                        insert(start_node, sw, ew, (2 << 30) | (w & 0xFFFF), *self.unk[w])

                grouped = False
                if (c >> 27) & 1:
                    grouped = True
                    if self.mgl == 0 or g - 1 <= self.mgl:
                        span(sw + g)
                        matched = True
                for i in range(1, min(c >> 28, g) + 1):
                    if grouped and i == g:
                        continue
                    span(sw + i)
                    matched = True
                if not matched:
                    span(sw + 1)
            start_word += 1
            start_node = start_word
        best, bi = None, 0
        for i, l in enumerate(ends[start_node]):
            v = self._wrap(l[6] + self.conn(l[4], 0))
            if best is None or v <= best:
                best, bi = v, i
        return ends, (start_node, bi), c2b

    @staticmethod
    def _wrap(x):
        return (x + (1 << 31)) % (1 << 32) - (1 << 31)


def constraints(boundaries, spans):
    """Per-sentence Constraints from per-sentence boundary and span lists (either may be None)."""
    n = len(boundaries if boundaries is not None else spans)
    return [Constraints(tuple(boundaries[i]) if boundaries else (), tuple(spans[i]) if spans else ()) for i in range(n)]
