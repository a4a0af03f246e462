"""A restatement of the output formats (Tokenizer.output_format, `tokenize -F`) written from their definition in
README.md: its own parser of the format strings, rendering of the oracle's tokens, fields split by the oracle's
`_csv_row`, costs wrapped to i32.  Test infrastructure; it shares no code with vibrato_b200/csrc/format.cpp."""
import numpy as np

from oracle import vibrato_oracle as vo

ESCAPES = {"0": b"\0", "a": b"\a", "b": b"\b", "t": b"\t", "n": b"\n", "v": b"\v", "f": b"\f", "r": b"\r", "s": b" ",
           "\\": b"\\"}
NO_VALUE = ("h", "t", "P", "pP", "pA", "pB", "pi", "pb", "pp")
TOKEN_DIRECTIVES = ("m", "M", "pS", "H", "c", "pw", "pc", "pn", "pC", "ps", "pe", "pl", "pL", "phl", "phr", "s")


class FormatError(Exception):
    pass


def wrap(x):
    return (int(x) + (1 << 31)) % (1 << 32) - (1 << 31)


def parse(fmt, tokens=True):
    """-> list of pieces: ("lit", bytes) | (directive,) | ("f", [indices], sep byte).  Raises FormatError(pos)."""
    s = fmt.encode("utf-8") if isinstance(fmt, str) else bytes(fmt)
    out, i = [], 0

    def lit(b):
        if out and out[-1][0] == "lit":
            out[-1] = ("lit", out[-1][1] + b)
        else:
            out.append(("lit", b))

    def esc(i):
        if i + 1 >= len(s) or chr(s[i + 1]) not in ESCAPES:
            raise FormatError(i)
        return ESCAPES[chr(s[i + 1])], i + 2

    while i < len(s):
        c = s[i:i + 1]
        if c == b"\\":
            b, i = esc(i)
            lit(b)
            continue
        if c != b"%":
            lit(c)
            i += 1
            continue
        at = i
        i += 1
        if i >= len(s):
            raise FormatError(at)
        d = chr(s[i])
        i += 1
        if d == "%":
            lit(b"%")
            continue
        if d in "SL":
            out.append((d,))
            continue
        if d == "p":
            if i >= len(s):
                raise FormatError(at)
            d += chr(s[i])
            i += 1
            if d == "ph" and i < len(s) and chr(s[i]) in "lr":
                d += chr(s[i])
                i += 1
        if d in NO_VALUE or not tokens:
            raise FormatError(at)
        if d in TOKEN_DIRECTIVES:
            out.append((d,))
            continue
        if d in ("f", "F"):
            sep = b"\t"
            if d == "F":
                if i >= len(s):
                    raise FormatError(at)
                if s[i:i + 1] == b"\\":
                    sep, i = esc(i)
                else:
                    sep, i = s[i:i + 1], i + 1
            if s[i:i + 1] != b"[":
                raise FormatError(at)
            j = s.find(b"]", i)
            if j < 0:
                raise FormatError(at)
            parts = s[i + 1:j].split(b",")
            if not all(p.isdigit() for p in parts) or any(int(p) > 255 for p in parts):
                raise FormatError(at)
            out.append(("f", [int(p) for p in parts], sep))
            i = j + 1
            continue
        raise FormatError(at)
    return out


class Format:
    def __init__(self, node, unk=None, bos="", eos="EOS\n"):
        self.node = parse(node)
        self.unk = self.node if unk is None else parse(unk)
        self.bos = parse(bos, tokens=False)
        self.eos = parse(eos, tokens=False)
        idx = {k for p in self.node + self.unk if p[0] == "f" for k in p[1]}
        if len(idx) > 16:
            raise FormatError("fields")


def render(pieces, sent, tok=None, prev=None, od=None, cache=None):
    out = bytearray()
    for p in pieces:
        d = p[0]
        if d == "lit":
            out += p[1]
        elif d == "S":
            out += sent
        elif d == "L":
            out += str(len(sent)).encode()
        else:
            w = int(tok["word_idx"])
            sb, eb, total = int(tok["start_byte"]), int(tok["end_byte"]), int(tok["total_cost"])
            pe, pt = (int(prev["end_byte"]), int(prev["total_cost"])) if prev is not None else (0, 0)
            if w not in cache:
                cache[w] = (od.feature(w).encode("utf-8"), od.word_param(w))
            feat, (lid, rid, wcost) = cache[w]
            if d == "m":
                out += sent[sb:eb]
            elif d == "M":
                out += sent[pe:eb]
            elif d == "pS":
                out += sent[pe:sb]
            elif d == "H":
                out += feat
            elif d == "f":
                fields = vo._csv_row(feat.decode("utf-8"))
                got = [fields[k] if k < len(fields) else "*" for k in p[1]]
                out += p[2].join(x.encode("utf-8") for x in got if not x.startswith("*"))
            else:
                v = {"c": wcost, "pw": wcost, "pc": total, "pn": wrap(total - pt), "pC": wrap(total - pt - wcost),
                     "ps": sb, "pe": eb, "pl": eb - sb, "pL": eb - pe, "phl": lid, "phr": rid, "s": int(w >> 30 == 2)}[d]
                out += str(v).encode()
    return bytes(out)


def format_batch(od, fmt, utf8, offsets, tok_off, toks):
    """(text_offsets uint64[n + 1], text bytes) of Format `fmt` over the oracle's tokens."""
    buf = bytes(memoryview(np.ascontiguousarray(utf8)))
    out = bytearray()
    text_off = np.zeros(len(offsets), dtype=np.uint64)
    cache = {}
    for i in range(len(offsets) - 1):
        text_off[i] = len(out)
        sent = buf[int(offsets[i]):int(offsets[i + 1])]
        out += render(fmt.bos, sent)
        prev = None
        for k in range(int(tok_off[i]), int(tok_off[i + 1])):
            t = toks[k]
            out += render(fmt.unk if int(t["word_idx"]) >> 30 == 2 else fmt.node, sent, t, prev, od, cache)
            prev = t
        out += render(fmt.eos, sent)
    text_off[len(offsets) - 1] = len(out)
    return text_off, bytes(out)
