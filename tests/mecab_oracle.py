"""Python restatement of mecab::generate_bigram_info (vibrato/src/mecab.rs:31-181) and of the bigram half of
FeatureExtractor (trainer/feature_extractor.rs:39-249) it uses.  Test infrastructure: written from the Rust with `re`
and dicts, sharing no code with the library's C++ (vibrato_b200/csrc/mecab_model.cpp), so that the tests can compare
the two byte for byte.

Errors are raised as MecabOracleError(kind, message), kind being the VibratoError variant's name."""
import re

from oracle.vibrato_oracle import _csv_row

ID_FEATURE_RE = re.compile(r"^([0-9]+) (.*)$", re.S)
MODEL_RE = re.compile(r"^([0-9\-\.]+)\t(.*)$", re.S)
LEFT_RE = re.compile(r"%(L|L\?)\[([0-9]+)\]")
RIGHT_RE = re.compile(r"%(R|R\?)\[([0-9]+)\]")
UNIGRAM_RE = re.compile(r"%((F|F\?)\[([0-9]+)\]|t)")
# f64::from_str restricted to the characters MODEL_RE admits
RUST_F64_RE = re.compile(r"^-?([0-9]+|[0-9]+\.[0-9]*|[0-9]*\.[0-9]+)$")
USIZE_MAX = (1 << 64) - 1
I32_MIN, I32_MAX = -(1 << 31), (1 << 31) - 1
# char::is_whitespace, which str::trim uses
WHITE_SPACE = "\t\n\v\f\r \x85\xa0\u1680" + "".join(map(chr, range(0x2000, 0x200B))) + "\u2028\u2029\u202f\u205f\u3000"


class MecabOracleError(Exception):
    def __init__(self, kind, msg):
        self.kind = kind
        super().__init__(f"{kind}: {msg}")


def _usize(digits):
    v = int(digits)
    if v > USIZE_MAX:
        raise MecabOracleError("ParseInt", "number too large to fit in target type")
    return v


def _lines(data):
    """BufRead::lines(): split on "\\n", a "\\r\\n" ending loses its "\\r"; a line that is not UTF-8 is an I/O error."""
    if isinstance(data, str):
        data = data.encode("utf-8")
    parts = data.split(b"\n")
    if parts[-1] == b"":
        parts.pop()
    for i, p in enumerate(parts):
        if i < len(parts) - 1 or data.endswith(b"\n"):
            p = p[:-1] if p.endswith(b"\r") else p
        try:
            yield p.decode("utf-8")
        except UnicodeDecodeError:
            raise MecabOracleError("StdIo", "stream did not contain valid UTF-8") from None


def _parse_template(template, pattern):
    """(template, [required index], [(start, end, index)])"""
    required, captures = [], []
    for m in pattern.finditer(template):
        idx = _usize(m.group(2))
        if m.group(1).endswith("?"):
            required.append(idx)
        captures.append((m.start(), m.end(), idx))
    return template, required, captures


class _Side:
    """One side's templates and the feature-id map all of them share (extract_feature_ids)."""

    def __init__(self):
        self.templates = []
        self.ids = {}

    def extract(self, features):
        def get(i):
            return features[i] if i < len(features) else "*"

        out = []
        for raw, required, captures in self.templates:
            if any(get(i) == "*" for i in required):
                out.append(None)
                continue
            s, start = [], 0
            for b, e, idx in captures:
                s.append(raw[start:b])
                s.append(get(idx))
                start = e
            s.append(raw[start:])
            out.append(self.ids.setdefault("".join(s), len(self.ids) + 1))
        return out


def parse_feature_config(feature_def):
    """TrainerConfig::parse_feature_config (trainer/config.rs:64-101) -> (left side, right side)."""
    left, right = _Side(), _Side()
    for line in _lines(feature_def):
        line = line.strip(WHITE_SPACE)
        if not line or line.startswith("#"):
            continue
        if line.startswith("UNIGRAM "):
            for m in UNIGRAM_RE.finditer(line[8:]):
                if m.group(3) is not None:
                    _usize(m.group(3))
        elif line.startswith("BIGRAM "):
            spl = line[7:].split("/")
            if len(spl) != 2:
                raise MecabOracleError("InvalidFormat", "feature.def: Invalid bigram template")
            left.templates.append(_parse_template(spl[0], LEFT_RE))
            right.templates.append(_parse_template(spl[1], RIGHT_RE))
        else:
            raise MecabOracleError("InvalidFormat", "feature: ")
    return left, right


def _read_id_def(data, side, name):
    out = {}
    for line in _lines(data):
        m = ID_FEATURE_RE.match(line)
        if not m:
            raise MecabOracleError("InvalidFormat", f"{name}: each line must be a pair of an ID and features")
        i = _usize(m.group(1))
        spl = _csv_row(m.group(2))
        if i == 0 and spl and spl[0] != "BOS/EOS":
            raise MecabOracleError("InvalidFormat", f"{name}: ID 0 must be BOS/EOS")
        out[i] = side.extract(spl)
    return out


def _cost(weight, cost_factor):
    """`-(weight * cost_factor) as i32`: negate, then a saturating cast toward zero; NaN is 0."""
    x = -(weight * cost_factor)
    if x != x:
        return 0
    if x in (float("inf"), float("-inf")):
        return I32_MAX if x > 0 else I32_MIN
    return max(I32_MIN, min(I32_MAX, int(x)))


def _write(features, name):
    out = []
    for i in range(1, len(features)):
        if i not in features:
            raise MecabOracleError("InvalidFormat", f"{name}: feature ID {i} is undefined")
        out.append(f"{i}\t" + ",".join("*" if f is None else str(f) for f in features[i]) + "\n")
    return "".join(out).encode("utf-8")


def generate_bigram_info(feature_def, right_id_def, left_id_def, model_def, cost_factor):
    """-> (bigram_right, bigram_left, bigram_cost) bytes; arguments as in mecab.rs:31-40."""
    left, right = parse_feature_config(feature_def)
    left_features = _read_id_def(right_id_def, left, "right_id_def_rdr")
    right_features = _read_id_def(left_id_def, right, "left_id_def_rdr")
    cost_lines = []
    for line in _lines(model_def):
        m = MODEL_RE.match(line)
        if not m:
            continue
        if not RUST_F64_RE.match(m.group(1)):
            raise MecabOracleError("ParseFloat", "invalid float literal")
        cost = _cost(float(m.group(1)), float(cost_factor))
        if cost == 0:
            continue
        spl = m.group(2).replace("BOS/EOS", "").split("/")
        if len(spl) < 2:
            continue
        lf, rf = spl[0], spl[1]
        if lf and lf not in left.ids:
            continue
        if rf and rf not in right.ids:
            continue
        lid = str(left.ids[lf]) if lf else ""
        rid = str(right.ids[rf]) if rf else ""
        cost_lines.append(f"{lid}/{rid}\t{cost}\n")
    return (_write(left_features, "right_id_def_rdr"), _write(right_features, "left_id_def_rdr"),
            "".join(cost_lines).encode("utf-8"))
