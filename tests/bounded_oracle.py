"""Required token boundaries over the oracle's dictionary: an independent restatement of the lattice of
Tokenizer::build_lattice_inner / add_lattice_edges (tokenizer.rs:94-199) and UnkHandler::gen_unk_words
(dictionary/unknown.rs:69-116), in Python, with the boundary rules of vbt_tokenize_batch_bounded:

  lim(sw) = the first boundary character position after sw, or the sentence's length;
  1. a lexicon word ending after lim(sw) is no candidate and no match;
  2. gen_unk_words uses min(groupable, lim(sw) - sw) in place of groupable;
  3. the ignore_space skip is unchanged;  4. nothing else changes.

Without boundaries it computes what the oracle's C restatement computes (the CPU tests check that).  It reads the
dictionary through the oracle's primitives (char_info, common_prefix, word_param, conn_cost); the unknown-word
entries of a category come from unk.def, grouped by category id as UnkHandler does (unknown.rs:63-66).
A sentence whose lattice has no path to EOS (possible when unk.def has no entry for a character category, with or
without boundaries) is not defined here: the reference indexes out of bounds there, and this restatement raises.
Test infrastructure."""
import numpy as np

from oracle import vibrato_oracle as vo

TOKEN_DTYPE = np.dtype([("start_char", "<u4"), ("end_char", "<u4"), ("start_byte", "<u4"), ("end_byte", "<u4"),
                        ("word_idx", "<u4"), ("total_cost", "<i4")])


def wrap(x):
    return (x + (1 << 31)) % (1 << 32) - (1 << 31)


def _categories(char_def):
    """Category names by id: DEFAULT first, then the order in which char.def defines them."""
    names = ["DEFAULT"]
    for line in char_def.splitlines():
        line = line.split("#", 1)[0].strip()
        if not line or line.startswith("0x"):
            continue
        name = line.split()[0]
        if name not in names:
            names.append(name)
    return names


class BoundedOracle:
    def __init__(self, od, char_def, unk_def, ignore_space=False, max_grouping_len=0):
        self.od = od
        self.ignore_space, self.mgl = ignore_space, max_grouping_len
        cats = _categories(char_def)
        self.space_mask = (1 << cats.index("SPACE")) if ignore_space else 0
        cate_of = [cats.index(line.split(",", 1)[0]) for line in unk_def.splitlines() if line.strip()]
        order = sorted(range(len(cate_of)), key=lambda i: cate_of[i])  # stable, as the reference sorts
        self.unk_off = [0] * (len(cats) + 1)
        for i in order:
            self.unk_off[cate_of[i] + 1] += 1
        for c in range(len(cats)):
            self.unk_off[c + 1] += self.unk_off[c]
        self.unk = [od.word_param((2 << 30) | w) for w in range(od.num_words(2))]
        assert len(self.unk) == len(cate_of)
        self.has_user = od.num_words(1) > 0
        self._param = {}
        self._conn = {}

    def param(self, widx):
        p = self._param.get(widx)
        if p is None:
            p = self._param[widx] = self.od.word_param(widx)
        return p

    def conn(self, right, left):
        c = self._conn.get((right, left))
        if c is None:
            c = self._conn[(right, left)] = self.od.conn_cost(right, left)
        return c

    def char_infos(self, text):
        """CharInfo of each character (Sentence::compute_basic, sentence.rs:48-55): out-of-table code points take
        entry 0 (character.rs:112-116)."""
        return [self.od.char_info(ord(ch)) for ch in text]

    @staticmethod
    def groupable(ci):
        """compute_groupable (sentence.rs:57-71): the length of the run from each character in which every two
        adjacent characters share a category bit."""
        n = len(ci)
        grp = [0] * n
        for i in range(n - 1, -1, -1):
            grp[i] = 1 if i == n - 1 or (ci[i] & ci[i + 1] & 0x3FFFF) == 0 else grp[i + 1] + 1
        return grp

    def skips(self, c):
        """Whether the ignore_space skip runs from a character of CharInfo c (tokenizer.rs:117-125): SPACE in its id
        set, secondary categories included."""
        return bool(self.space_mask and c & self.space_mask)

    def lattice(self, sent, bounds, trace=None):
        """sent: bytes.  Returns (ends, eos, c2b): ends[i] = nodes ending at character i, a node being
        [start_node, start_word, word_idx, left, right, min_idx, min_cost, word_cost] (word_cost from the entry
        itself: an unknown word's word_idx keeps only 16 bits of its entry, unknown.rs:133).  `trace` (a list) receives
        (start_node, start_word, end, word_idx) for every inserted node, in insertion order."""
        text = sent.decode("utf-8")
        n = len(text)
        c2b = [0] * (n + 1)
        for i, ch in enumerate(text):
            c2b[i + 1] = c2b[i] + len(ch.encode("utf-8"))
        b2c = {b: i for i, b in enumerate(c2b)}
        brk = sorted({b2c[b] for b in bounds if 0 < b < len(sent)})
        ci = self.char_infos(text)
        grp = self.groupable(ci)
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
                v = wrap(l[6] + self.conn(l[4], left))
                if best is None or v <= best:
                    best, bi = v, i
            ends[ew].append([start_node, sw, widx, left, right, bi, wrap(best + cost), cost])
            if trace is not None:
                trace.append((start_node, sw, ew, widx))

        start_node = start_word = 0
        while start_word < n:
            if not ends[start_node]:
                start_word += 1
                start_node = start_word
                continue
            if self.skips(ci[start_node]):
                start_word += grp[start_node]
            if start_word == n:
                break
            sw = start_word
            limit = lim(sw)
            matched = False
            lex_types = (1, 0) if self.has_user else (0,)
            for lt in lex_types:  # rule 1: the walk sees the characters up to the boundary only
                for wid, end_char in self.od.common_prefix(text[sw:limit], lt):
                    widx = (lt << 30) | wid
                    left, right, cost = self.param(widx)
                    insert(start_node, sw, sw + end_char, widx, left, right, cost)
                    matched = True
            c = ci[sw]
            if not (matched and not (c >> 26) & 1):
                g = min(grp[sw], limit - sw)  # rule 2
                base = (c >> 18) & 0xFF

                def span(ew):
                    for w in range(self.unk_off[base], self.unk_off[base + 1]):
                        left, right, cost = self.unk[w]
                        insert(start_node, sw, ew, (2 << 30) | (w & 0xFFFF), left, right, cost)

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
            v = wrap(l[6] + self.conn(l[4], 0))
            if best is None or v <= best:
                best, bi = v, i
        return ends, (start_node, bi), c2b

    def best_cost(self, sent, bounds=()):
        """Cost of the best path, EOS connection included (the min_cost of EOS)."""
        if not sent:
            return 0
        ends, (end_node, idx), _ = self.lattice(sent, bounds)
        return wrap(ends[end_node][idx][6] + self.conn(ends[end_node][idx][4], 0))

    def tokenize(self, sent, bounds=()):
        """Tokens of one sentence (bytes) as a TOKEN_DTYPE array.  The reference keeps the best predecessor's row
        index as u16 (lattice.rs:144, EOS too), so in a row of more than 65 536 nodes the backtrack follows the
        truncated index."""
        if not sent:
            return np.zeros(0, dtype=TOKEN_DTYPE)
        ends, (end_node, idx), c2b = self.lattice(sent, bounds)
        idx &= 0xFFFF
        out = []
        while end_node != 0:
            nd = ends[end_node][idx]
            out.append((nd[1], end_node, c2b[nd[1]], c2b[end_node], nd[2], nd[6]))
            end_node, idx = nd[0], nd[5] & 0xFFFF
        return np.array(out[::-1], dtype=TOKEN_DTYPE)

    def tokenize_batch(self, sentences, boundaries=None):
        """sentences: list of bytes; boundaries: one list per sentence or None.  Returns (tok_off u64[n+1], tokens)."""
        toks = [self.tokenize(s, boundaries[i] if boundaries else ()) for i, s in enumerate(sentences)]
        off = np.zeros(len(toks) + 1, dtype=np.uint64)
        off[1:] = np.cumsum([len(t) for t in toks])
        return off, (np.concatenate(toks) if toks else np.zeros(0, dtype=TOKEN_DTYPE))

    def connid_counts(self, sentences, boundaries=None):
        """Lattice::add_connid_counts (lattice.rs:170-183) summed over the batch, in the dictionary's own ids."""
        lid = np.zeros(self.od.num_left, dtype=np.uint64)
        rid = np.zeros(self.od.num_right, dtype=np.uint64)
        for i, s in enumerate(sentences):
            if not s:
                continue
            ends, (end_node, _), _ = self.lattice(s, boundaries[i] if boundaries else ())
            n = len(ends) - 1
            for e in range(1, n + 1):
                for r in ends[e]:
                    for l in ends[r[0]]:
                        lid[r[3]] += 1
                        rid[l[4]] += 1
            for l in ends[n]:
                lid[0] += 1
                rid[l[4]] += 1
        return lid, rid


def vo_dictionary(lex, matrix, char_def, unk_def, user=None, dual=False):
    od = vo.OracleDictionary(lex, matrix, char_def, unk_def, dual_connector=dual)
    if user is not None:
        od.set_user_csv(user)
    return od
