/*
 * vibrato_oracle.c — CPU restatement of daac-tools/vibrato 0.5.2's tokenisation path (plain C).
 *
 * TEST INFRASTRUCTURE ONLY (see vibrato_oracle.h).  It is the parity checker for the CUDA path
 * and the timed CPU baseline ("port") of bench.py; it is never part of the product path.
 *
 * Each function cites the reference file:line (relative to /root/reference/vibrato/src/) it
 * restates.  Data-structure layouts are this file's own; only results (and their order) follow
 * the reference.
 */
#define _GNU_SOURCE
#include "vibrato_oracle.h"

#include <pthread.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

/* ------------------------------------------------------------------------------------------ */
/* small utilities                                                                             */
/* ------------------------------------------------------------------------------------------ */

static void set_err(char *err, size_t cap, const char *fmt, ...) {
    if (!err || cap == 0) return;
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(err, cap, fmt, ap);
    va_end(ap);
}

static void *xmalloc(size_t n) {
    void *p = malloc(n ? n : 1);
    if (!p) {
        fprintf(stderr, "vibrato_oracle: out of memory (%zu bytes)\n", n);
        abort();
    }
    return p;
}
static void *xcalloc(size_t n, size_t m) {
    void *p = calloc(n ? n : 1, m ? m : 1);
    if (!p) {
        fprintf(stderr, "vibrato_oracle: out of memory\n");
        abort();
    }
    return p;
}
static void *xrealloc(void *q, size_t n) {
    void *p = realloc(q, n ? n : 1);
    if (!p) {
        fprintf(stderr, "vibrato_oracle: out of memory (%zu bytes)\n", n);
        abort();
    }
    return p;
}

void vo_free(void *p) { free(p); }

/* std::str::from_utf8 acceptance (what `stdin.lines()` / `&str` guarantee before worker.rs:34). */
int vo_utf8_valid(const char *s_, size_t len) {
    const unsigned char *s = (const unsigned char *)s_;
    size_t i = 0;
    while (i < len) {
        unsigned c = s[i];
        if (c < 0x80) {
            i++;
        } else if (c >= 0xC2 && c <= 0xDF) {
            if (i + 1 >= len || (s[i + 1] & 0xC0) != 0x80) return 0;
            i += 2;
        } else if (c >= 0xE0 && c <= 0xEF) {
            if (i + 2 >= len) return 0;
            unsigned c1 = s[i + 1], c2 = s[i + 2];
            if ((c1 & 0xC0) != 0x80 || (c2 & 0xC0) != 0x80) return 0;
            if (c == 0xE0 && c1 < 0xA0) return 0; /* overlong */
            if (c == 0xED && c1 > 0x9F) return 0; /* surrogates */
            i += 3;
        } else if (c >= 0xF0 && c <= 0xF4) {
            if (i + 3 >= len) return 0;
            unsigned c1 = s[i + 1], c2 = s[i + 2], c3 = s[i + 3];
            if ((c1 & 0xC0) != 0x80 || (c2 & 0xC0) != 0x80 || (c3 & 0xC0) != 0x80) return 0;
            if (c == 0xF0 && c1 < 0x90) return 0;
            if (c == 0xF4 && c1 > 0x8F) return 0;
            i += 4;
        } else {
            return 0;
        }
    }
    return 1;
}

/* Decodes one scalar value from valid UTF-8; returns bytes consumed. */
static inline unsigned utf8_decode(const unsigned char *s, uint32_t *cp) {
    unsigned c = s[0];
    if (c < 0x80) {
        *cp = c;
        return 1;
    }
    if (c < 0xE0) {
        *cp = ((c & 0x1F) << 6) | (s[1] & 0x3F);
        return 2;
    }
    if (c < 0xF0) {
        *cp = ((c & 0x0F) << 12) | ((s[1] & 0x3F) << 6) | (s[2] & 0x3F);
        return 3;
    }
    *cp = ((c & 0x07) << 18) | ((s[1] & 0x3F) << 12) | ((s[2] & 0x3F) << 6) | (s[3] & 0x3F);
    return 4;
}

/* ------------------------------------------------------------------------------------------ */
/* CharInfo / CharProperty  (dictionary/character.rs)                                          */
/* ------------------------------------------------------------------------------------------ */

/* character.rs:10-24: cate_idset 18 bits | base_id 8 | invoke 1 | group 1 | length 4 */
#define CI_CATE_BITS 18
#define CI_CATE_MASK ((1u << CI_CATE_BITS) - 1)
#define CI_BASE_BITS 8
static inline uint32_t ci_cate_idset(uint32_t ci) { return ci & CI_CATE_MASK; }                     /* :72-74 */
static inline uint32_t ci_base_id(uint32_t ci) { return (ci >> CI_CATE_BITS) & 0xFF; }              /* :77-79 */
static inline int ci_invoke(uint32_t ci) { return (ci >> (CI_CATE_BITS + CI_BASE_BITS)) & 1; }      /* :82-84 */
static inline int ci_group(uint32_t ci) { return (ci >> (CI_CATE_BITS + CI_BASE_BITS + 1)) & 1; }   /* :87-89 */
static inline uint32_t ci_length(uint32_t ci) { return ci >> (CI_CATE_BITS + CI_BASE_BITS + 2); }   /* :92-94 */

/* ------------------------------------------------------------------------------------------ */
/* data model                                                                                  */
/* ------------------------------------------------------------------------------------------ */

#define DA_MASK 0x7FFFFFFFu
#define DA_FLAG 0x80000000u
#define CODE_INVALID 0xFFFFFFFFu

typedef struct {
    uint32_t base;  /* low 31 bits: xor-base, or the value when MSB (is_leaf) is set */
    uint32_t check; /* low 31 bits: parent index; MSB: has_leaf (terminal child at base^0) */
} da_node;

typedef struct {
    uint32_t *table; /* code point -> dense code (>=1), CODE_INVALID when unmapped */
    uint32_t table_len;
    uint32_t alphabet; /* number of codes incl. the reserved terminator code 0 */
    da_node *nodes;
    uint32_t num_nodes;
} trie_t;

typedef struct {
    uint16_t left_id, right_id;
    int16_t word_cost;
} word_param; /* lexicon/param.rs:6-10 */

typedef struct {
    trie_t trie;
    uint32_t *postings; /* lexicon/map/posting.rs:7-21: [len, id...]* */
    size_t n_postings;
    word_param *params; /* lexicon/param.rs:24-41 */
    char *feat_blob;    /* lexicon/feature.rs:4-25 */
    uint64_t *feat_off; /* n_words + 1 */
    uint32_t n_words;
    int lex_type;
} lexicon_t;

typedef struct {
    uint16_t cate_id, left_id, right_id;
    int16_t word_cost;
    char *feature;
    size_t feature_len;
} unk_entry; /* unknown.rs:21-27 */

struct vo_dict {
    lexicon_t sys;
    lexicon_t *user; /* dictionary.rs:43-51 user_lexicon: Option<Lexicon> */
    int16_t *matrix; /* matrix_connector.rs:11-15; NULL for a Raw connector */
    uint32_t num_right, num_left;
    /* RawConnector (raw_connector.rs:22-27): feature-id rows of feat_T ids per connection id + Scorer */
    uint32_t *right_feats, *left_feats;
    uint32_t feat_T;
    uint32_t *sc_bases, *sc_checks;
    int32_t *sc_costs;
    uint32_t n_bases, n_checks;
    /* DualConnector (dual_connector.rs:15-23): `matrix` is the reduced matrix [m_num_left][m_num_right], the maps
     * take a connection id to its column / row of it, and the raw fields above (feat_T == 8) hold the 8-lane term */
    uint16_t *dual_rmap, *dual_lmap;
    uint32_t m_num_right, m_num_left;
    uint32_t *chr2inf; /* character.rs:105-108 */
    uint32_t chr2inf_len;
    char **categories;
    uint32_t n_categories;
    uint32_t *unk_offsets; /* unknown.rs:63-66 */
    unk_entry *unk_entries;
    uint32_t n_unk;
    uint16_t *map_left, *map_right; /* dictionary.rs:48 mapper: Option<ConnIdMapper> (mapper.rs:9-12) */
};

/* ------------------------------------------------------------------------------------------ */
/* CSV parsing (dictionary/lexicon.rs:111-200 over csv-core 0.1.10's field reader)             */
/* ------------------------------------------------------------------------------------------ */

typedef struct {
    char *surface; /* unescaped first field (lexicon.rs:144) */
    size_t surface_len;
    word_param param;
    const char *feature; /* raw slice after the 4th field (lexicon.rs:155-156,178) */
    size_t feature_len;
} raw_entry;

typedef struct {
    raw_entry *v;
    size_t n, cap;
} raw_entries;

static void raw_entries_free(raw_entries *e) {
    for (size_t i = 0; i < e->n; i++) free(e->v[i].surface);
    free(e->v);
    e->v = NULL;
    e->n = e->cap = 0;
}

/* Rust's <u16 as FromStr>/<i16 as FromStr>: optional sign ('+', and '-' for signed), >=1 digit,
 * nothing else, range-checked. */
static int parse_int_strict(const char *s, size_t n, long lo, long hi, long *out) {
    size_t i = 0;
    int neg = 0;
    if (n == 0) return 0;
    if (s[0] == '+') {
        i = 1;
    } else if (s[0] == '-') {
        if (lo >= 0) return 0; /* unsigned types reject '-' */
        neg = 1;
        i = 1;
    }
    if (i >= n) return 0;
    long v = 0;
    for (; i < n; i++) {
        if (s[i] < '0' || s[i] > '9') return 0;
        if (v > (0x7FFFFFFFFFFFFFFFL - 9) / 10) return 0; /* beyond every integer type this parser serves */
        v = v * 10 + (s[i] - '0');
    }
    if (neg) v = -v;
    if (v < lo || v > hi) return 0;
    *out = v;
    return 1;
}

#define CSV_FIELD_MAX 4096 /* lexicon.rs:124 `output = [0; 4096]` -> "Field too large" :138-140 */

/*
 * One csv-core field: RFC-4180-style, delimiter ',', quote '"' with "" escaping, record
 * terminators \n, \r and \r\n, blank lines skipped.  Returns the unescaped field in out[0..*nout),
 * advances *pos past the field and its delimiter / terminator; *rec_end says whether the record
 * ended; *at_eof says the input was exhausted inside the field (csv-core's InputEmpty).
 * Returns 0 when no more records (End), 1 for a field, -1 for "Field too large".
 */
static int csv_read_field(const char *b, size_t len, size_t *pos, int *start_of_record, char *out, size_t *nout,
                          int *rec_end, int *at_eof) {
    size_t i = *pos;
    *nout = 0;
    *rec_end = 0;
    *at_eof = 0;
    if (*start_of_record) {
        /* StartRecord: swallow record terminators (blank lines; also the '\n' of a "\r\n"). */
        while (i < len && (b[i] == '\n' || b[i] == '\r')) i++;
        if (i >= len) {
            *pos = i;
            return 0;
        }
        *start_of_record = 0;
    } else if (i >= len) {
        /* EOF directly after a delimiter: csv-core flushes one empty final field. */
        *pos = i;
        *rec_end = 1;
        *start_of_record = 1;
        return 1;
    }
    int quoted = 0, after_quote = 0;
    if (b[i] == '"') {
        quoted = 1;
        i++;
    }
    for (;;) {
        if (i >= len) {
            *at_eof = 1;
            *rec_end = 1;
            *start_of_record = 1;
            *pos = i;
            return 1;
        }
        char c = b[i];
        if (quoted && !after_quote) {
            if (c == '"') {
                after_quote = 1; /* InDoubleEscapedQuote */
                i++;
                continue;
            }
        } else {
            if (after_quote && c == '"') { /* "" -> literal quote, back in the quoted field */
                after_quote = 0;
                if (*nout >= CSV_FIELD_MAX) return -1;
                out[(*nout)++] = '"';
                i++;
                continue;
            }
            if (c == ',') {
                *pos = i + 1;
                return 1;
            }
            if (c == '\n' || c == '\r') {
                *pos = i + 1; /* a following '\n' of "\r\n" is swallowed at the next StartRecord */
                *rec_end = 1;
                *start_of_record = 1;
                return 1;
            }
            if (after_quote) { /* junk after a closing quote: continue as an unquoted field */
                quoted = 0;
                after_quote = 0;
            }
        }
        if (*nout >= CSV_FIELD_MAX) return -1;
        out[(*nout)++] = c;
        i++;
    }
}

/* Lexicon::parse_csv (lexicon.rs:111-200). `name` is used in messages only. */
static int parse_csv(const char *bytes, size_t len, const char *name, raw_entries *entries, char *err, size_t errcap) {
    size_t pos = 0;
    int start_of_record = 1;
    char out[CSV_FIELD_MAX + 8];
    size_t nout;
    int rec_end, at_eof;
    size_t field_cnt = 0;
    char *surface = NULL;
    size_t surface_len = 0;
    long left = 0, right = 0, cost = 0;
    size_t feat_start = 0;
    memset(entries, 0, sizeof(*entries));

    for (;;) {
        size_t before = pos;
        int r = csv_read_field(bytes, len, &pos, &start_of_record, out, &nout, &rec_end, &at_eof);
        if (r == 0) break;
        if (r < 0) {
            set_err(err, errcap, "InvalidFormat(%s): Field too large", name);
            goto fail;
        }
        /* lexicon.rs:170: a flushed empty field at EOF when nothing of a record was read */
        if (rec_end && field_cnt == 0 && pos == before) continue;
        if (at_eof && field_cnt <= 3) {
            /* lexicon.rs:133-137 + :171-177: the partial field is not counted -> too few items */
            set_err(err, errcap, "InvalidFormat(%s): A csv row of lexicon must have five items at least", name);
            goto fail;
        }
        switch (at_eof ? 99 : field_cnt) {
        case 0:
            free(surface);
            surface = (char *)xmalloc(nout + 1);
            memcpy(surface, out, nout);
            surface[nout] = 0;
            surface_len = nout;
            if (!vo_utf8_valid(surface, surface_len)) {
                set_err(err, errcap, "Utf8(%s): invalid utf-8 in surface", name);
                goto fail;
            }
            break;
        case 1:
            if (!parse_int_strict(out, nout, 0, 65535, &left)) {
                set_err(err, errcap, "ParseInt(%s): invalid left_id", name);
                goto fail;
            }
            break;
        case 2:
            if (!parse_int_strict(out, nout, 0, 65535, &right)) {
                set_err(err, errcap, "ParseInt(%s): invalid right_id", name);
                goto fail;
            }
            break;
        case 3:
            if (!parse_int_strict(out, nout, -32768, 32767, &cost)) {
                set_err(err, errcap, "ParseInt(%s): invalid word_cost", name);
                goto fail;
            }
            feat_start = pos; /* lexicon.rs:155: features_bytes = &bytes[nin..] */
            break;
        default:
            break;
        }
        if (rec_end) {
            if (field_cnt <= 3) { /* lexicon.rs:171-177 */
                set_err(err, errcap, "InvalidFormat(%s): A csv row of lexicon must have five items at least", name);
                goto fail;
            }
            /* lexicon.rs:178: raw bytes up to, not including, the record terminator */
            size_t feat_end = at_eof ? pos : pos - 1;
            if (feat_end < feat_start) { /* "a,1,2,3," at EOF: the reference panics here */
                set_err(err, errcap, "InvalidFormat(%s): truncated final record", name);
                goto fail;
            }
            if (!vo_utf8_valid(bytes + feat_start, feat_end - feat_start)) {
                set_err(err, errcap, "Utf8(%s): invalid utf-8 in feature", name);
                goto fail;
            }
            if (surface_len == 0) {
                /* lexicon.rs:179-183: "Skipped an empty surface" */
            } else {
                if (entries->n == entries->cap) {
                    entries->cap = entries->cap ? entries->cap * 2 : 1024;
                    entries->v = (raw_entry *)xrealloc(entries->v, entries->cap * sizeof(raw_entry));
                }
                raw_entry *e = &entries->v[entries->n++];
                e->surface = surface;
                e->surface_len = surface_len;
                e->param.left_id = (uint16_t)left;
                e->param.right_id = (uint16_t)right;
                e->param.word_cost = (int16_t)cost;
                e->feature = bytes + feat_start;
                e->feature_len = feat_end - feat_start;
                surface = NULL;
            }
            free(surface);
            surface = NULL;
            surface_len = 0;
            field_cnt = 0;
        } else {
            field_cnt++;
        }
    }
    free(surface);
    return 0;
fail:
    free(surface);
    raw_entries_free(entries);
    return -1;
}

/* ------------------------------------------------------------------------------------------ */
/* double-array trie (behaviour of crawdad 0.3 `Trie`; call sites lexicon/map/trie.rs:39-56)   */
/* ------------------------------------------------------------------------------------------ */

typedef struct {
    uint32_t *cps; /* key as code points */
    uint32_t len;
    uint32_t value;
} trie_key;

typedef struct {
    da_node *nodes;
    uint32_t *prev, *next; /* circular free list over vacant slots */
    uint32_t size, cap;
    uint32_t free_head; /* UINT32_MAX when none */
    uint32_t block;     /* power of two > every code */
} da_builder;

#define NIL 0xFFFFFFFFu

static void dab_grow(da_builder *b) {
    uint32_t old = b->size, nsz = old + b->block;
    if (nsz > b->cap) {
        uint32_t ncap = b->cap ? b->cap : b->block;
        while (ncap < nsz) ncap *= 2;
        b->nodes = (da_node *)xrealloc(b->nodes, (size_t)ncap * sizeof(da_node));
        b->prev = (uint32_t *)xrealloc(b->prev, (size_t)ncap * sizeof(uint32_t));
        b->next = (uint32_t *)xrealloc(b->next, (size_t)ncap * sizeof(uint32_t));
        b->cap = ncap;
    }
    for (uint32_t i = old; i < nsz; i++) {
        b->nodes[i].base = DA_MASK;
        b->nodes[i].check = DA_MASK;
        b->prev[i] = i - 1;
        b->next[i] = i + 1;
    }
    /* splice [old, nsz) at the tail of the circular list */
    if (b->free_head == NIL) {
        b->free_head = old;
        b->prev[old] = nsz - 1;
        b->next[nsz - 1] = old;
    } else {
        uint32_t tail = b->prev[b->free_head];
        b->next[tail] = old;
        b->prev[old] = tail;
        b->next[nsz - 1] = b->free_head;
        b->prev[b->free_head] = nsz - 1;
    }
    b->size = nsz;
}

static inline int dab_vacant(const da_builder *b, uint32_t i) {
    return b->nodes[i].base == DA_MASK && b->nodes[i].check == DA_MASK;
}

static void dab_take(da_builder *b, uint32_t i) {
    uint32_t p = b->prev[i], n = b->next[i];
    if (n == i) {
        b->free_head = NIL;
    } else {
        b->next[p] = n;
        b->prev[n] = p;
        if (b->free_head == i) b->free_head = n;
    }
}

/* Finds a base such that base^codes[j] is vacant for every j. */
static uint32_t dab_find_base(da_builder *b, const uint32_t *codes, uint32_t k) {
    if (b->free_head != NIL) {
        if (k == 1) return b->free_head ^ codes[0];
        /* newest slots first: they sit in the emptiest blocks */
        uint32_t s = b->prev[b->free_head];
        for (int tries = 0; tries < 512; tries++) {
            uint32_t base = s ^ codes[0];
            uint32_t j = 1;
            for (; j < k; j++)
                if (!dab_vacant(b, base ^ codes[j])) break;
            if (j == k) return base;
            if (s == b->free_head) break;
            s = b->prev[s];
        }
    }
    uint32_t base = b->size; /* fresh block: every base^code lands inside it */
    dab_grow(b);
    return base;
}

typedef struct {
    uint32_t node, lo, hi, depth;
} da_frame;

/* keys must be sorted by code-point sequence and unique. */
static void trie_build(trie_t *t, const trie_key *keys, uint32_t n_keys) {
    memset(t, 0, sizeof(*t));
    /* code mapper: dense codes by descending frequency, 0 reserved for the terminator */
    uint32_t max_cp = 0;
    for (uint32_t i = 0; i < n_keys; i++)
        for (uint32_t j = 0; j < keys[i].len; j++)
            if (keys[i].cps[j] > max_cp) max_cp = keys[i].cps[j];
    t->table_len = n_keys ? max_cp + 1 : 0;
    t->table = (uint32_t *)xmalloc((size_t)t->table_len * sizeof(uint32_t));
    uint32_t *freq = (uint32_t *)xcalloc(t->table_len ? t->table_len : 1, sizeof(uint32_t));
    for (uint32_t i = 0; i < n_keys; i++)
        for (uint32_t j = 0; j < keys[i].len; j++) freq[keys[i].cps[j]]++;
    uint32_t n_used = 0;
    for (uint32_t c = 0; c < t->table_len; c++)
        if (freq[c]) n_used++;
    uint64_t *order = (uint64_t *)xmalloc((size_t)(n_used ? n_used : 1) * sizeof(uint64_t));
    uint32_t k = 0;
    for (uint32_t c = 0; c < t->table_len; c++)
        if (freq[c]) order[k++] = ((uint64_t)(0xFFFFFFFFu - freq[c]) << 32) | c;
    /* ascending on (inverted freq, cp) == descending freq */
    for (uint32_t gap = n_used / 2; gap > 0; gap /= 2) /* shell sort: n_used is at most a few 10^4 */
        for (uint32_t i = gap; i < n_used; i++) {
            uint64_t v = order[i];
            uint32_t j = i;
            for (; j >= gap && order[j - gap] > v; j -= gap) order[j] = order[j - gap];
            order[j] = v;
        }
    for (uint32_t c = 0; c < t->table_len; c++) t->table[c] = CODE_INVALID;
    for (uint32_t i = 0; i < n_used; i++) t->table[(uint32_t)order[i]] = i + 1;
    t->alphabet = n_used + 1;
    free(order);
    free(freq);

    da_builder b;
    memset(&b, 0, sizeof(b));
    b.free_head = NIL;
    b.block = 1;
    while (b.block < t->alphabet) b.block <<= 1;
    if (b.block < 256) b.block = 256;
    dab_grow(&b);
    dab_take(&b, 0); /* root */
    b.nodes[0].base = 0;
    b.nodes[0].check = DA_MASK;

    size_t stack_cap = 1024, sp = 0;
    da_frame *stack = (da_frame *)xmalloc(stack_cap * sizeof(da_frame));
    uint32_t *codes = (uint32_t *)xmalloc((size_t)t->alphabet * sizeof(uint32_t));
    uint32_t *los = (uint32_t *)xmalloc((size_t)(t->alphabet + 1) * sizeof(uint32_t));
    if (n_keys) stack[sp++] = (da_frame){0, 0, n_keys, 0};
    while (sp) {
        da_frame f = stack[--sp];
        uint32_t lo = f.lo;
        int terminal = 0;
        uint32_t tvalue = 0;
        if (keys[lo].len == f.depth) {
            terminal = 1;
            tvalue = keys[lo].value;
            lo++;
        }
        if (lo == f.hi) { /* nothing continues: the node itself is the leaf */
            b.nodes[f.node].base = DA_FLAG | tvalue;
            continue;
        }
        uint32_t nc = 0;
        if (terminal) {
            codes[nc] = 0;
            los[nc] = lo;
            nc++;
        }
        for (uint32_t i = lo; i < f.hi;) {
            uint32_t cp = keys[i].cps[f.depth];
            uint32_t j = i + 1;
            while (j < f.hi && keys[j].cps[f.depth] == cp) j++;
            codes[nc] = t->table[cp];
            los[nc] = i;
            nc++;
            i = j;
        }
        los[nc] = f.hi;
        uint32_t base = dab_find_base(&b, codes, nc);
        b.nodes[f.node].base = base; /* MSB clear: not a leaf */
        if (terminal) b.nodes[f.node].check |= DA_FLAG;
        for (uint32_t c = 0; c < nc; c++) {
            uint32_t child = base ^ codes[c];
            dab_take(&b, child);
            b.nodes[child].check = f.node;
            if (terminal && c == 0) {
                b.nodes[child].base = DA_FLAG | tvalue;
                continue;
            }
            b.nodes[child].base = 0;
            if (sp == stack_cap) {
                stack_cap *= 2;
                stack = (da_frame *)xrealloc(stack, stack_cap * sizeof(da_frame));
            }
            stack[sp++] = (da_frame){child, los[c], los[c + 1], f.depth + 1};
        }
    }
    free(stack);
    free(codes);
    free(los);
    free(b.prev);
    free(b.next);
    t->nodes = b.nodes;
    t->num_nodes = b.size;
}

static void trie_free(trie_t *t) {
    free(t->table);
    free(t->nodes);
    memset(t, 0, sizeof(*t));
}

/* ------------------------------------------------------------------------------------------ */
/* Lexicon (dictionary/lexicon.rs, lexicon/map.rs, lexicon/map/posting.rs)                     */
/* ------------------------------------------------------------------------------------------ */

typedef struct {
    const raw_entry *e;
    uint32_t id;
} sort_item;

static int sort_item_cmp(const void *a_, const void *b_) {
    const sort_item *a = (const sort_item *)a_, *b = (const sort_item *)b_;
    size_t n = a->e->surface_len < b->e->surface_len ? a->e->surface_len : b->e->surface_len;
    int c = memcmp(a->e->surface, b->e->surface, n);
    if (c) return c;
    if (a->e->surface_len != b->e->surface_len) return a->e->surface_len < b->e->surface_len ? -1 : 1;
    return a->id < b->id ? -1 : (a->id > b->id ? 1 : 0); /* ids pushed in input order, map.rs:26-28,57-59 */
}

/* Lexicon::from_entries (lexicon.rs:85-96) -> WordMap::new / WordMapBuilder::build (map.rs:20-73). */
static void lexicon_build(lexicon_t *lx, const raw_entries *ents, int lex_type) {
    memset(lx, 0, sizeof(*lx));
    lx->lex_type = lex_type;
    uint32_t n = (uint32_t)ents->n;
    lx->n_words = n;
    lx->params = (word_param *)xmalloc((size_t)n * sizeof(word_param));
    lx->feat_off = (uint64_t *)xmalloc((size_t)(n + 1) * sizeof(uint64_t));
    size_t total = 0;
    for (uint32_t i = 0; i < n; i++) total += ents->v[i].feature_len;
    lx->feat_blob = (char *)xmalloc(total + 1);
    total = 0;
    for (uint32_t i = 0; i < n; i++) {
        lx->params[i] = ents->v[i].param;
        lx->feat_off[i] = total;
        memcpy(lx->feat_blob + total, ents->v[i].feature, ents->v[i].feature_len);
        total += ents->v[i].feature_len;
    }
    lx->feat_off[n] = total;

    /* BTreeMap<String, Vec<u32>> in key order (map.rs:46-73) */
    sort_item *items = (sort_item *)xmalloc((size_t)(n ? n : 1) * sizeof(sort_item));
    for (uint32_t i = 0; i < n; i++) items[i] = (sort_item){&ents->v[i], i};
    qsort(items, n, sizeof(sort_item), sort_item_cmp);
    lx->postings = (uint32_t *)xmalloc(((size_t)2 * n + 1) * sizeof(uint32_t));
    trie_key *keys = (trie_key *)xmalloc((size_t)(n ? n : 1) * sizeof(trie_key));
    uint32_t n_keys = 0;
    size_t np = 0;
    for (uint32_t i = 0; i < n;) {
        uint32_t j = i + 1;
        while (j < n && items[j].e->surface_len == items[i].e->surface_len &&
               memcmp(items[j].e->surface, items[i].e->surface, items[i].e->surface_len) == 0)
            j++;
        uint32_t offset = (uint32_t)np; /* PostingsBuilder::push, posting.rs:33-38 */
        lx->postings[np++] = j - i;
        for (uint32_t q = i; q < j; q++) lx->postings[np++] = items[q].id;
        const raw_entry *e = items[i].e;
        trie_key *key = &keys[n_keys++];
        key->cps = (uint32_t *)xmalloc((e->surface_len + 1) * sizeof(uint32_t));
        key->len = 0;
        for (size_t p = 0; p < e->surface_len;) {
            uint32_t cp;
            p += utf8_decode((const unsigned char *)e->surface + p, &cp);
            key->cps[key->len++] = cp;
        }
        key->value = offset;
        i = j;
    }
    lx->n_postings = np;
    trie_build(&lx->trie, keys, n_keys); /* byte-wise order of UTF-8 == code-point order */
    for (uint32_t i = 0; i < n_keys; i++) free(keys[i].cps);
    free(keys);
    free(items);
}

static void lexicon_free(lexicon_t *lx) {
    trie_free(&lx->trie);
    free(lx->postings);
    free(lx->params);
    free(lx->feat_blob);
    free(lx->feat_off);
    memset(lx, 0, sizeof(*lx));
}

/* Lexicon::verify (lexicon.rs:68-82) */
static int lexicon_verify(const lexicon_t *lx, uint32_t num_left, uint32_t num_right) {
    for (uint32_t i = 0; i < lx->n_words; i++) {
        if (num_left <= lx->params[i].left_id) return 0;
        if (num_right <= lx->params[i].right_id) return 0;
    }
    return 1;
}

/* ------------------------------------------------------------------------------------------ */
/* matrix.def (connector/matrix_connector.rs:27-77)                                            */
/* ------------------------------------------------------------------------------------------ */

/* BufRead::lines(): split on '\n', strip one trailing '\r'. Returns 0 at end. */
static int next_line(const char *b, size_t len, size_t *pos, const char **line, size_t *n) {
    if (*pos >= len) return 0;
    size_t s = *pos, e = s;
    while (e < len && b[e] != '\n') e++;
    *pos = e < len ? e + 1 : e;
    if (e > s && b[e - 1] == '\r' && e < len) e--; /* "\r\n" only; a lone trailing '\r' at EOF stays */
    *line = b + s;
    *n = e - s;
    return 1;
}

static size_t split_char(const char *s, size_t n, char sep, const char **tok, size_t *tlen, size_t cap) {
    size_t cnt = 0, st = 0;
    for (size_t i = 0; i <= n; i++) {
        if (i == n || s[i] == sep) {
            if (cnt < cap) {
                tok[cnt] = s + st;
                tlen[cnt] = i - st;
            }
            cnt++;
            st = i + 1;
        }
    }
    return cnt;
}

static int matrix_from_text(vo_dict *d, const char *b, size_t len, char *err, size_t errcap) {
    size_t pos = 0, n;
    const char *line;
    const char *tok[4];
    size_t tl[4];
    if (!next_line(b, len, &pos, &line, &n)) { /* `lines.next().unwrap()` panics in the reference */
        set_err(err, errcap, "InvalidFormat(matrix.def): empty input");
        return -1;
    }
    long nr, nl; /* parse_header :53-64: exactly two columns separated by one space, each a u16 */
    if (split_char(line, n, ' ', tok, tl, 4) != 2) {
        set_err(err, errcap, "InvalidFormat(matrix.def): The header must consists of two integers separated by spaces");
        return -1;
    }
    if (!parse_int_strict(tok[0], tl[0], 0, 65535, &nr) || !parse_int_strict(tok[1], tl[1], 0, 65535, &nl)) {
        set_err(err, errcap, "ParseInt(matrix.def): the header holds something that is not a u16"); /* `.parse()?` :60-61 */
        return -1;
    }
    d->num_right = (uint32_t)nr;
    d->num_left = (uint32_t)nl;
    d->matrix = (int16_t *)xcalloc((size_t)nr * (size_t)nl, sizeof(int16_t));
    while (next_line(b, len, &pos, &line, &n)) {
        if (n == 0) continue; /* :38 */
        long r, l, c;         /* parse_body :66-77: three columns, then usize, usize, i16 */
        if (split_char(line, n, ' ', tok, tl, 4) != 3) {
            set_err(err, errcap, "InvalidFormat(matrix.def): A row other than the header must consists of three integers");
            return -1;
        }
        if (!parse_int_strict(tok[0], tl[0], 0, 0x7FFFFFFFFFFFFFFFL, &r) || !parse_int_strict(tok[1], tl[1], 0, 0x7FFFFFFFFFFFFFFFL, &l) ||
            !parse_int_strict(tok[2], tl[2], -32768, 32767, &c)) {
            set_err(err, errcap, "ParseInt(matrix.def): a row holds something that is not an integer of its type"); /* :75 */
            return -1;
        }
        if (nr <= r || nl <= l) { /* :40-45 */
            set_err(err, errcap, "InvalidFormat(matrix.def): left/right_id must be within num_left/right.");
            return -1;
        }
        d->matrix[(size_t)l * (size_t)nr + (size_t)r] = (int16_t)c; /* :47 */
    }
    return 0;
}

/* ------------------------------------------------------------------------------------------ */
/* char.def (dictionary/character.rs:140-281)                                                  */
/* ------------------------------------------------------------------------------------------ */

static int is_ws(unsigned char c) { return c == ' ' || c == '\t' || c == '\n' || c == '\v' || c == '\f' || c == '\r'; }

static size_t split_ws(const char *s, size_t n, const char **tok, size_t *tlen, size_t cap) {
    size_t cnt = 0, i = 0;
    while (i < n) {
        while (i < n && is_ws((unsigned char)s[i])) i++;
        if (i >= n) break;
        size_t st = i;
        while (i < n && !is_ws((unsigned char)s[i])) i++;
        if (cnt < cap) {
            tok[cnt] = s + st;
            tlen[cnt] = i - st;
        }
        cnt++;
    }
    return cnt;
}

static int find_category(const vo_dict *d, const char *name, size_t n) { /* character.rs:119-124 */
    for (uint32_t i = 0; i < d->n_categories; i++)
        if (strlen(d->categories[i]) == n && memcmp(d->categories[i], name, n) == 0) return (int)i;
    return -1;
}

static int add_category(vo_dict *d, const char *name, size_t n) {
    d->categories = (char **)xrealloc(d->categories, (size_t)(d->n_categories + 1) * sizeof(char *));
    char *s = (char *)xmalloc(n + 1);
    memcpy(s, name, n);
    s[n] = 0;
    d->categories[d->n_categories] = s;
    return (int)d->n_categories++;
}

static int parse_hex(const char *s, size_t n, unsigned long *out) {
    while (n >= 2 && s[0] == '0' && s[1] == 'x') { /* trim_start_matches("0x") :255 */
        s += 2;
        n -= 2;
    }
    if (n && s[0] == '+') { /* usize::from_str_radix takes an optional plus sign */
        s++;
        n--;
    }
    if (n == 0) return 0;
    unsigned long v = 0;
    for (size_t i = 0; i < n; i++) {
        char c = s[i];
        int dgt = (c >= '0' && c <= '9') ? c - '0' : (c >= 'a' && c <= 'f') ? c - 'a' + 10 : (c >= 'A' && c <= 'F') ? c - 'A' + 10 : -1;
        if (dgt < 0) return 0;
        if (v >> 60) return 0; /* would not fit a 64-bit usize */
        v = v * 16 + (unsigned long)dgt;
    }
    *out = v;
    return 1;
}

#define MAX_RANGE_CATS 32
typedef struct {
    uint32_t start, end; /* [start, end) */
    int cats[MAX_RANGE_CATS];
    int n_cats;
} char_range;

/* encode_cate_info (character.rs:193-216); cate_info[id] = CharInfo::new(0,id,invoke,group,length) or 0 w/ defined=0 */
static int encode_cate_info(const int *cats, int n, const uint32_t *cate_info, const uint8_t *defined, uint32_t *out) {
    if (n == 0 || cats[0] < 0 || !defined[cats[0]]) return 0;
    uint32_t base = cate_info[cats[0]];
    uint32_t idset = ci_cate_idset(base);
    for (int i = 0; i < n; i++) {
        if (cats[i] < 0 || !defined[cats[i]]) return 0; /* `.unwrap()` panics in the reference */
        idset |= 1u << (ci_base_id(cate_info[cats[i]]) & 31); /* release-build `1 << id`: the shift wraps at 32 */
    }
    *out = (base & ~CI_CATE_MASK) | idset; /* reset_cate_idset :66-69: OR-ed unchecked */
    return 1;
}

static int char_prop_from_text(vo_dict *d, const char *b, size_t len, char *err, size_t errcap) {
    uint32_t cate_info[256];
    uint8_t defined[256];
    memset(defined, 0, sizeof(defined));
    memset(cate_info, 0, sizeof(cate_info));
    char_range *ranges = NULL;
    size_t n_ranges = 0, cap_ranges = 0;
    add_category(d, "DEFAULT", 7); /* :148 */

    size_t pos = 0, n;
    const char *line;
    int rc = -1;
    while (next_line(b, len, &pos, &line, &n)) {
        while (n && is_ws((unsigned char)line[0])) { /* trim :152 (ASCII whitespace) */
            line++;
            n--;
        }
        while (n && is_ws((unsigned char)line[n - 1])) n--;
        if (n == 0 || line[0] == '#') continue;
        const char *tok[MAX_RANGE_CATS + 2];
        size_t tl[MAX_RANGE_CATS + 2];
        size_t nt = split_ws(line, n, tok, tl, MAX_RANGE_CATS + 2);
        if (!(n >= 2 && line[0] == '0' && line[1] == 'x')) {
            /* parse_char_category :218-244 */
            if (nt < 4) {
                set_err(err, errcap, "InvalidFormat(char.def): A character category must consists of four items separated by spaces");
                goto done;
            }
            int invoke, group;
            long length;
            if (tl[1] == 1 && (tok[1][0] == '0' || tok[1][0] == '1')) {
                invoke = tok[1][0] == '1';
            } else {
                set_err(err, errcap, "InvalidFormat(char.def): INVOKE must be 1 or 0.");
                goto done;
            }
            if (tl[2] == 1 && (tok[2][0] == '0' || tok[2][0] == '1')) {
                group = tok[2][0] == '1';
            } else {
                set_err(err, errcap, "InvalidFormat(char.def): GROUP must be 1 or 0.");
                goto done;
            }
            if (!parse_int_strict(tok[3], tl[3], 0, 65535, &length)) {
                set_err(err, errcap, "ParseInt(char.def): invalid LENGTH");
                goto done;
            }
            int id = find_category(d, tok[0], tl[0]); /* :161-162 first-seen order */
            if (id < 0) id = add_category(d, tok[0], tl[0]);
            if (id >= 256 || length >= 16) { /* CharInfo::new(...).unwrap() :165 panics */
                set_err(err, errcap, "InvalidFormat(char.def): category id/length out of range");
                goto done;
            }
            cate_info[id] = ((uint32_t)id << CI_CATE_BITS) | ((uint32_t)invoke << (CI_CATE_BITS + CI_BASE_BITS)) |
                            ((uint32_t)group << (CI_CATE_BITS + CI_BASE_BITS + 1)) |
                            ((uint32_t)length << (CI_CATE_BITS + CI_BASE_BITS + 2));
            defined[id] = 1;
        } else {
            /* parse_char_range :246-281 */
            if (nt < 2) {
                set_err(err, errcap, "InvalidFormat(char.def): A character range must have two items at least");
                goto done;
            }
            const char *dots = NULL;
            for (size_t i = 0; i + 1 < tl[0]; i++)
                if (tok[0][i] == '.' && tok[0][i + 1] == '.') {
                    dots = tok[0] + i;
                    break;
                }
            unsigned long start, end;
            if (dots) {
                const char *rhs = dots + 2;
                size_t rn = tl[0] - (size_t)(rhs - tok[0]);
                const char *d2 = NULL; /* split("..") may yield >2 parts; only r[1] is used */
                for (size_t i = 0; i + 1 < rn; i++)
                    if (rhs[i] == '.' && rhs[i + 1] == '.') {
                        d2 = rhs + i;
                        break;
                    }
                if (d2) rn = (size_t)(d2 - rhs);
                if (!parse_hex(tok[0], (size_t)(dots - tok[0]), &start) || !parse_hex(rhs, rn, &end)) {
                    set_err(err, errcap, "ParseInt(char.def): invalid range");
                    goto done;
                }
                end += 1;
            } else {
                if (!parse_hex(tok[0], tl[0], &start)) {
                    set_err(err, errcap, "ParseInt(char.def): invalid range");
                    goto done;
                }
                end = start + 1;
            }
            if (start >= end) {
                set_err(err, errcap, "InvalidFormat(char.def): The start of a character range must be no more than the end");
                goto done;
            }
            if (start > 0xFFFF || end > 0x10000) {
                set_err(err, errcap, "InvalidFormat(char.def): A character range must be no more 0xFFFF");
                goto done;
            }
            if (n_ranges == cap_ranges) {
                cap_ranges = cap_ranges ? cap_ranges * 2 : 64;
                ranges = (char_range *)xrealloc(ranges, cap_ranges * sizeof(char_range));
            }
            char_range *r = &ranges[n_ranges++];
            r->start = (uint32_t)start;
            r->end = (uint32_t)end;
            r->n_cats = 0;
            for (size_t i = 1; i < nt && i < MAX_RANGE_CATS + 1; i++) {
                if (tok[i][0] == '#') break; /* :270 take_while(!starts_with('#')) */
                /* names are resolved after the whole file is read (:175-180); stash token index */
                r->cats[r->n_cats++] = -2 - (int)(tok[i] - b);
                (void)tl;
            }
            /* remember lengths by re-splitting later: store pointer offsets only */
        }
    }
    {
        int dflt = 0;
        uint32_t init;
        if (!encode_cate_info(&dflt, 1, cate_info, defined, &init)) { /* :172 */
            set_err(err, errcap, "InvalidFormat(char.def): Undefined category: DEFAULT");
            goto done;
        }
        d->chr2inf_len = 1u << 16; /* :173 */
        d->chr2inf = (uint32_t *)xmalloc((size_t)d->chr2inf_len * sizeof(uint32_t));
        for (uint32_t i = 0; i < d->chr2inf_len; i++) d->chr2inf[i] = init;
        for (size_t ri = 0; ri < n_ranges; ri++) {
            char_range *r = &ranges[ri];
            int cats[MAX_RANGE_CATS];
            for (int i = 0; i < r->n_cats; i++) {
                const char *nm = b + (size_t)(-2 - r->cats[i]);
                size_t nl = 0;
                while (nm + nl < b + len && !is_ws((unsigned char)nm[nl])) nl++;
                cats[i] = find_category(d, nm, nl);
            }
            uint32_t ci;
            if (!encode_cate_info(cats, r->n_cats, cate_info, defined, &ci)) {
                set_err(err, errcap, "InvalidFormat(char.def): Undefined category in a range line");
                goto done;
            }
            for (uint32_t c = r->start; c < r->end; c++) d->chr2inf[c] = ci; /* :176-179 later lines overwrite */
        }
    }
    rc = 0;
done:
    free(ranges);
    return rc;
}

/* ------------------------------------------------------------------------------------------ */
/* unk.def (dictionary/unknown.rs:230-263)                                                     */
/* ------------------------------------------------------------------------------------------ */

static int unk_from_text(vo_dict *d, const char *b, size_t len, char *err, size_t errcap) {
    raw_entries ents;
    if (parse_csv(b, len, "unk.def", &ents, err, errcap) != 0) return -1;
    uint32_t nc = d->n_categories;
    uint32_t *counts = (uint32_t *)xcalloc(nc + 1, sizeof(uint32_t));
    int *cate = (int *)xmalloc((ents.n ? ents.n : 1) * sizeof(int));
    for (size_t i = 0; i < ents.n; i++) {
        cate[i] = find_category(d, ents.v[i].surface, ents.v[i].surface_len);
        if (cate[i] < 0) { /* :237-241 */
            set_err(err, errcap, "InvalidFormat(unk.def): Undefined category: %s", ents.v[i].surface);
            free(counts);
            free(cate);
            raw_entries_free(&ents);
            return -1;
        }
        counts[cate[i]]++;
    }
    d->unk_offsets = (uint32_t *)xmalloc((size_t)(nc + 1) * sizeof(uint32_t)); /* :255-262 */
    uint32_t acc = 0;
    for (uint32_t c = 0; c < nc; c++) {
        d->unk_offsets[c] = acc;
        acc += counts[c];
    }
    d->unk_offsets[nc] = acc;
    d->n_unk = acc;
    d->unk_entries = (unk_entry *)xcalloc(acc ? acc : 1, sizeof(unk_entry));
    memset(counts, 0, (nc + 1) * sizeof(uint32_t));
    for (size_t i = 0; i < ents.n; i++) { /* stable within a category */
        unk_entry *e = &d->unk_entries[d->unk_offsets[cate[i]] + counts[cate[i]]++];
        e->cate_id = (uint16_t)cate[i];
        e->left_id = ents.v[i].param.left_id;
        e->right_id = ents.v[i].param.right_id;
        e->word_cost = ents.v[i].param.word_cost;
        e->feature = (char *)xmalloc(ents.v[i].feature_len + 1);
        memcpy(e->feature, ents.v[i].feature, ents.v[i].feature_len);
        e->feature[ents.v[i].feature_len] = 0;
        e->feature_len = ents.v[i].feature_len;
    }
    free(counts);
    free(cate);
    raw_entries_free(&ents);
    return 0;
}

/* ------------------------------------------------------------------------------------------ */
/* Dictionary construction (dictionary/builder.rs:16-89, dictionary.rs:209-229)                */
/* ------------------------------------------------------------------------------------------ */

void vo_dict_free(vo_dict *d) {
    if (!d) return;
    lexicon_free(&d->sys);
    if (d->user) {
        lexicon_free(d->user);
        free(d->user);
    }
    free(d->matrix);
    free(d->dual_rmap);
    free(d->dual_lmap);
    free(d->right_feats);
    free(d->left_feats);
    free(d->sc_bases);
    free(d->sc_checks);
    free(d->sc_costs);
    free(d->chr2inf);
    for (uint32_t i = 0; i < d->n_categories; i++) free(d->categories[i]);
    free(d->categories);
    free(d->unk_offsets);
    for (uint32_t i = 0; i < d->n_unk; i++) free(d->unk_entries[i].feature);
    free(d->unk_entries);
    free(d->map_left);
    free(d->map_right);
    free(d);
}

static vo_dict *dict_finish(vo_dict *d, const char *lex_csv, size_t lex_len, const char *char_def, size_t char_len,
                            const char *unk_def, size_t unk_len, char *err, size_t errcap) {
    raw_entries ents;
    if (parse_csv(lex_csv, lex_len, "lex.csv", &ents, err, errcap) != 0) goto fail; /* builder.rs:79 */
    if (char_prop_from_text(d, char_def, char_len, err, errcap) != 0) {             /* :81 */
        raw_entries_free(&ents);
        goto fail;
    }
    if (unk_from_text(d, unk_def, unk_len, err, errcap) != 0) { /* :82 */
        raw_entries_free(&ents);
        goto fail;
    }
    /* A category id OR-ed past bit 17 (encode_cate_info) can move a base id past the last category, whose unk.def
     * slot the reference would index out of bounds; the device image refuses such a dictionary, and so does this. */
    for (uint32_t c = 0; c < d->chr2inf_len; c++)
        if (ci_base_id(d->chr2inf[c]) >= d->n_categories) {
            set_err(err, errcap, "BincodeDecode: CharInfo base_id has no unk.def slot");
            raw_entries_free(&ents);
            goto fail;
        }
    lexicon_build(&d->sys, &ents, 0); /* builder.rs:22 */
    raw_entries_free(&ents);
    if (!lexicon_verify(&d->sys, d->num_left, d->num_right)) { /* :24-29 */
        set_err(err, errcap, "InvalidArgument(system_lexicon_rdr): system_lexicon_rdr includes invalid connection ids.");
        goto fail;
    }
    for (uint32_t i = 0; i < d->n_unk; i++) /* UnkHandler::verify unknown.rs:213-226, builder.rs:30-35 */
        if (d->num_left <= d->unk_entries[i].left_id || d->num_right <= d->unk_entries[i].right_id) {
            set_err(err, errcap, "InvalidArgument(unk_handler_rdr): unk_handler_rdr includes invalid connection ids.");
            goto fail;
        }
    return d;
fail:
    vo_dict_free(d);
    return NULL;
}

vo_dict *vo_dict_from_mecab(const char *lex_csv, size_t lex_len, const char *matrix_def, size_t matrix_len,
                            const char *char_def, size_t char_len, const char *unk_def, size_t unk_len, char *err,
                            size_t errcap) {
    vo_dict *d = (vo_dict *)xcalloc(1, sizeof(vo_dict));
    if (matrix_from_text(d, matrix_def, matrix_len, err, errcap) != 0) {
        vo_dict_free(d);
        return NULL;
    }
    return dict_finish(d, lex_csv, lex_len, char_def, char_len, unk_def, unk_len, err, errcap);
}

vo_dict *vo_dict_from_parts(const char *lex_csv, size_t lex_len, const int16_t *matrix, uint32_t num_right,
                            uint32_t num_left, const char *char_def, size_t char_len, const char *unk_def,
                            size_t unk_len, char *err, size_t errcap) {
    vo_dict *d = (vo_dict *)xcalloc(1, sizeof(vo_dict));
    d->num_right = num_right;
    d->num_left = num_left;
    size_t n = (size_t)num_right * (size_t)num_left;
    d->matrix = (int16_t *)xmalloc(n * sizeof(int16_t));
    memcpy(d->matrix, matrix, n * sizeof(int16_t));
    return dict_finish(d, lex_csv, lex_len, char_def, char_len, unk_def, unk_len, err, errcap);
}

/* Dictionary::reset_user_lexicon_from_reader (dictionary.rs:209-229). Dictionaries built from
 * MeCab files carry no ConnIdMapper (builder.rs:42), so the remap of :215-217 is the identity. */
int vo_dict_set_user_csv(vo_dict *d, const char *csv, size_t len, char *err, size_t errcap) {
    if (!csv) {
        if (d->user) {
            lexicon_free(d->user);
            free(d->user);
            d->user = NULL;
        }
        return 0;
    }
    raw_entries ents;
    if (parse_csv(csv, len, "lex.csv", &ents, err, errcap) != 0) return -1; /* Lexicon::from_reader lexicon.rs:99-109 */
    if (d->map_left) { /* dictionary.rs:215-217: user ids go through the stored mapper */
        for (size_t i = 0; i < ents.n; i++) {
            if (ents.v[i].param.left_id >= d->num_left || ents.v[i].param.right_id >= d->num_right) {
                raw_entries_free(&ents);
                set_err(err, errcap, "InvalidArgument(user_lexicon_rdr): includes invalid connection ids.");
                return -1;
            }
            ents.v[i].param.left_id = d->map_left[ents.v[i].param.left_id];
            ents.v[i].param.right_id = d->map_right[ents.v[i].param.right_id];
        }
    }
    lexicon_t *lx = (lexicon_t *)xmalloc(sizeof(lexicon_t));
    lexicon_build(lx, &ents, 1);
    raw_entries_free(&ents);
    if (!lexicon_verify(lx, d->num_left, d->num_right)) { /* :218-223 */
        lexicon_free(lx);
        free(lx);
        set_err(err, errcap, "InvalidArgument(user_lexicon_rdr): includes invalid connection ids.");
        return -1;
    }
    if (d->user) {
        lexicon_free(d->user);
        free(d->user);
    }
    d->user = lx;
    return 0;
}

/* ------------------------------------------------------------------------------------------ */
/* lookups                                                                                     */
/* ------------------------------------------------------------------------------------------ */

static inline uint32_t char_info(const vo_dict *d, uint32_t cp) { /* character.rs:112-116 */
    return cp < d->chr2inf_len ? d->chr2inf[cp] : d->chr2inf[0];
}
uint32_t vo_dict_char_info(const vo_dict *d, uint32_t cp) { return char_info(d, cp); }

/* Scorer::retrieve_cost + accumulate_cost (scorer.rs:240-267), RawConnector::cost (raw_connector.rs:155-160) */
static int32_t raw_conn_cost(const vo_dict *d, uint32_t right_id, uint32_t left_id) {
    const uint32_t *k1 = d->right_feats + (size_t)right_id * d->feat_T;
    const uint32_t *k2 = d->left_feats + (size_t)left_id * d->feat_T;
    int32_t score = 0;
    for (uint32_t t = 0; t < d->feat_T; t++) {
        uint32_t key1 = k1[t], key2 = k2[t];
        if (key1 < d->n_bases) {
            uint32_t pos = d->sc_bases[key1] ^ key2;
            if (pos < d->n_checks && d->sc_checks[pos] == key1) score = (int32_t)((uint32_t)score + (uint32_t)d->sc_costs[pos]);
        }
    }
    return score;
}

static inline int32_t conn_cost(const vo_dict *d, uint32_t right_id, uint32_t left_id) { /* matrix_connector.rs:79-85,121-124 */
    if (__builtin_expect(d->matrix != NULL && d->dual_rmap == NULL, 1))
        return (int32_t)d->matrix[(size_t)left_id * d->num_right + right_id];
    if (d->dual_rmap) { /* DualConnector::cost dual_connector.rs:269-280 */
        int32_t m = (int32_t)d->matrix[(size_t)d->dual_lmap[left_id] * d->m_num_right + d->dual_rmap[right_id]];
        return (int32_t)((uint32_t)m + (uint32_t)raw_conn_cost(d, right_id, left_id));
    }
    return raw_conn_cost(d, right_id, left_id);
}
int32_t vo_dict_conn_cost(const vo_dict *d, uint16_t right_id, uint16_t left_id) { return conn_cost(d, right_id, left_id); }
uint32_t vo_dict_num_left(const vo_dict *d) { return d->num_left; }
uint32_t vo_dict_num_right(const vo_dict *d) { return d->num_right; }
uint32_t vo_dict_num_words(const vo_dict *d, int lex_type) {
    if (lex_type == 0) return d->sys.n_words;
    if (lex_type == 1) return d->user ? d->user->n_words : 0;
    return d->n_unk;
}

const char *vo_dict_feature(const vo_dict *d, uint32_t word_idx, size_t *len) { /* dictionary.rs:108-114 */
    uint32_t lex = word_idx >> 30, id = word_idx & 0x3FFFFFFFu;
    if (lex == 2) {
        if (id >= d->n_unk) return NULL;
        *len = d->unk_entries[id].feature_len;
        return d->unk_entries[id].feature;
    }
    const lexicon_t *lx = lex == 0 ? &d->sys : d->user;
    if (!lx || id >= lx->n_words) return NULL;
    *len = (size_t)(lx->feat_off[id + 1] - lx->feat_off[id]);
    return lx->feat_blob + lx->feat_off[id];
}

int vo_dict_word_param(const vo_dict *d, uint32_t word_idx, uint16_t *left, uint16_t *right, int16_t *cost) { /* dictionary.rs:98-104 */
    uint32_t lex = word_idx >> 30, id = word_idx & 0x3FFFFFFFu;
    if (lex == 2) {
        if (id >= d->n_unk) return -1;
        *left = d->unk_entries[id].left_id;
        *right = d->unk_entries[id].right_id;
        *cost = d->unk_entries[id].word_cost;
        return 0;
    }
    const lexicon_t *lx = lex == 0 ? &d->sys : d->user;
    if (!lx || id >= lx->n_words) return -1;
    *left = lx->params[id].left_id;
    *right = lx->params[id].right_id;
    *cost = lx->params[id].word_cost;
    return 0;
}

/* ------------------------------------------------------------------------------------------ */
/* Sentence / Lattice / Worker  (sentence.rs, tokenizer/lattice.rs, tokenizer/worker.rs)       */
/* ------------------------------------------------------------------------------------------ */

typedef struct { /* lattice.rs:13-23 */
    uint32_t word_id;
    uint32_t start_node;
    uint32_t start_word;
    int32_t min_cost;
    uint16_t left_id, right_id, min_idx;
    uint8_t lex_type;
} lnode;

typedef struct {
    lnode *v;
    uint32_t n, cap;
} lnode_vec;

struct vo_worker {
    const vo_dict *dict;
    int has_space_cateset; /* tokenizer.rs:16 Option<u32> */
    uint32_t space_cateset;
    int has_max_grouping;
    uint64_t max_grouping_len; /* tokenizer.rs:17 Option<usize> */
    /* Sentence (sentence.rs:4-10) */
    uint32_t *chars;
    uint32_t *c2b;
    uint32_t *cinfos;
    uint32_t *groupable;
    uint32_t len_char, cap_char;
    /* Lattice (lattice.rs:38-43) */
    lnode_vec *ends;
    uint32_t ends_len;
    lnode eos;
    /* top_nodes (worker.rs:17) materialised as tokens, already in sentence order */
    vo_token *tokens;
    uint32_t n_tokens, cap_tokens;
};

vo_worker *vo_worker_new(const vo_dict *d, int ignore_space, uint64_t max_grouping_len, char *err, size_t errcap) {
    vo_worker *w = (vo_worker *)xcalloc(1, sizeof(vo_worker));
    w->dict = d;
    if (ignore_space) { /* tokenizer.rs:42-55 */
        int id = find_category(d, "SPACE", 5);
        if (id < 0) {
            set_err(err, errcap, "InvalidArgument(dict): SPACE is not defined in the input dictionary (i.e., char.def).");
            free(w);
            return NULL;
        }
        w->has_space_cateset = 1;
        w->space_cateset = 1u << (id & 31); /* release-build `1 << id` */
    }
    if (max_grouping_len != 0) { /* tokenizer.rs:67-74 */
        w->has_max_grouping = 1;
        w->max_grouping_len = max_grouping_len;
    }
    return w;
}

void vo_worker_free(vo_worker *w) {
    if (!w) return;
    free(w->chars);
    free(w->c2b);
    free(w->cinfos);
    free(w->groupable);
    for (uint32_t i = 0; i < w->ends_len; i++) free(w->ends[i].v);
    free(w->ends);
    free(w->tokens);
    free(w);
}

const vo_token *vo_worker_tokens(const vo_worker *w) { return w->tokens; }

static inline void lv_push(lnode_vec *v, const lnode *n) {
    if (v->n == v->cap) {
        v->cap = v->cap ? v->cap * 2 : 16; /* lattice.rs:61 Vec::with_capacity(16) */
        v->v = (lnode *)xrealloc(v->v, (size_t)v->cap * sizeof(lnode));
    }
    v->v[v->n++] = *n;
}

/* Sentence::compile (sentence.rs:34-71) */
static void sentence_compile(vo_worker *w, const unsigned char *s, size_t len) {
    if (len + 1 > w->cap_char) {
        w->cap_char = (uint32_t)(len + 1) * 2;
        w->chars = (uint32_t *)xrealloc(w->chars, (size_t)w->cap_char * 4);
        w->c2b = (uint32_t *)xrealloc(w->c2b, (size_t)w->cap_char * 4);
        w->cinfos = (uint32_t *)xrealloc(w->cinfos, (size_t)w->cap_char * 4);
        w->groupable = (uint32_t *)xrealloc(w->groupable, (size_t)w->cap_char * 4);
    }
    uint32_t n = 0;
    for (size_t bi = 0; bi < len;) { /* compute_basic :40-46 */
        uint32_t cp;
        w->c2b[n] = (uint32_t)bi;
        bi += utf8_decode(s + bi, &cp);
        w->chars[n++] = cp;
    }
    w->c2b[n] = (uint32_t)len;
    w->len_char = n;
    const vo_dict *d = w->dict;
    for (uint32_t i = 0; i < n; i++) w->cinfos[i] = char_info(d, w->chars[i]); /* compute_categories :48-55 */
    if (n == 0) return;
    for (uint32_t i = 0; i < n; i++) w->groupable[i] = 1; /* compute_groupable :57-71 */
    uint32_t rhs = ci_cate_idset(w->cinfos[n - 1]);
    for (uint32_t i = n - 1; i >= 1; i--) {
        uint32_t lhs = ci_cate_idset(w->cinfos[i - 1]);
        if ((lhs & rhs) != 0) w->groupable[i - 1] = w->groupable[i] + 1;
        rhs = lhs;
    }
}

/* Lattice::reset + insert_bos (lattice.rs:46-64, 72-83) */
static void lattice_reset(vo_worker *w, uint32_t len_char) {
    for (uint32_t i = 0; i < w->ends_len; i++) w->ends[i].n = 0;
    if (w->ends_len <= len_char + 1) {
        w->ends = (lnode_vec *)xrealloc(w->ends, (size_t)(len_char + 1) * sizeof(lnode_vec));
        for (uint32_t i = w->ends_len; i < len_char + 1; i++) {
            w->ends[i].v = (lnode *)xmalloc(16 * sizeof(lnode));
            w->ends[i].n = 0;
            w->ends[i].cap = 16;
        }
        w->ends_len = len_char + 1;
    }
    lnode bos;
    memset(&bos, 0, sizeof(bos));
    bos.word_id = 0xFFFFFFFFu;
    bos.start_node = 0xFFFFFFFFu;
    bos.start_word = 0xFFFFFFFFu;
    bos.left_id = 0xFFFF;
    bos.right_id = 0; /* BOS_EOS_CONNECTION_ID common.rs:18 */
    bos.min_idx = 0xFFFF;
    bos.min_cost = 0;
    lv_push(&w->ends[0], &bos);
}

#ifdef VO_ANALYSIS
/* Lattice statistics for kernel design (tools/lattice_stats.py; single-threaded runs only). Never compiled into
 * libvibrato_oracle.so. */
enum { ANA_CALLS = 0, ANA_PAIRS, ANA_DISTINCT_RIGHT, ANA_SURV_COLMIN, ANA_SURV_BOTH, ANA_SURV_SORTED, ANA_POSITIONS,
       ANA_CANDS, ANA_DISTINCT_LEFT, ANA_DISTINCT_PAIRS, ANA_SURV_NATURAL, ANA_SURV_NATURAL_BOTH, ANA_SURV_HEUR, ANA_FIRST_STATIC, ANA_FIRST_B4, ANA_ARGMIN_B4, ANA_LAST_B4, ANA_NUM };
uint64_t vo_ana[ANA_NUM];
static int16_t *ana_colmin, *ana_rowmin; /* min over right of M[left][right]; min over left */
static uint16_t ana_lefts[4096];
static uint32_t ana_nleft;
void vo_ana_prepare(const vo_dict *d) {
    ana_colmin = (int16_t *)xcalloc(d->num_left, 2);
    ana_rowmin = (int16_t *)xcalloc(d->num_right, 2);
    for (uint32_t r = 0; r < d->num_right; r++) ana_rowmin[r] = INT16_MAX;
    for (uint32_t l = 0; l < d->num_left; l++) {
        int16_t m = INT16_MAX;
        for (uint32_t r = 0; r < d->num_right; r++) {
            int16_t v = d->matrix[(size_t)l * d->num_right + r];
            if (v < m) m = v;
            if (v < ana_rowmin[r]) ana_rowmin[r] = v;
        }
        ana_colmin[l] = m;
    }
    memset(vo_ana, 0, sizeof vo_ana);
}
static void ana_search(const vo_worker *w, const lnode_vec *v, uint32_t left_id) {
    const vo_dict *d = w->dict;
    uint32_t K = v->n;
    if (!K) return;
    vo_ana[ANA_CALLS]++;
    vo_ana[ANA_PAIRS] += K;
    uint32_t distinct = 0;
    for (uint32_t i = 0; i < K; i++) {
        int seen = 0;
        for (uint32_t j = 0; j < i; j++) seen |= v->v[j].right_id == v->v[i].right_id;
        distinct += !seen;
    }
    vo_ana[ANA_DISTINCT_RIGHT] += distinct;
    /* exact pruning: evaluate the cheapest predecessor first, then only those whose lower bound can still tie */
    uint32_t a = 0;
    for (uint32_t i = 1; i < K; i++)
        if (v->v[i].min_cost < v->v[a].min_cost) a = i;
    int64_t best0 = (int64_t)v->v[a].min_cost + conn_cost(d, v->v[a].right_id, left_id);
    uint32_t s1 = 1, s2 = 1;
    for (uint32_t i = 0; i < K; i++) {
        if (i == a) continue;
        int64_t pc = v->v[i].min_cost;
        if (pc + ana_colmin[left_id] <= best0) s1++;
        int16_t lb = ana_colmin[left_id] > ana_rowmin[v->v[i].right_id] ? ana_colmin[left_id] : ana_rowmin[v->v[i].right_id];
        if (pc + lb <= best0) s2++;
    }
    vo_ana[ANA_SURV_COLMIN] += s1;
    vo_ana[ANA_SURV_BOTH] += s2;
    /* ascending predecessor cost with a running best: stop at the first one whose bound exceeds it */
    {
        uint32_t idx[256];
        uint32_t n = K < 256 ? K : 256;
        for (uint32_t i = 0; i < n; i++) idx[i] = i;
        for (uint32_t i = 1; i < n; i++) {
            uint32_t t = idx[i], j = i;
            while (j && v->v[idx[j - 1]].min_cost > v->v[t].min_cost) { idx[j] = idx[j - 1]; j--; }
            idx[j] = t;
        }
        int64_t best = INT64_MAX;
        uint32_t ev = 0;
        for (uint32_t i = 0; i < n; i++) {
            const lnode *ln = &v->v[idx[i]];
            if (best != INT64_MAX && (int64_t)ln->min_cost + ana_colmin[left_id] > best) break;
            int16_t lb = ana_rowmin[ln->right_id];
            if (best != INT64_MAX && (int64_t)ln->min_cost + lb > best) continue;
            ev++;
            int64_t c = (int64_t)ln->min_cost + conn_cost(d, ln->right_id, left_id);
            if (c < best) best = c;
        }
        vo_ana[ANA_SURV_SORTED] += ev;
    }
    { /* row order, running best */
        int64_t best = INT64_MAX, best2 = INT64_MAX;
        uint32_t ev = 0, ev2 = 0;
        for (uint32_t i = 0; i < K; i++) {
            const lnode *ln = &v->v[i];
            int64_t c = (int64_t)ln->min_cost + conn_cost(d, ln->right_id, left_id);
            if (best == INT64_MAX || (int64_t)ln->min_cost + ana_colmin[left_id] <= best) {
                ev++;
                if (c < best) best = c;
            }
            int16_t lb = ana_colmin[left_id] > ana_rowmin[ln->right_id] ? ana_colmin[left_id] : ana_rowmin[ln->right_id];
            if (best2 == INT64_MAX || (int64_t)ln->min_cost + lb <= best2) {
                ev2++;
                if (c < best2) best2 = c;
            }
        }
        vo_ana[ANA_SURV_NATURAL] += ev;
        vo_ana[ANA_SURV_NATURAL_BOTH] += ev2;
    }
    { /* cheapest of the first 8 predecessors first, then row order with a running best */
        uint32_t a8 = 0;
        for (uint32_t i = 1; i < K && i < 8; i++)
            if (v->v[i].min_cost < v->v[a8].min_cost) a8 = i;
        int64_t best = (int64_t)v->v[a8].min_cost + conn_cost(d, v->v[a8].right_id, left_id);
        uint32_t ev = 1;
        for (uint32_t i = 0; i < K; i++) {
            if (i == a8) continue;
            const lnode *ln = &v->v[i];
            if ((int64_t)ln->min_cost + ana_colmin[left_id] <= best) {
                ev++;
                int64_t c = (int64_t)ln->min_cost + conn_cost(d, ln->right_id, left_id);
                if (c < best) best = c;
            }
        }
        vo_ana[ANA_SURV_HEUR] += ev;
    }
    { /* GPU-shaped schedules: one predecessor evaluated alone, the rest in batches of 4 whose bound is the best
       * total known when the batch starts (loads of a batch are issued together) */
        for (int variant = 0; variant < 4; variant++) {
            uint32_t a = 0;
            if (variant == 2)
                for (uint32_t i = 1; i < K; i++)
                    if (v->v[i].min_cost < v->v[a].min_cost) a = i;
            if (variant == 3) a = K - 1;
            int64_t B = (int64_t)v->v[a].min_cost + conn_cost(d, v->v[a].right_id, left_id);
            uint32_t ev = 1;
            int64_t Bnext = B;
            uint32_t inb = 0;
            for (uint32_t i = 0; i < K; i++) {
                if (i == a && variant != 2) continue; /* variant 2 re-evaluates the argmin in row order */
                const lnode *ln = &v->v[i];
                if ((int64_t)ln->min_cost + ana_colmin[left_id] <= B) {
                    ev++;
                    int64_t c = (int64_t)ln->min_cost + conn_cost(d, ln->right_id, left_id);
                    if (c < Bnext) Bnext = c;
                }
                if (++inb == 4) {
                    inb = 0;
                    if (variant != 0) B = Bnext;
                }
            }
            vo_ana[ANA_FIRST_STATIC + variant] += ev;
        }
    }
    if (ana_nleft < 4096) ana_lefts[ana_nleft++] = (uint16_t)left_id;
}
static void ana_position(uint32_t K, const lnode_vec *v) {
    if (!ana_nleft) return;
    vo_ana[ANA_POSITIONS]++;
    vo_ana[ANA_CANDS] += ana_nleft;
    uint32_t dl = 0, dr = 0;
    for (uint32_t i = 0; i < ana_nleft; i++) {
        int seen = 0;
        for (uint32_t j = 0; j < i; j++) seen |= ana_lefts[j] == ana_lefts[i];
        dl += !seen;
    }
    for (uint32_t i = 0; i < K; i++) {
        int seen = 0;
        for (uint32_t j = 0; j < i; j++) seen |= v->v[j].right_id == v->v[i].right_id;
        dr += !seen;
    }
    vo_ana[ANA_DISTINCT_LEFT] += dl;
    vo_ana[ANA_DISTINCT_PAIRS] += (uint64_t)dl * dr;
    ana_nleft = 0;
}
#endif

/* Lattice::search_min_node (lattice.rs:129-151): `<=` keeps the LAST minimal predecessor.  VO_STRICT_TIES builds a
 * deliberately wrong variant with `<` (the FIRST minimum wins, EOS included) that the tests use to show that their
 * corpora contain ties which decide tokens. */
#ifdef VO_STRICT_TIES
#define VO_TIE_CMP(a, b) ((a) < (b) || i == 0) /* the first predecessor is taken even at INT32_MAX */
#else
#define VO_TIE_CMP(a, b) ((a) <= (b))
#endif
static inline void search_min_node(const vo_worker *w, uint32_t start_node, uint32_t left_id, uint16_t *min_idx,
                                   int32_t *min_cost, uint64_t *cnt) {
    const lnode_vec *v = &w->ends[start_node];
    uint16_t bi = 0xFFFF;
    int32_t bc = INT32_MAX;
    const vo_dict *d = w->dict;
    for (uint32_t i = 0; i < v->n; i++) {
        const lnode *ln = &v->v[i];
        int32_t cc = conn_cost(d, ln->right_id, left_id);
        int32_t nc = (int32_t)((uint32_t)ln->min_cost + (uint32_t)cc); /* release-mode wrapping add */
        if (VO_TIE_CMP(nc, bc)) {
            bi = (uint16_t)i; /* :144 `i as u16` */
            bc = nc;
        }
    }
    if (cnt) cnt[VO_CNT_E] += v->n;
#ifdef VO_ANALYSIS
    ana_search(w, v, left_id);
#endif
    *min_idx = bi;
    *min_cost = bc;
}

/* Lattice::insert_node (lattice.rs:103-127) */
static inline void insert_node(vo_worker *w, uint32_t start_node, uint32_t start_word, uint32_t end_word,
                               uint32_t word_id, uint8_t lex_type, word_param p, uint64_t *cnt) {
    lnode n;
    search_min_node(w, start_node, p.left_id, &n.min_idx, &n.min_cost, cnt);
    n.min_cost = (int32_t)((uint32_t)n.min_cost + (uint32_t)(int32_t)p.word_cost);
    n.word_id = word_id;
    n.lex_type = lex_type;
    n.start_node = start_node;
    n.start_word = start_word;
    n.left_id = p.left_id;
    n.right_id = p.right_id;
    lv_push(&w->ends[end_word], &n);
    if (cnt) cnt[VO_CNT_N]++;
}

/* Lexicon::common_prefix_iterator (lexicon.rs:33-46) over WordMap (map.rs:33-42), the trie search
 * (trie.rs:49-56 -> crawdad common_prefix_search) and Postings::ids (posting.rs:18-21); each match
 * goes straight into Lattice::insert_node as in tokenizer.rs:155-181. Returns has_matched. */
static inline int lexicon_walk(vo_worker *w, const lexicon_t *lx, uint32_t start_node, uint32_t start_word,
                               uint64_t *cnt) {
    const trie_t *t = &lx->trie;
    const uint32_t *chars = w->chars + start_word;
    uint32_t n = w->len_char - start_word;
    int matched = 0;
    uint32_t node = 0, d = 0, hits = 0;
    if (t->num_nodes == 0) goto out;
    for (uint32_t pos = 0; pos < n; pos++) {
        uint32_t c = chars[pos];
        if (c >= t->table_len) break;
        uint32_t code = t->table[c];
        if (code == CODE_INVALID) break;
        uint32_t base = t->nodes[node].base;
        if (base & DA_FLAG) break; /* a leaf has no children */
        uint32_t child = base ^ code;
        if ((t->nodes[child].check & DA_MASK) != node) break;
        node = child;
        d++;
        uint32_t value;
        uint32_t nb = t->nodes[node].base;
        if (nb & DA_FLAG) {
            value = nb & DA_MASK;
        } else if (t->nodes[node].check & DA_FLAG) {
            value = t->nodes[nb].base & DA_MASK; /* terminal child at base ^ 0 */
        } else {
            continue;
        }
        hits++;
        uint32_t plen = lx->postings[value];
        for (uint32_t q = 0; q < plen; q++) {
            uint32_t word_id = lx->postings[value + 1 + q];
            insert_node(w, start_node, start_word, start_word + pos + 1, word_id, (uint8_t)lx->lex_type,
                        lx->params[word_id], cnt);
        }
        if (cnt) {
            cnt[VO_CNT_P] += 1 + plen;
            cnt[VO_CNT_W] += plen;
        }
        matched = 1;
    }
out:
    if (cnt) {
        uint32_t f = d < n ? 1 : 0;
        cnt[VO_CNT_M] += d + f;
        cnt[VO_CNT_T] += d + f + hits;
        cnt[VO_CNT_WALKS]++;
    }
    return matched;
}

/* UnkHandler::scan_entries (unknown.rs:119-137) */
static inline void unk_scan_entries(vo_worker *w, uint32_t start_node, uint32_t start_char, uint32_t end_char,
                                    uint32_t cinfo, uint64_t *cnt) {
    const vo_dict *d = w->dict;
    uint32_t s = d->unk_offsets[ci_base_id(cinfo)], e = d->unk_offsets[ci_base_id(cinfo) + 1];
    for (uint32_t word_id = s; word_id < e; word_id++) {
        const unk_entry *ue = &d->unk_entries[word_id];
        word_param p = {ue->left_id, ue->right_id, ue->word_cost};
        /* :133 `word_id as u16`; tokenizer.rs:189-196 inserts with the driver's start_node */
        insert_node(w, start_node, start_char, end_char, (uint32_t)(uint16_t)word_id, 2, p, cnt);
    }
    if (cnt) cnt[VO_CNT_W] += e - s;
}

/* UnkHandler::gen_unk_words (unknown.rs:69-116) */
static inline void gen_unk_words(vo_worker *w, uint32_t start_node, uint32_t start_char, int has_matched,
                                 uint64_t *cnt) {
    uint32_t cinfo = w->cinfos[start_char];
    if (has_matched && !ci_invoke(cinfo)) return;
    int grouped = 0;
    uint32_t groupable = w->groupable[start_char];
    if (ci_group(cinfo)) {
        grouped = 1;
        /* :91-93: compare groupable-1 against the limit (usize::MAX when unset) */
        if (!w->has_max_grouping || (uint64_t)(groupable - 1) <= w->max_grouping_len) {
            unk_scan_entries(w, start_node, start_char, start_char + groupable, cinfo, cnt);
            has_matched = 1;
        }
    }
    uint32_t lim = ci_length(cinfo) < groupable ? ci_length(cinfo) : groupable;
    for (uint32_t i = 1; i <= lim; i++) {
        if (grouped && i == groupable) continue;
        uint32_t end_char = start_char + i;
        if (w->len_char < end_char) break;
        unk_scan_entries(w, start_node, start_char, end_char, cinfo, cnt);
        has_matched = 1;
    }
    if (!has_matched) unk_scan_entries(w, start_node, start_char, start_char + 1, cinfo, cnt); /* :112-115 */
}

/* Tokenizer::add_lattice_edges (tokenizer.rs:141-199) */
static inline void add_lattice_edges(vo_worker *w, uint32_t start_node, uint32_t start_word, uint64_t *cnt) {
    int has_matched = 0;
    if (w->dict->user) has_matched |= lexicon_walk(w, w->dict->user, start_node, start_word, cnt); /* :155-168 */
    has_matched |= lexicon_walk(w, &w->dict->sys, start_node, start_word, cnt);                    /* :170-181 */
    gen_unk_words(w, start_node, start_word, has_matched, cnt);                                     /* :183-198 */
}

static inline __attribute__((always_inline)) size_t tokenize_impl(vo_worker *w, const char *utf8, size_t len,
                                                                  uint64_t *cnt) {
    /* Worker::reset_sentence (worker.rs:34-45) */
    w->n_tokens = 0;
    w->len_char = 0;
    if (len == 0) return 0;
    sentence_compile(w, (const unsigned char *)utf8, len);
    if (cnt) {
        cnt[VO_CNT_U] += len;
        cnt[VO_CNT_C] += w->len_char;
    }
    /* Worker::tokenize (worker.rs:49-55) -> Tokenizer::build_lattice_inner (tokenizer.rs:94-139) */
    uint32_t n = w->len_char;
    lattice_reset(w, n);
    if (cnt) cnt[VO_CNT_N]++; /* BOS */
    uint32_t start_node = 0, start_word = 0;
    while (start_word < n) {
        if (w->ends[start_node].n == 0) { /* has_previous_node lattice.rs:155-157 */
            start_word += 1;
            start_node = start_word;
            continue;
        }
        if (w->has_space_cateset) { /* :117-125 */
            int is_space = (ci_cate_idset(w->cinfos[start_node]) & w->space_cateset) != 0;
            if (is_space) start_word += w->groupable[start_node];
        }
        if (start_word == n) break; /* :128-130 */
        add_lattice_edges(w, start_node, start_word, cnt);
#ifdef VO_ANALYSIS
        ana_position(w->ends[start_node].n, &w->ends[start_node]);
#endif
        start_word += 1;
        start_node = start_word;
    }
    /* Lattice::insert_eos (lattice.rs:85-101) */
    search_min_node(w, start_node, 0, &w->eos.min_idx, &w->eos.min_cost, cnt);
#ifdef VO_ANALYSIS
    ana_nleft = 0;
#endif
    w->eos.start_node = start_node;
    w->eos.start_word = n;
    if (cnt) cnt[VO_CNT_N]++;
    if (w->eos.min_idx == 0xFFFF && w->ends[start_node].n == 0) {
        /* Dead end: some visited position produced no node at all (possible only when unk.def has
         * no entry for a character category).  The reference then indexes ends[..][u16::MAX] in
         * append_top_nodes (lattice.rs:163) and panics; oracle and product both define the result
         * as "no tokens" instead. */
        return 0;
    }
    /* Lattice::append_top_nodes (lattice.rs:159-168), then worker.rs:65-68 reverses */
    uint32_t k = 0;
    {
        uint32_t end_node = w->eos.start_node;
        uint16_t min_idx = w->eos.min_idx;
        while (end_node != 0) {
            const lnode *nd = &w->ends[end_node].v[min_idx];
            k++;
            end_node = nd->start_node;
            min_idx = nd->min_idx;
        }
    }
    if (k > w->cap_tokens) {
        w->cap_tokens = k * 2;
        w->tokens = (vo_token *)xrealloc(w->tokens, (size_t)w->cap_tokens * sizeof(vo_token));
    }
    {
        uint32_t end_node = w->eos.start_node;
        uint16_t min_idx = w->eos.min_idx;
        uint32_t i = k;
        while (end_node != 0) {
            const lnode *nd = &w->ends[end_node].v[min_idx];
            vo_token *t = &w->tokens[--i];
            t->start_char = nd->start_word; /* token.rs:21-24 */
            t->end_char = end_node;
            t->start_byte = w->c2b[nd->start_word]; /* token.rs:28-32 */
            t->end_byte = w->c2b[end_node];
            t->word_idx = ((uint32_t)nd->lex_type << 30) | (nd->word_id & 0x3FFFFFFFu);
            t->total_cost = nd->min_cost; /* token.rs:89-92 */
            end_node = nd->start_node;
            min_idx = nd->min_idx;
        }
    }
    w->n_tokens = k;
    if (cnt) cnt[VO_CNT_K] += k;
    return k;
}

size_t vo_worker_tokenize(vo_worker *w, const char *utf8, size_t len) { return tokenize_impl(w, utf8, len, NULL); }
size_t vo_worker_tokenize_counted(vo_worker *w, const char *utf8, size_t len, uint64_t *cnt) {
    return tokenize_impl(w, utf8, len, cnt);
}

size_t vo_dict_common_prefix(const vo_dict *d, int lex_type, const uint32_t *chars, size_t n, uint32_t *word_ids,
                             uint32_t *end_chars, size_t cap) {
    const lexicon_t *lx = lex_type == 0 ? &d->sys : d->user;
    if (!lx || lx->trie.num_nodes == 0) return 0;
    const trie_t *t = &lx->trie;
    size_t out = 0;
    uint32_t node = 0;
    for (size_t pos = 0; pos < n; pos++) {
        uint32_t c = chars[pos];
        if (c >= t->table_len) break;
        uint32_t code = t->table[c];
        if (code == CODE_INVALID) break;
        uint32_t base = t->nodes[node].base;
        if (base & DA_FLAG) break;
        uint32_t child = base ^ code;
        if ((t->nodes[child].check & DA_MASK) != node) break;
        node = child;
        uint32_t value, nb = t->nodes[node].base;
        if (nb & DA_FLAG)
            value = nb & DA_MASK;
        else if (t->nodes[node].check & DA_FLAG)
            value = t->nodes[nb].base & DA_MASK;
        else
            continue;
        uint32_t plen = lx->postings[value];
        for (uint32_t q = 0; q < plen; q++) {
            if (out < cap) {
                word_ids[out] = lx->postings[value + 1 + q];
                end_chars[out] = (uint32_t)pos + 1;
            }
            out++;
        }
    }
    return out;
}

/* ------------------------------------------------------------------------------------------ */
/* batch drivers                                                                               */
/* ------------------------------------------------------------------------------------------ */

typedef struct {
    const vo_dict *d;
    int ignore_space;
    uint64_t max_grouping_len;
    const char *utf8;
    const uint64_t *off;
    uint64_t lo, hi;
    int want_tokens, want_cnt, runs;
    uint64_t *tok_off; /* per-sentence counts written at [i+1] */
    vo_token *toks;
    uint64_t n_toks, cap_toks;
    uint64_t cnt[VO_NUM_COUNTERS];
    uint64_t n_words;
} batch_job;

static void *batch_thread(void *arg) {
    batch_job *j = (batch_job *)arg;
    vo_worker *w = vo_worker_new(j->d, j->ignore_space, j->max_grouping_len, NULL, 0);
    if (!w) return NULL;
    for (int r = 0; r < j->runs; r++) {
        for (uint64_t i = j->lo; i < j->hi; i++) {
            const char *s = j->utf8 + j->off[i];
            size_t len = (size_t)(j->off[i + 1] - j->off[i]);
            size_t k = j->want_cnt ? tokenize_impl(w, s, len, j->cnt) : tokenize_impl(w, s, len, NULL);
            j->n_words += k;
            if (j->tok_off) j->tok_off[i + 1] = k;
            if (j->want_tokens) {
                if (j->n_toks + k > j->cap_toks) {
                    j->cap_toks = (j->n_toks + k) * 2 + 1024;
                    j->toks = (vo_token *)xrealloc(j->toks, (size_t)j->cap_toks * sizeof(vo_token));
                }
                memcpy(j->toks + j->n_toks, w->tokens, k * sizeof(vo_token));
                j->n_toks += k;
            }
        }
    }
    vo_worker_free(w);
    return NULL;
}

static uint64_t run_batch(const vo_dict *d, int ignore_space, uint64_t max_grouping_len, const char *utf8,
                          const uint64_t *off, uint64_t n, int n_threads, int runs, uint64_t *tok_off,
                          vo_token **toks, uint64_t *cnt) {
    if (n_threads < 1) n_threads = 1;
    if ((uint64_t)n_threads > n && n > 0) n_threads = (int)n;
    batch_job *jobs = (batch_job *)xcalloc((size_t)n_threads, sizeof(batch_job));
    pthread_t *th = (pthread_t *)xmalloc((size_t)n_threads * sizeof(pthread_t));
    for (int t = 0; t < n_threads; t++) {
        batch_job *j = &jobs[t];
        j->d = d;
        j->ignore_space = ignore_space;
        j->max_grouping_len = max_grouping_len;
        j->utf8 = utf8;
        j->off = off;
        j->lo = n * (uint64_t)t / (uint64_t)n_threads;
        j->hi = n * (uint64_t)(t + 1) / (uint64_t)n_threads;
        j->want_tokens = toks != NULL;
        j->want_cnt = cnt != NULL;
        j->runs = runs;
        j->tok_off = tok_off;
    }
    if (n_threads == 1) {
        batch_thread(&jobs[0]);
    } else {
        for (int t = 0; t < n_threads; t++) pthread_create(&th[t], NULL, batch_thread, &jobs[t]);
        for (int t = 0; t < n_threads; t++) pthread_join(th[t], NULL);
    }
    uint64_t total = 0;
    for (int t = 0; t < n_threads; t++) total += jobs[t].n_words;
    if (cnt)
        for (int t = 0; t < n_threads; t++)
            for (int c = 0; c < VO_NUM_COUNTERS; c++) cnt[c] += jobs[t].cnt[c];
    if (tok_off) {
        tok_off[0] = 0;
        for (uint64_t i = 0; i < n; i++) tok_off[i + 1] += tok_off[i];
    }
    if (toks) {
        uint64_t all = 0;
        for (int t = 0; t < n_threads; t++) all += jobs[t].n_toks;
        vo_token *out = (vo_token *)xmalloc((size_t)(all ? all : 1) * sizeof(vo_token));
        uint64_t p = 0;
        for (int t = 0; t < n_threads; t++) {
            memcpy(out + p, jobs[t].toks, (size_t)jobs[t].n_toks * sizeof(vo_token));
            p += jobs[t].n_toks;
            free(jobs[t].toks);
        }
        *toks = out;
    }
    free(jobs);
    free(th);
    return total;
}

uint64_t vo_tokenize_batch(const vo_dict *d, int ignore_space, uint64_t max_grouping_len, const char *utf8,
                           const uint64_t *off, uint64_t n, int n_threads, uint64_t *tok_off, vo_token **toks,
                           uint64_t *cnt) {
    if (ignore_space && find_category(d, "SPACE", 5) < 0) return 0;
    return run_batch(d, ignore_space, max_grouping_len, utf8, off, n, n_threads, 1, tok_off, toks, cnt);
}

/* The timed body of benchmark/src/main.rs:53-65 (reset_sentence + tokenize + num_tokens per line),
 * `runs` passes; returns elapsed wall-clock seconds for all passes. */
double vo_benchmark(const vo_dict *d, int ignore_space, uint64_t max_grouping_len, const char *utf8,
                    const uint64_t *off, uint64_t n, int n_threads, int runs, uint64_t *n_words) {
    struct timespec t0, t1;
    clock_gettime(CLOCK_MONOTONIC, &t0);
    uint64_t total = run_batch(d, ignore_space, max_grouping_len, utf8, off, n, n_threads, runs, NULL, NULL, NULL);
    clock_gettime(CLOCK_MONOTONIC, &t1);
    if (n_words) *n_words = total;
    return (double)(t1.tv_sec - t0.tv_sec) + 1e-9 * (double)(t1.tv_nsec - t0.tv_nsec);
}


/* ------------------------------------------------------------------------------------------ */
/* connection-id statistics and remapping (dictionary/mapper.rs, lattice.rs:170-183)           */
/* ------------------------------------------------------------------------------------------ */

/* Lattice::add_connid_counts (lattice.rs:170-183) for the lattice of the last tokenize call. */
static void add_connid_counts(const vo_worker *w, uint64_t *lid, uint64_t *rid) {
    if (w->len_char == 0) return;
    for (uint32_t end_char = 1; end_char <= w->len_char; end_char++) {
        const lnode_vec *row = &w->ends[end_char];
        for (uint32_t i = 0; i < row->n; i++) {
            const lnode *r_node = &row->v[i];
            const lnode_vec *prev = &w->ends[r_node->start_node];
            for (uint32_t k = 0; k < prev->n; k++) { /* ConnIdCounter::add mapper.rs:101-104 */
                lid[r_node->left_id] += 1;
                rid[prev->v[k].right_id] += 1;
            }
        }
    }
    const lnode_vec *last = &w->ends[w->len_char]; /* :178-181: the EOS edges use ends[len_char] */
    for (uint32_t k = 0; k < last->n; k++) {
        lid[0] += 1;
        rid[last->v[k].right_id] += 1;
    }
}

typedef struct {
    const vo_dict *d;
    int ignore_space;
    uint64_t max_grouping_len;
    const char *utf8;
    const uint64_t *off;
    uint64_t lo, hi;
    uint64_t *lid, *rid;
} connid_job;

static void *connid_thread(void *arg) {
    connid_job *j = (connid_job *)arg;
    vo_worker *w = vo_worker_new(j->d, j->ignore_space, j->max_grouping_len, NULL, 0);
    if (!w) return NULL;
    for (uint64_t i = j->lo; i < j->hi; i++) {
        size_t len = (size_t)(j->off[i + 1] - j->off[i]);
        tokenize_impl(w, j->utf8 + j->off[i], len, NULL);
        if (len) add_connid_counts(w, j->lid, j->rid);
    }
    vo_worker_free(w);
    return NULL;
}

int vo_connid_counts_batch(const vo_dict *d, int ignore_space, uint64_t max_grouping_len, const char *utf8,
                           const uint64_t *off, uint64_t n, int n_threads, uint64_t *lid_count,
                           uint64_t *rid_count) {
    if (ignore_space && find_category(d, "SPACE", 5) < 0) return -1;
    if (n_threads < 1) n_threads = 1;
    if ((uint64_t)n_threads > n && n > 0) n_threads = (int)n;
    connid_job *jobs = (connid_job *)xcalloc((size_t)n_threads, sizeof(connid_job));
    pthread_t *th = (pthread_t *)xmalloc((size_t)n_threads * sizeof(pthread_t));
    for (int t = 0; t < n_threads; t++) {
        jobs[t] = (connid_job){d, ignore_space, max_grouping_len, utf8, off, n * (uint64_t)t / (uint64_t)n_threads,
                               n * (uint64_t)(t + 1) / (uint64_t)n_threads,
                               (uint64_t *)xcalloc(d->num_left, sizeof(uint64_t)),
                               (uint64_t *)xcalloc(d->num_right, sizeof(uint64_t))};
        pthread_create(&th[t], NULL, connid_thread, &jobs[t]);
    }
    memset(lid_count, 0, d->num_left * sizeof(uint64_t));
    memset(rid_count, 0, d->num_right * sizeof(uint64_t));
    for (int t = 0; t < n_threads; t++) {
        pthread_join(th[t], NULL);
        for (uint32_t i = 0; i < d->num_left; i++) lid_count[i] += jobs[t].lid[i];
        for (uint32_t i = 0; i < d->num_right; i++) rid_count[i] += jobs[t].rid[i];
        free(jobs[t].lid);
        free(jobs[t].rid);
    }
    free(jobs);
    free(th);
    return 0;
}

/* ConnIdMapper::parse (mapper.rs:49-80): `map` lists OLD ids in their NEW order (new id = 1-origin rank);
 * returns new_ids[old_id], length n + 1. */
static uint16_t *mapper_parse(const uint16_t *map, size_t n, char *err, size_t errcap) {
    if (n + 1 > 65536) {
        set_err(err, errcap, "TryFromInt(map): too many ids");
        return NULL;
    }
    uint16_t *new_ids = (uint16_t *)xmalloc((n + 1) * sizeof(uint16_t));
    for (size_t i = 0; i <= n; i++) new_ids[i] = 0xFFFF;
    new_ids[0] = 0;
    for (size_t i = 0; i < n; i++) {
        uint16_t old_id = map[i];
        if (old_id == 0) { /* :55-58 */
            set_err(err, errcap, "InvalidArgument(map): Id 0 is reserved.");
            free(new_ids);
            return NULL;
        }
        if ((size_t)old_id > n) { /* :72-77 */
            set_err(err, errcap, "InvalidArgument(map): ids are out of range.");
            free(new_ids);
            return NULL;
        }
        if (new_ids[old_id] != 0xFFFF) { /* :68-70 */
            set_err(err, errcap, "InvalidArgument(map): ids are duplicate.");
            free(new_ids);
            return NULL;
        }
        new_ids[old_id] = (uint16_t)(i + 1);
    }
    return new_ids;
}

int vo_dict_map_connection_ids(vo_dict *d, const uint16_t *lmap, size_t n_lmap, const uint16_t *rmap, size_t n_rmap,
                               char *err, size_t errcap) {
    uint16_t *L = mapper_parse(lmap, n_lmap, err, errcap);
    if (!L) return -1;
    uint16_t *Rm = mapper_parse(rmap, n_rmap, err, errcap);
    if (!Rm) {
        free(L);
        return -1;
    }
    /* matrix_connector.rs:100-101 asserts the mapper covers the matrix exactly (a panic upstream) */
    if (n_lmap + 1 != d->num_left || n_rmap + 1 != d->num_right) {
        set_err(err, errcap, "InvalidArgument(map): the mapping must cover every connection id of the matrix");
        free(L);
        free(Rm);
        return -1;
    }
    lexicon_t *lexs[2] = {&d->sys, d->user};
    for (int li = 0; li < 2; li++) { /* WordParams::map_connection_ids param.rs:48-53 */
        if (!lexs[li]) continue;
        for (uint32_t i = 0; i < lexs[li]->n_words; i++) {
            lexs[li]->params[i].left_id = L[lexs[li]->params[i].left_id];
            lexs[li]->params[i].right_id = Rm[lexs[li]->params[i].right_id];
        }
    }
    size_t nr = d->num_right, nl = d->num_left;
    if (d->matrix && !d->dual_rmap) { /* matrix_connector.rs:103-115 */
        int16_t *mapped = (int16_t *)xcalloc(nr * nl, sizeof(int16_t));
        for (size_t r = 0; r < nr; r++)
            for (size_t l = 0; l < nl; l++) mapped[(size_t)L[l] * nr + Rm[r]] = d->matrix[l * nr + r];
        free(d->matrix);
        d->matrix = mapped;
    } else { /* DualConnector moves its rows alike (dual_connector.rs:227-245); RawConnector::map_connection_ids raw_connector.rs:124-152: move the feature rows */
        size_t T = d->feat_T;
        uint32_t *mr = (uint32_t *)xcalloc(nr * T + 1, sizeof(uint32_t));
        uint32_t *ml = (uint32_t *)xcalloc(nl * T + 1, sizeof(uint32_t));
        for (size_t r = 0; r < nr; r++) memcpy(mr + (size_t)Rm[r] * T, d->right_feats + r * T, T * sizeof(uint32_t));
        for (size_t l = 0; l < nl; l++) memcpy(ml + (size_t)L[l] * T, d->left_feats + l * T, T * sizeof(uint32_t));
        free(d->right_feats);
        free(d->left_feats);
        d->right_feats = mr;
        d->left_feats = ml;
    }
    if (d->dual_rmap) { /* dual_connector.rs:227-266 */
        uint16_t *nrm = (uint16_t *)xcalloc(nr, sizeof(uint16_t)), *nlm = (uint16_t *)xcalloc(nl, sizeof(uint16_t));
        for (size_t r = 0; r < nr; r++) nrm[Rm[r]] = d->dual_rmap[r];
        for (size_t l = 0; l < nl; l++) nlm[L[l]] = d->dual_lmap[l];
        free(d->dual_rmap);
        free(d->dual_lmap);
        d->dual_rmap = nrm;
        d->dual_lmap = nlm;
        /* the reduced matrix is renumbered by first appearance in the new order (dual_connector.rs:247-265) */
        size_t mr_n = d->m_num_right, ml_n = d->m_num_left;
        uint16_t *ren_l = (uint16_t *)xmalloc(ml_n * sizeof(uint16_t)), *ren_r = (uint16_t *)xmalloc(mr_n * sizeof(uint16_t));
        memset(ren_l, 0xFF, ml_n * sizeof(uint16_t));
        memset(ren_r, 0xFF, mr_n * sizeof(uint16_t));
        uint16_t next = 0;
        for (size_t l = 0; l < nl; l++) {
            uint16_t *slot = &ren_l[d->dual_lmap[l]];
            if (*slot == 0xFFFF) *slot = next++;
            d->dual_lmap[l] = *slot;
        }
        next = 0;
        for (size_t r = 0; r < nr; r++) {
            uint16_t *slot = &ren_r[d->dual_rmap[r]];
            if (*slot == 0xFFFF) *slot = next++;
            d->dual_rmap[r] = *slot;
        }
        int16_t *mapped = (int16_t *)xcalloc(mr_n * ml_n, sizeof(int16_t));
        for (size_t l = 0; l < ml_n; l++)
            for (size_t r = 0; r < mr_n; r++)
                if (ren_l[l] != 0xFFFF && ren_r[r] != 0xFFFF) mapped[(size_t)ren_l[l] * mr_n + ren_r[r]] = d->matrix[l * mr_n + r];
        free(d->matrix);
        d->matrix = mapped;
        free(ren_l);
        free(ren_r);
    }
    for (uint32_t i = 0; i < d->n_unk; i++) { /* unknown.rs:203-208 */
        d->unk_entries[i].left_id = L[d->unk_entries[i].left_id];
        d->unk_entries[i].right_id = Rm[d->unk_entries[i].right_id];
    }
    free(d->map_left);
    free(d->map_right);
    d->map_left = L; /* dictionary.rs:257 */
    d->map_right = Rm;
    return 0;
}


/* ------------------------------------------------------------------------------------------ */
/* RawConnector from bigram.{right,left,cost} (connector/raw_connector.rs, raw_connector/scorer.rs) */
/* ------------------------------------------------------------------------------------------ */

#define INVALID_FEATURE_ID 0x7FFFFFFFu /* raw_connector.rs:19 U31::MAX */
#define UNUSED_CHECK 0xFFFFFFFFu       /* scorer.rs:15 */

/* string -> id map with ids in first-seen order (the HashMap of raw_connector.rs:195-198,296-309) */
typedef struct {
    char **keys;
    size_t *lens;
    uint32_t *ids;
    size_t cap, n;
} str_map;

static uint64_t str_hash(const char *s, size_t n) {
    uint64_t h = 1469598103934665603ull;
    for (size_t i = 0; i < n; i++) h = (h ^ (unsigned char)s[i]) * 1099511628211ull;
    return h;
}
static void sm_init(str_map *m) {
    m->cap = 1024;
    m->n = 0;
    m->keys = (char **)xcalloc(m->cap, sizeof(char *));
    m->lens = (size_t *)xcalloc(m->cap, sizeof(size_t));
    m->ids = (uint32_t *)xcalloc(m->cap, sizeof(uint32_t));
}
static void sm_free(str_map *m) {
    for (size_t i = 0; i < m->cap; i++) free(m->keys[i]);
    free(m->keys);
    free(m->lens);
    free(m->ids);
}
static int sm_find(const str_map *m, const char *s, size_t n, uint32_t *id) {
    for (size_t i = str_hash(s, n) & (m->cap - 1);; i = (i + 1) & (m->cap - 1)) {
        if (!m->keys[i]) return 0;
        if (m->lens[i] == n && memcmp(m->keys[i], s, n) == 0) {
            *id = m->ids[i];
            return 1;
        }
    }
}
static uint32_t sm_get_or_insert(str_map *m, const char *s, size_t n) {
    uint32_t id;
    if (sm_find(m, s, n, &id)) return id;
    if ((m->n + 1) * 2 > m->cap) {
        str_map big;
        big.cap = m->cap * 2;
        big.n = m->n;
        big.keys = (char **)xcalloc(big.cap, sizeof(char *));
        big.lens = (size_t *)xcalloc(big.cap, sizeof(size_t));
        big.ids = (uint32_t *)xcalloc(big.cap, sizeof(uint32_t));
        for (size_t i = 0; i < m->cap; i++)
            if (m->keys[i]) {
                size_t j = str_hash(m->keys[i], m->lens[i]) & (big.cap - 1);
                while (big.keys[j]) j = (j + 1) & (big.cap - 1);
                big.keys[j] = m->keys[i];
                big.lens[j] = m->lens[i];
                big.ids[j] = m->ids[i];
            }
        free(m->keys);
        free(m->lens);
        free(m->ids);
        *m = big;
    }
    size_t i = str_hash(s, n) & (m->cap - 1);
    while (m->keys[i]) i = (i + 1) & (m->cap - 1);
    m->keys[i] = (char *)xmalloc(n + 1);
    memcpy(m->keys[i], s, n);
    m->keys[i][n] = 0;
    m->lens[i] = n;
    m->ids[i] = (uint32_t)m->n; /* new id = map.len() before the insert (raw_connector.rs:297,303) */
    return (uint32_t)m->n++;
}

typedef struct {
    uint32_t k1, k2;
    int32_t cost;
} sc_triple;

typedef struct {
    sc_triple t;
    size_t idx;
} sc_dec;

static int sc_triple_cmp(const void *a_, const void *b_);
static int sc_dec_cmp(const void *a_, const void *b_) { /* (k1, k2, insertion index) */
    const sc_dec *a = (const sc_dec *)a_, *b = (const sc_dec *)b_;
    int c = sc_triple_cmp(&a->t, &b->t);
    if (c) return c;
    return a->idx < b->idx ? -1 : (a->idx > b->idx ? 1 : 0);
}

static int sc_triple_cmp(const void *a_, const void *b_) {
    const sc_triple *a = (const sc_triple *)a_, *b = (const sc_triple *)b_;
    if (a->k1 != b->k1) return a->k1 < b->k1 ? -1 : 1;
    if (a->k2 != b->k2) return a->k2 < b->k2 ? -1 : 1;
    return 0;
}

/* ScorerBuilder::build (scorer.rs:133-168): per key1 in ascending order the smallest base whose
 * slots base^key2 are all unused (slots past the current end count as unused).  `t` holds the
 * insertions in order; a later insert of the same (key1, key2) replaces the earlier cost
 * (BTreeMap::insert, scorer.rs:115-121). */
static void scorer_build(vo_dict *d, sc_triple *t, size_t n) {
    /* BTreeMap order per key1; of equal (k1, k2) inserts the LAST cost stays */
    sc_dec *v = (sc_dec *)xmalloc((n ? n : 1) * sizeof(sc_dec));
    for (size_t i = 0; i < n; i++) {
        v[i].t = t[i];
        v[i].idx = i;
    }
    qsort(v, n, sizeof(sc_dec), sc_dec_cmp);
    size_t m = 0;
    for (size_t i = 0; i < n; i++) {
        if (i + 1 < n && v[i + 1].t.k1 == v[i].t.k1 && v[i + 1].t.k2 == v[i].t.k2) continue; /* a later insert wins */
        t[m++] = v[i].t;
    }
    free(v);
    uint32_t max_k1 = 0;
    for (size_t i = 0; i < m; i++)
        if (t[i].k1 > max_k1) max_k1 = t[i].k1;
    d->n_bases = m ? max_k1 + 1 : 0; /* trie.resize(key1 + 1) scorer.rs:117-119 */
    d->sc_bases = (uint32_t *)xcalloc(d->n_bases ? d->n_bases : 1, sizeof(uint32_t));
    size_t cap = 1024;
    d->sc_checks = (uint32_t *)xmalloc(cap * sizeof(uint32_t));
    d->sc_costs = (int32_t *)xmalloc(cap * sizeof(int32_t));
    size_t len = 0;
    for (size_t i = 0; i < m;) {
        size_t j = i;
        while (j < m && t[j].k1 == t[i].k1) j++;
        uint32_t base = 0;
        for (;; base++) { /* check_base scorer.rs:123-131 */
            int ok = 1;
            for (size_t q = i; q < j; q++) {
                size_t pos = base ^ t[q].k2;
                if (pos < len && d->sc_checks[pos] != UNUSED_CHECK) {
                    ok = 0;
                    break;
                }
            }
            if (ok) break;
        }
        d->sc_bases[t[i].k1] = base;
        for (size_t q = i; q < j; q++) {
            size_t pos = base ^ t[q].k2;
            if (pos >= len) {
                if (pos + 1 > cap) {
                    while (cap < pos + 1) cap *= 2;
                    d->sc_checks = (uint32_t *)xrealloc(d->sc_checks, cap * sizeof(uint32_t));
                    d->sc_costs = (int32_t *)xrealloc(d->sc_costs, cap * sizeof(int32_t));
                }
                for (size_t z = len; z <= pos; z++) {
                    d->sc_checks[z] = UNUSED_CHECK;
                    d->sc_costs[z] = 0;
                }
                len = pos + 1;
            }
            d->sc_checks[pos] = t[i].k1;
            d->sc_costs[pos] = t[q].cost;
        }
        i = j;
    }
    d->n_checks = (uint32_t)len;
}

int32_t vo_scorer_accumulate(const uint32_t *triples, size_t n_triples, const uint32_t *keys1, const uint32_t *keys2,
                             size_t n_keys) {
    vo_dict d;
    memset(&d, 0, sizeof(d));
    sc_triple *t = (sc_triple *)xmalloc((n_triples ? n_triples : 1) * sizeof(sc_triple));
    for (size_t i = 0; i < n_triples; i++) t[i] = (sc_triple){triples[3 * i], triples[3 * i + 1], (int32_t)triples[3 * i + 2]};
    scorer_build(&d, t, n_triples);
    free(t);
    d.feat_T = (uint32_t)n_keys;
    d.right_feats = (uint32_t *)keys1;
    d.left_feats = (uint32_t *)keys2;
    int32_t r = raw_conn_cost(&d, 0, 0);
    free(d.sc_bases);
    free(d.sc_checks);
    free(d.sc_costs);
    return r;
}

/* utils::parse_csv_row (utils.rs:41-61): the fields of one csv row (no record terminator inside) */
static size_t parse_csv_row(const char *row, size_t n, char out[][CSV_FIELD_MAX + 8], size_t *out_len, size_t cap) {
    size_t pos = 0, cnt = 0;
    int start = 1, rec_end, at_eof;
    if (n == 0) { /* read_field on empty input reports End; the row still yields one empty field */
        if (cap) out_len[0] = 0;
        return 1;
    }
    for (;;) {
        size_t nout;
        char *dst = cnt < cap ? out[cnt] : out[cap - 1];
        int r = csv_read_field(row, n, &pos, &start, dst, &nout, &rec_end, &at_eof);
        if (r <= 0) break;
        if (cnt < cap) out_len[cnt] = nout;
        cnt++;
        if (rec_end) break;
    }
    return cnt;
}

#define MAX_TEMPLATES 256

/* RawConnectorBuilder::parse_features (raw_connector.rs:252-274) */
static int parse_feature_line(const char *line, size_t n, const str_map *ids, uint32_t *id_out, uint32_t *feats,
                              uint32_t *n_feats) {
    const char *tab = (const char *)memchr(line, '\t', n);
    if (!tab) return 0;
    if (memchr(tab + 1, '\t', n - (size_t)(tab + 1 - line))) return 0;
    long id;
    if (!parse_int_strict(line, (size_t)(tab - line), 0, 1L << 40, &id)) return -1;
    static __thread char fields[MAX_TEMPLATES][CSV_FIELD_MAX + 8];
    static __thread size_t flen[MAX_TEMPLATES];
    size_t k = parse_csv_row(tab + 1, n - (size_t)(tab + 1 - line), fields, flen, MAX_TEMPLATES);
    if (k > MAX_TEMPLATES) return 0;
    for (size_t i = 0; i < k; i++) {
        uint32_t fid;
        feats[i] = sm_find(ids, fields[i], flen[i], &fid) ? fid : INVALID_FEATURE_ID;
    }
    *n_feats = (uint32_t)k;
    *id_out = (uint32_t)id;
    return 1;
}

/* RawConnectorBuilder (raw_connector.rs:163-245): what bigram.{right,left,cost} hold before any padding */
typedef struct {
    uint32_t *rrows, *lrows, *rlen, *llen; /* rows of MAX_TEMPLATES ids; row i belongs to connection id i + 1 */
    uint32_t n_right, n_left, T;           /* T = longest row (feat_template_size) */
    sc_triple *tri;                        /* ScorerBuilder::insert calls in order */
    size_t n_tri;
    uint32_t trie_len; /* ScorerBuilder::trie.len() */
} bigram_info;

static void bigram_info_free(bigram_info *bi) {
    free(bi->tri);
    free(bi->rrows);
    free(bi->lrows);
    free(bi->rlen);
    free(bi->llen);
}

static int bigram_parse(bigram_info *bi, const char *right, size_t right_len, const char *left, size_t left_len,
                        const char *cost, size_t cost_len, char *err, size_t errcap) {
    memset(bi, 0, sizeof(*bi));
    str_map rmap, lmap;
    sm_init(&rmap);
    sm_init(&lmap);
    sm_get_or_insert(&rmap, "", 0); /* raw_connector.rs:197-198 */
    sm_get_or_insert(&lmap, "", 0);
    sc_triple *tri = NULL;
    size_t n_tri = 0, cap_tri = 0;
    int rc = -1;
    uint32_t *rrows = NULL, *lrows = NULL, *rlen = NULL, *llen = NULL;
    size_t pos = 0, n;
    const char *line;
    while (next_line(cost, cost_len, &pos, &line, &n)) { /* parse_cost raw_connector.rs:276-321 */
        const char *tab = (const char *)memchr(line, '\t', n);
        long c;
        if (!tab || memchr(tab + 1, '\t', n - (size_t)(tab + 1 - line))) {
            set_err(err, errcap, "InvalidFormat(bigram.cost): The format must be right/left<tab>cost");
            goto done;
        }
        if (!parse_int_strict(tab + 1, n - (size_t)(tab + 1 - line), -2147483648L, 2147483647L, &c)) {
            set_err(err, errcap, "ParseInt(bigram.cost): invalid cost");
            goto done;
        }
        const char *slash = (const char *)memchr(line, '/', (size_t)(tab - line));
        if (!slash || memchr(slash + 1, '/', (size_t)(tab - slash - 1))) {
            set_err(err, errcap, "InvalidFormat(bigram.cost): The format must be right/left<tab>cost");
            goto done;
        }
        uint32_t rid = sm_get_or_insert(&rmap, line, (size_t)(slash - line));
        uint32_t lid = sm_get_or_insert(&lmap, slash + 1, (size_t)(tab - slash - 1));
        if (n_tri == cap_tri) {
            cap_tri = cap_tri ? cap_tri * 2 : 1024;
            tri = (sc_triple *)xrealloc(tri, cap_tri * sizeof(sc_triple));
        }
        tri[n_tri++] = (sc_triple){rid, lid, (int32_t)c};
    }
    uint32_t T = 0, n_right = 0, n_left = 0;
    for (int side = 0; side < 2; side++) { /* raw_connector.rs:212-240 */
        const char *txt = side == 0 ? right : left;
        size_t tlen = side == 0 ? right_len : left_len;
        const str_map *ids = side == 0 ? &rmap : &lmap;
        uint32_t *rows = NULL, *lens = NULL, cnt = 0, cap = 0;
        pos = 0;
        while (next_line(txt, tlen, &pos, &line, &n)) {
            uint32_t id, nf, feats[MAX_TEMPLATES];
            int r = parse_feature_line(line, n, ids, &id, feats, &nf);
            if (r <= 0) {
                set_err(err, errcap, r < 0 ? "ParseInt(bigram): invalid id" : "InvalidFormat(bigram): The format must be id<tab>csv_row");
                free(rows);
                free(lens);
                goto done;
            }
            if (id != cnt + 1) {
                set_err(err, errcap, "InvalidFormat(bigram): must be ascending order");
                free(rows);
                free(lens);
                goto done;
            }
            if (cnt == cap) {
                cap = cap ? cap * 2 : 256;
                rows = (uint32_t *)xrealloc(rows, (size_t)cap * MAX_TEMPLATES * sizeof(uint32_t));
                lens = (uint32_t *)xrealloc(lens, (size_t)cap * sizeof(uint32_t));
            }
            memcpy(rows + (size_t)cnt * MAX_TEMPLATES, feats, nf * sizeof(uint32_t));
            lens[cnt++] = nf;
            if (nf > T) T = nf;
        }
        if (side == 0) {
            rrows = rows;
            rlen = lens;
            n_right = cnt;
        } else {
            lrows = rows;
            llen = lens;
            n_left = cnt;
        }
    }
    bi->rrows = rrows, bi->lrows = lrows, bi->rlen = rlen, bi->llen = llen;
    bi->n_right = n_right, bi->n_left = n_left, bi->T = T;
    bi->tri = tri, bi->n_tri = n_tri;
    for (size_t i = 0; i < n_tri; i++)
        if (tri[i].k1 + 1 > bi->trie_len) bi->trie_len = tri[i].k1 + 1;
    tri = NULL, rrows = lrows = rlen = llen = NULL;
    rc = 0;
done:
    free(tri);
    free(rrows);
    free(lrows);
    free(rlen);
    free(llen);
    sm_free(&rmap);
    sm_free(&lmap);
    return rc;
}

/* RawConnector::from_readers (raw_connector.rs:45-105) */
static void raw_from_bigram(vo_dict *d, bigram_info *bi) {
    uint32_t T = bi->T, n_right = bi->n_right, n_left = bi->n_left;
    uint32_t *rrows = bi->rrows, *lrows = bi->lrows, *rlen = bi->rlen, *llen = bi->llen;
    if (T != 0) T = ((T - 1) / 8 + 1) * 8; /* raw_connector.rs:64-66: next multiple of SIMD_SIZE */
    d->feat_T = T;
    d->num_right = n_right + 1;
    d->num_left = n_left + 1;
    d->right_feats = (uint32_t *)xmalloc(((size_t)d->num_right * T + 1) * sizeof(uint32_t));
    d->left_feats = (uint32_t *)xmalloc(((size_t)d->num_left * T + 1) * sizeof(uint32_t));
    for (size_t i = 0; i < (size_t)d->num_right * T; i++) d->right_feats[i] = i < T ? 0 : INVALID_FEATURE_ID; /* :72-79 */
    for (size_t i = 0; i < (size_t)d->num_left * T; i++) d->left_feats[i] = i < T ? 0 : INVALID_FEATURE_ID;
    for (uint32_t i = 0; i < n_right; i++)
        memcpy(d->right_feats + (size_t)(i + 1) * T, rrows + (size_t)i * MAX_TEMPLATES, rlen[i] * sizeof(uint32_t));
    for (uint32_t i = 0; i < n_left; i++)
        memcpy(d->left_feats + (size_t)(i + 1) * T, lrows + (size_t)i * MAX_TEMPLATES, llen[i] * sizeof(uint32_t));
    scorer_build(d, bi->tri, bi->n_tri);
}

/* ------------------------------------------------------------------------------------------ */
/* DualConnector from bigram.{right,left,cost} (connector/dual_connector.rs)                     */
/* ------------------------------------------------------------------------------------------ */

/* one row projected on a template subset: key[0] = length, then the kept feature ids */
static __thread size_t g_key_words;
static int key_cmp(const void *a, const void *b) { return memcmp(a, b, g_key_words * sizeof(uint32_t)); }

/* number of distinct projections of `rows` on the templates in `in` other than `trial`; templates past a
 * row's end contribute nothing (`row.get(i)` is None, dual_connector.rs:45-53) */
static size_t distinct_rows(const uint32_t *rows, const uint32_t *lens, uint32_t n, uint32_t T, const char *in,
                            uint32_t trial, uint32_t *scratch) {
    size_t kw = (size_t)T + 1;
    for (uint32_t r = 0; r < n; r++) {
        uint32_t *key = scratch + (size_t)r * kw, m = 0;
        memset(key, 0, kw * sizeof(uint32_t));
        for (uint32_t i = 0; i < T && i < lens[r]; i++)
            if (in[i] && i != trial) key[1 + m++] = rows[(size_t)r * MAX_TEMPLATES + i];
        key[0] = m;
    }
    g_key_words = kw;
    qsort(scratch, n, kw * sizeof(uint32_t), key_cmp);
    size_t cnt = 0;
    for (uint32_t r = 0; r < n; r++)
        if (r == 0 || memcmp(scratch + (size_t)r * kw, scratch + (size_t)(r - 1) * kw, kw * sizeof(uint32_t)) != 0) cnt++;
    return cnt;
}

/* DualConnector::remove_feature_templates_greedy (dual_connector.rs:27-70).  The reference iterates a
 * hashbrown HashSet, so among equally good templates its pick follows that set's internal order; this
 * restatement walks the templates in ascending index and lets `<=` keep the last minimum.  Which
 * templates go where does not change DualConnector::cost (it is the sum over all templates either way)
 * except through the i16 clamp of the matrix part (dual_connector.rs:104). */
static void dual_choose_templates(const bigram_info *bi, char *in) {
    uint32_t T = bi->T;
    uint32_t nmax = bi->n_right > bi->n_left ? bi->n_right : bi->n_left;
    uint32_t *scratch = (uint32_t *)xmalloc(((size_t)nmax + 1) * ((size_t)T + 1) * sizeof(uint32_t));
    memset(in, 1, T);
    for (int round = 0; round < 8; round++) { /* SIMD_SIZE templates move to the raw part */
        uint32_t cand = 0;
        size_t best = (size_t)bi->n_left * bi->n_right;
        for (uint32_t trial = 0; trial < T; trial++) {
            if (!in[trial]) continue;
            size_t sz = distinct_rows(bi->rrows, bi->rlen, bi->n_right, T, in, trial, scratch) *
                        distinct_rows(bi->lrows, bi->llen, bi->n_left, T, in, trial, scratch);
            if (sz <= best) {
                best = sz;
                cand = trial;
            }
        }
        in[cand] = 0;
    }
    free(scratch);
}

/* generate_feature_map of create_matrix_connector (dual_connector.rs:79-94): matrix id per connection id in
 * first-seen order, id 0 = the all-zero row; returns the distinct projected rows (P ids each, zero padded
 * like U31x8::to_simd_vec, scorer.rs:27-46). */
static uint32_t *dual_feature_map(const uint32_t *rows, const uint32_t *lens, uint32_t n, const uint32_t *midx, uint32_t nm,
                                  uint32_t P, uint16_t **conn_map_out, uint32_t *n_ids_out, int *overflow) {
    uint32_t cap = 64, n_ids = 1;
    uint32_t *uniq = (uint32_t *)xcalloc((size_t)cap * (P ? P : 1), sizeof(uint32_t));
    uint16_t *conn_map = (uint16_t *)xcalloc((size_t)n + 1, sizeof(uint16_t));
    uint32_t *feats = (uint32_t *)xcalloc(P ? P : 1, sizeof(uint32_t));
    for (uint32_t r = 0; r < n; r++) {
        memset(feats, 0, (P ? P : 1) * sizeof(uint32_t));
        for (uint32_t k = 0; k < nm; k++)
            feats[k] = midx[k] < lens[r] ? rows[(size_t)r * MAX_TEMPLATES + midx[k]] : INVALID_FEATURE_ID;
        uint32_t id = 0;
        for (; id < n_ids; id++)
            if (memcmp(uniq + (size_t)id * P, feats, nm * sizeof(uint32_t)) == 0) break;
        if (id == n_ids) {
            if (n_ids == cap) {
                cap *= 2;
                uniq = (uint32_t *)xrealloc(uniq, (size_t)cap * (P ? P : 1) * sizeof(uint32_t));
            }
            memcpy(uniq + (size_t)n_ids * P, feats, P * sizeof(uint32_t));
            n_ids++;
        }
        if (id > 0xFFFF) *overflow = 1; /* u16::try_from(conn_id).unwrap() dual_connector.rs:91 */
        conn_map[r + 1] = (uint16_t)id;
    }
    free(feats);
    *conn_map_out = conn_map;
    *n_ids_out = n_ids;
    return uniq;
}

/* DualConnector::from_readers (dual_connector.rs:155-213) */
static int dual_from_bigram(vo_dict *d, bigram_info *bi, char *err, size_t errcap) {
    uint32_t T = bi->T;
    if (T < 8) { /* `feat_template_size - SIMD_SIZE` (dual_connector.rs:82) would underflow */
        set_err(err, errcap, "InvalidArgument(bigram): the Dual connector needs at least 8 feature templates");
        return -1;
    }
    /* the scorer over every pair (dual_connector.rs:167) */
    vo_dict full;
    memset(&full, 0, sizeof(full));
    sc_triple *tcopy = (sc_triple *)xmalloc((bi->n_tri ? bi->n_tri : 1) * sizeof(sc_triple));
    memcpy(tcopy, bi->tri, bi->n_tri * sizeof(sc_triple));
    scorer_build(&full, tcopy, bi->n_tri);
    free(tcopy);

    char in[MAX_TEMPLATES];
    dual_choose_templates(bi, in);
    uint32_t midx[MAX_TEMPLATES], ridx[MAX_TEMPLATES], nm = 0, nraw = 0;
    for (uint32_t i = 0; i < T; i++) {
        if (in[i]) midx[nm++] = i;
        else ridx[nraw++] = i;
    }

    /* create_matrix_connector (dual_connector.rs:72-110) */
    uint32_t P = (nm + 7) / 8 * 8, n_rids, n_lids;
    int overflow = 0;
    uint32_t *rfeat = dual_feature_map(bi->rrows, bi->rlen, bi->n_right, midx, nm, P, &d->dual_rmap, &n_rids, &overflow);
    uint32_t *lfeat = dual_feature_map(bi->lrows, bi->llen, bi->n_left, midx, nm, P, &d->dual_lmap, &n_lids, &overflow);
    if (overflow) {
        set_err(err, errcap, "TryFromInt(bigram): the reduced matrix has too many ids");
        free(rfeat);
        free(lfeat);
        free(full.sc_bases);
        free(full.sc_checks);
        free(full.sc_costs);
        return -1;
    }
    d->m_num_right = n_rids;
    d->m_num_left = n_lids;
    d->matrix = (int16_t *)xcalloc((size_t)n_rids * n_lids, sizeof(int16_t));
    full.feat_T = P;
    full.right_feats = rfeat;
    full.left_feats = lfeat;
    for (uint32_t l = 0; l < n_lids; l++)
        for (uint32_t r = 0; r < n_rids; r++) {
            int32_t c = raw_conn_cost(&full, r, l);
            d->matrix[(size_t)l * n_rids + r] = (int16_t)(c < -32768 ? -32768 : c > 32767 ? 32767 : c); /* :104 */
        }
    free(rfeat);
    free(lfeat);
    free(full.sc_bases);
    free(full.sc_checks);
    free(full.sc_costs);

    /* create_raw_connector (dual_connector.rs:112-153): a zero row for BOS/EOS, then the 8 raw templates per id */
    d->feat_T = 8;
    d->num_right = bi->n_right + 1;
    d->num_left = bi->n_left + 1;
    d->right_feats = (uint32_t *)xcalloc((size_t)d->num_right * 8 + 1, sizeof(uint32_t));
    d->left_feats = (uint32_t *)xcalloc((size_t)d->num_left * 8 + 1, sizeof(uint32_t));
    for (uint32_t r = 0; r < bi->n_right; r++)
        for (uint32_t k = 0; k < 8; k++)
            d->right_feats[(size_t)(r + 1) * 8 + k] =
                ridx[k] < bi->rlen[r] ? bi->rrows[(size_t)r * MAX_TEMPLATES + ridx[k]] : INVALID_FEATURE_ID;
    for (uint32_t l = 0; l < bi->n_left; l++)
        for (uint32_t k = 0; k < 8; k++)
            d->left_feats[(size_t)(l + 1) * 8 + k] =
                ridx[k] < bi->llen[l] ? bi->lrows[(size_t)l * MAX_TEMPLATES + ridx[k]] : INVALID_FEATURE_ID;
    /* the raw scorer keeps a pair only when both of its ids occur in the raw rows (:137-152) */
    uint32_t max_k2 = 0;
    for (size_t i = 0; i < bi->n_tri; i++)
        if (bi->tri[i].k2 > max_k2) max_k2 = bi->tri[i].k2;
    char *r_used = (char *)xcalloc((size_t)bi->trie_len + 1, 1), *l_used = (char *)xcalloc((size_t)max_k2 + 2, 1);
    for (size_t q = 0; q < (size_t)d->num_right * 8; q++)
        if (d->right_feats[q] < bi->trie_len) r_used[d->right_feats[q]] = 1;
    for (size_t q = 0; q < (size_t)d->num_left * 8; q++)
        if (d->left_feats[q] <= max_k2) l_used[d->left_feats[q]] = 1;
    size_t kept = 0;
    for (size_t i = 0; i < bi->n_tri; i++)
        if (r_used[bi->tri[i].k1] && l_used[bi->tri[i].k2]) bi->tri[kept++] = bi->tri[i];
    free(r_used);
    free(l_used);
    scorer_build(d, bi->tri, kept);
    if (d->n_bases < bi->trie_len) { /* emptied key1 maps still own a base slot (bases = vec![0; trie.len()]) */
        d->sc_bases = (uint32_t *)xrealloc(d->sc_bases, (size_t)bi->trie_len * sizeof(uint32_t));
        for (uint32_t i = d->n_bases; i < bi->trie_len; i++) d->sc_bases[i] = 0;
        d->n_bases = bi->trie_len;
    }
    return 0;
}

vo_dict *vo_dict_from_bigram(const char *lex_csv, size_t lex_len, const char *bigram_right, size_t right_len,
                             const char *bigram_left, size_t left_len, const char *bigram_cost, size_t cost_len,
                             const char *char_def, size_t char_len, const char *unk_def, size_t unk_len, char *err,
                             size_t errcap) {
    vo_dict *d = (vo_dict *)xcalloc(1, sizeof(vo_dict));
    bigram_info bi;
    if (bigram_parse(&bi, bigram_right, right_len, bigram_left, left_len, bigram_cost, cost_len, err, errcap) != 0) {
        vo_dict_free(d);
        return NULL;
    }
    raw_from_bigram(d, &bi);
    bigram_info_free(&bi);
    return dict_finish(d, lex_csv, lex_len, char_def, char_len, unk_def, unk_len, err, errcap);
}

vo_dict *vo_dict_from_bigram_dual(const char *lex_csv, size_t lex_len, const char *bigram_right, size_t right_len,
                                  const char *bigram_left, size_t left_len, const char *bigram_cost, size_t cost_len,
                                  const char *char_def, size_t char_len, const char *unk_def, size_t unk_len, char *err,
                                  size_t errcap) {
    vo_dict *d = (vo_dict *)xcalloc(1, sizeof(vo_dict));
    bigram_info bi;
    if (bigram_parse(&bi, bigram_right, right_len, bigram_left, left_len, bigram_cost, cost_len, err, errcap) != 0) {
        vo_dict_free(d);
        return NULL;
    }
    int rc = dual_from_bigram(d, &bi, err, errcap);
    bigram_info_free(&bi);
    if (rc != 0) {
        vo_dict_free(d);
        return NULL;
    }
    return dict_finish(d, lex_csv, lex_len, char_def, char_len, unk_def, unk_len, err, errcap);
}
