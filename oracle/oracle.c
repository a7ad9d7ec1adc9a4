/*
 * oracle.c — single-threaded CPU restatement of the TinySQL vectorized-execution hot path.
 *
 * TEST INFRASTRUCTURE ONLY (see oracle.h).  Written for obviousness, not speed.
 * Compile with -fwrapv: Go integer arithmetic wraps, C's is undefined.
 * Paths in comments are relative to the reference repository (pingcap-incubator/tinysql).
 */
#include "oracle.h"
#include <math.h>
#include <stdlib.h>
#include <string.h>

#define DBL_MAX_ 1.7976931348623157e308 /* math.MaxFloat64 */

/* ------------------------------------------------------------------ column helpers */
/* util/chunk/column.go:89-92 IsNull: bit == 0 means NULL */
static inline int col_is_null(const orc_column *c, int64_t i) {
  if (!c->null_bitmap) return 0;
  return !((c->null_bitmap[i >> 3] >> (i & 7)) & 1);
}
static inline void col_set_null(orc_column *c, int64_t i, int is_null) {
  if (is_null) c->null_bitmap[i >> 3] &= (uint8_t)~(1u << (i & 7));
  else c->null_bitmap[i >> 3] |= (uint8_t)(1u << (i & 7));
}
static inline int64_t col_i64(const orc_column *c, int64_t i) { return ((const int64_t *)c->data)[i]; }
static inline uint64_t col_u64(const orc_column *c, int64_t i) { return ((const uint64_t *)c->data)[i]; }
static inline double col_f64(const orc_column *c, int64_t i) { return ((const double *)c->data)[i]; }

/* out column preparation == Column.ResizeInt64(n, false) (util/chunk/column.go:241-249,331):
 * all rows start NOT NULL; we additionally keep the tail bits of the last byte 0. */
static void out_init(orc_column *o, int64_t n) {
  o->length = n;
  int64_t nb = (n + 7) >> 3;
  memset(o->null_bitmap, 0xFF, (size_t)nb);
  if (n & 7) o->null_bitmap[nb - 1] = (uint8_t)((1u << (n & 7)) - 1);
}
/* Column.MergeNulls (util/chunk/column.go:559-574): result.null |= arg.null */
static void merge_nulls(orc_column *o, const orc_column *a, int64_t n) {
  for (int64_t i = 0; i < n; i++)
    if (col_is_null(a, i)) col_set_null(o, i, 1);
}

/* ------------------------------------------------------------------ key encoding + FNV-1 */
enum { NIL_FLAG = 0, COMPACT_BYTES_FLAG = 2, FLOAT_FLAG = 5, VARINT_FLAG = 8, UVARINT_FLAG = 9 }; /* util/codec/codec.go:32-45 */

/* encodeHashChunkRowIdx (util/codec/codec.go:212-240): (flag, raw bytes).  *raw holds the 8 raw bytes of the fixed-width
 * types; for the var-len types (*bytes, *blen) is the cell (row.GetBytes). */
static int encode_key(int type, const orc_column *c, int64_t row, uint8_t *flag, uint64_t *raw, const uint8_t **bytes, int64_t *blen) {
  *bytes = NULL; *blen = 8;
  if (col_is_null(c, row)) { *flag = NIL_FLAG; *raw = 0; *blen = 0; return 1; }
  switch (type) {
    case ORC_TYPE_INT64: *raw = col_u64(c, row); *flag = VARINT_FLAG; break;
    case ORC_TYPE_UINT64: *raw = col_u64(c, row); *flag = (col_i64(c, row) < 0) ? UVARINT_FLAG : VARINT_FLAG; break; /* :220-224 */
    case ORC_TYPE_FLOAT64: *raw = col_u64(c, row); *flag = FLOAT_FLAG; break;
    case ORC_TYPE_FLOAT32: { /* :226-229: f := float64(row.GetFloat32(idx)) */
      float f; memcpy(&f, c->data + 4 * row, 4);
      double d = (double)f; memcpy(raw, &d, 8); *flag = FLOAT_FLAG; break;
    }
    case ORC_TYPE_BYTES: /* :230-233 compactBytesFlag + row.GetBytes(idx) */
      *flag = COMPACT_BYTES_FLAG; *raw = 0; *bytes = c->data + c->offsets[row]; *blen = c->offsets[row + 1] - c->offsets[row]; break;
    default: *flag = 0xFF; *raw = 0; break;
  }
  return 0;
}

/* Go hash/fnv New64(): FNV-1 (multiply then xor); restated in-repo at util/mvmap/fnv.go:16-29 */
static inline uint64_t fnv1_byte(uint64_t h, uint8_t b) { return (h * 1099511628211ULL) ^ b; }

uint64_t orc_hash_row(int n_keys, const int *types, const orc_column *cols, const int *key_idx, int64_t row,
                      int *has_null) {
  uint64_t h = 14695981039346656037ULL;
  int hn = 0;
  for (int k = 0; k < n_keys; k++) {
    int ci = key_idx[k];
    uint8_t flag; uint64_t raw; const uint8_t *bytes; int64_t blen;
    int isnull = encode_key(types[ci], &cols[ci], row, &flag, &raw, &bytes, &blen);
    h = fnv1_byte(h, flag);                     /* h[i].Write(buf)  codec.go:273 */
    if (isnull) { hn = 1; continue; }           /* b = nil; isNull[i] = true  codec.go:263-264 */
    if (flag == COMPACT_BYTES_FLAG) { for (int64_t b = 0; b < blen; b++) h = fnv1_byte(h, bytes[b]); }  /* h[i].Write(column.GetBytes(i)) codec.go:330-331 */
    else for (int b = 0; b < 8; b++) h = fnv1_byte(h, (uint8_t)(raw >> (8 * b))); /* h[i].Write(b) little-endian raw */
  }
  if (has_null) *has_null = hn;
  return h;
}

int orc_equal_row(int n_keys, const int *types1, const orc_column *cols1, const int *idx1, int64_t row1,
                  const int *types2, const orc_column *cols2, const int *idx2, int64_t row2) {
  for (int k = 0; k < n_keys; k++) { /* util/codec/codec.go:367-380: flag1 == flag2 && bytes.Equal(b1, b2) */
    uint8_t f1, f2; uint64_t r1, r2; const uint8_t *b1, *b2; int64_t l1, l2;
    int n1 = encode_key(types1[idx1[k]], &cols1[idx1[k]], row1, &f1, &r1, &b1, &l1);
    int n2 = encode_key(types2[idx2[k]], &cols2[idx2[k]], row2, &f2, &r2, &b2, &l2);
    if (f1 != f2) return 0;
    if (n1 != n2) return 0;
    if (n1) continue;
    if (l1 != l2) return 0;
    if (f1 == COMPACT_BYTES_FLAG) { if (l1 && memcmp(b1, b2, (size_t)l1)) return 0; }
    else if (r1 != r2) return 0;
  }
  return 1;
}

/* ------------------------------------------------------------------ rowHashMap */
/* executor/hash_table.go:181-272.  Go's map[uint64]entryAddr is an associative container;
 * here an open-addressed table keyed by the 64-bit hash, value = head entry index.
 * Entries form a chain through `next` (newest first); Get reverses to insertion order. */
typedef struct { uint32_t chk, row; int64_t next; } rm_entry;
struct orc_rowmap {
  uint64_t *keys; int64_t *heads; uint8_t *used; int64_t cap, n_keys;
  rm_entry *entries; int64_t n_entries, cap_entries;
};
orc_rowmap *orc_rowmap_new(void) {
  orc_rowmap *m = (orc_rowmap *)calloc(1, sizeof(*m));
  m->cap = 1024;
  m->keys = (uint64_t *)calloc((size_t)m->cap, 8); m->heads = (int64_t *)calloc((size_t)m->cap, 8);
  m->used = (uint8_t *)calloc((size_t)m->cap, 1);
  m->cap_entries = 1024; m->entries = (rm_entry *)malloc(sizeof(rm_entry) * (size_t)m->cap_entries);
  return m;
}
static int64_t rm_find(const orc_rowmap *m, uint64_t k) {
  uint64_t x = k * 0x9E3779B97F4A7C15ULL;
  int64_t i = (int64_t)(x >> 20) & (m->cap - 1);
  while (m->used[i] && m->keys[i] != k) i = (i + 1) & (m->cap - 1);
  return i;
}
static void rm_grow(orc_rowmap *m) {
  int64_t oc = m->cap; uint64_t *ok = m->keys; int64_t *oh = m->heads; uint8_t *ou = m->used;
  m->cap = oc * 2;
  m->keys = (uint64_t *)calloc((size_t)m->cap, 8); m->heads = (int64_t *)calloc((size_t)m->cap, 8);
  m->used = (uint8_t *)calloc((size_t)m->cap, 1);
  for (int64_t i = 0; i < oc; i++) if (ou[i]) { int64_t s = rm_find(m, ok[i]); m->used[s] = 1; m->keys[s] = ok[i]; m->heads[s] = oh[i]; }
  free(ok); free(oh); free(ou);
}
void orc_rowmap_put(orc_rowmap *m, uint64_t hash_key, uint32_t chk_idx, uint32_t row_idx) {
  if ((m->n_keys + 1) * 2 > m->cap) rm_grow(m);
  int64_t s = rm_find(m, hash_key);
  int64_t old = -1;                               /* nullEntryAddr */
  if (m->used[s]) old = m->heads[s]; else { m->used[s] = 1; m->keys[s] = hash_key; m->n_keys++; }
  if (m->n_entries == m->cap_entries) { m->cap_entries *= 2; m->entries = (rm_entry *)realloc(m->entries, sizeof(rm_entry) * (size_t)m->cap_entries); }
  rm_entry e = { chk_idx, row_idx, old };          /* e.next = oldEntryAddr  hash_table.go:249-252 */
  m->entries[m->n_entries] = e;
  m->heads[s] = m->n_entries++;                    /* m.hashTable[hashKey] = newEntryAddr */
}
int64_t orc_rowmap_get(orc_rowmap *m, uint64_t hash_key, uint32_t *pairs, int64_t cap) {
  int64_t s = rm_find(m, hash_key);
  if (!m->used[s]) return 0;
  int64_t cnt = 0;
  for (int64_t e = m->heads[s]; e != -1; e = m->entries[e].next) cnt++;
  int64_t pos = cnt;                               /* "Keep the order of input" hash_table.go:266-270 */
  for (int64_t e = m->heads[s]; e != -1; e = m->entries[e].next) {
    pos--;
    if (pos < cap) { pairs[2 * pos] = m->entries[e].chk; pairs[2 * pos + 1] = m->entries[e].row; }
  }
  return cnt;
}
int64_t orc_rowmap_len(orc_rowmap *m) { return m->n_entries; }
void orc_rowmap_free(orc_rowmap *m) { if (!m) return; free(m->keys); free(m->heads); free(m->used); free(m->entries); free(m); }

/* ------------------------------------------------------------------ growable output */
/* One output column under construction.  elem = 8 (every integer type, DOUBLE), 4 (FLOAT) or 0 (var-len: bytes +
 * offsets) — util/chunk/codec.go:171-181 getFixedLen. */
typedef struct {
  uint64_t *data; uint8_t *nn; int64_t n, cap; /* nn: byte per row, 1 = not null */
  int elem;
  uint8_t *bytes; int64_t nbytes, bcap; int64_t *offs; int64_t ocap;
} outbuf;
static int elem_of_type(int t) { return t == ORC_TYPE_FLOAT32 ? 4 : (t == ORC_TYPE_BYTES ? 0 : 8); }
static void ob_push(outbuf *b, uint64_t v, int not_null) {
  if (b->n == b->cap) {
    b->cap = b->cap ? b->cap * 2 : 1024;
    b->data = (uint64_t *)realloc(b->data, 8 * (size_t)b->cap);
    b->nn = (uint8_t *)realloc(b->nn, (size_t)b->cap);
  }
  b->data[b->n] = v; b->nn[b->n] = (uint8_t)not_null; b->n++;
}
/* Append cell `row` of src (row < 0: a NULL cell).  Restates the per-column copy of chunk.CopySelectedJoinRows
 * (util/chunk/chunk_util.go:38-66,84-110): fixed-width cells copy elemLen bytes, var-len cells copy
 * data[offsets[i]:offsets[i+1]] and push the new end offset; the NULL bit travels separately. */
static void ob_push_cell(outbuf *b, const orc_column *src, int64_t row) {
  int not_null = row >= 0 && !col_is_null(src, row);
  if (b->elem == 8) { ob_push(b, row >= 0 ? col_u64(src, row) : 0, not_null); return; }
  if (b->elem == 4) {
    uint32_t v = 0;
    if (row >= 0) memcpy(&v, src->data + 4 * row, 4);
    ob_push(b, v, not_null);
    return;
  }
  int64_t start = 0, end = 0;
  if (row >= 0) { start = src->offsets[row]; end = src->offsets[row + 1]; }
  if (b->nbytes + (end - start) > b->bcap) {
    b->bcap = b->bcap ? b->bcap * 2 : 4096;
    while (b->bcap < b->nbytes + (end - start)) b->bcap *= 2;
    b->bytes = (uint8_t *)realloc(b->bytes, (size_t)b->bcap);
  }
  if (end > start) memcpy(b->bytes + b->nbytes, src->data + start, (size_t)(end - start));
  b->nbytes += end - start;
  if (b->n + 2 > b->ocap) { b->ocap = b->ocap ? b->ocap * 2 : 1024; b->offs = (int64_t *)realloc(b->offs, 8 * (size_t)b->ocap); }
  if (b->n == 0) b->offs[0] = 0;
  b->offs[b->n + 1] = b->nbytes;
  ob_push(b, 0, not_null);
}
static void ob_finish(outbuf *b, orc_column *c) {
  int64_t n = b->n;
  c->length = n; c->offsets = NULL;
  if (b->elem == 8) {
    c->data = (uint8_t *)malloc(8 * (size_t)(n ? n : 1));
    if (n) memcpy(c->data, b->data, 8 * (size_t)n);
  } else if (b->elem == 4) {
    c->data = (uint8_t *)malloc(4 * (size_t)(n ? n : 1));
    for (int64_t i = 0; i < n; i++) { uint32_t v = (uint32_t)b->data[i]; memcpy(c->data + 4 * i, &v, 4); }
  } else {
    c->data = (uint8_t *)malloc((size_t)(b->nbytes ? b->nbytes : 1));
    if (b->nbytes) memcpy(c->data, b->bytes, (size_t)b->nbytes);
    c->offsets = (int64_t *)malloc(8 * (size_t)(n + 1));
    c->offsets[0] = 0;
    if (n) memcpy(c->offsets, b->offs, 8 * (size_t)(n + 1));
  }
  int64_t nb = (n + 7) >> 3;
  c->null_bitmap = (uint8_t *)calloc((size_t)(nb ? nb : 1), 1);
  for (int64_t i = 0; i < n; i++) if (b->nn[i]) c->null_bitmap[i >> 3] |= (uint8_t)(1u << (i & 7));
  free(b->data); free(b->nn); free(b->bytes); free(b->offs);
}
void orc_free_columns(int n, orc_column *cols) {
  for (int i = 0; i < n; i++) {
    free(cols[i].data); free(cols[i].null_bitmap); free(cols[i].offsets);
    cols[i].data = NULL; cols[i].null_bitmap = NULL; cols[i].offsets = NULL;
  }
}

/* ------------------------------------------------------------------ hash join */
static void append_row(outbuf *obs, int base, int ncols, const orc_column *cols, int64_t row) {
  for (int c = 0; c < ncols; c++) ob_push_cell(&obs[base + c], &cols[c], row); /* row < 0: defaultInner, all NULL (builder.go:463-465) */
}

static int cmp_int(int ua, int ub, int64_t x, int64_t y);
static int cmp_f64(double x, double y);
static int64_t cmp_result(int op, int c);

/* One OtherCondition `out[lhs_col] op out[rhs_col]` (or `op constant`) on the joined row lhs ++ rhs.  baseJoiner.filter
 * (joiner.go:155-167) keeps the joined rows for which every condition is TRUE — a NULL operand makes it not true
 * (VectorizedFilter, chunk_executor.go:196-245). */
typedef struct { int type; uint64_t bits; int is_null; } cond_operand;
static cond_operand joined_cell(int o, int outer_is_right, int n_build_cols, const int *bt, const orc_column *bc, int64_t brow,
                                int n_probe_cols, const int *pt, const orc_column *pc, int64_t prow) {
  cond_operand r;
  int first_is_build = outer_is_right;
  int n_first = first_is_build ? n_build_cols : n_probe_cols;
  int from_build = first_is_build ? (o < n_first) : (o >= n_first);
  int c = o < n_first ? o : o - n_first;
  const orc_column *col = from_build ? &bc[c] : &pc[c];
  int64_t row = from_build ? brow : prow;
  r.type = from_build ? bt[c] : pt[c];
  r.is_null = col_is_null(col, row);
  r.bits = r.is_null ? 0 : col_u64(col, row);
  return r;
}
static int conds_true(int n_conds, const orc_join_cond *conds, int outer_is_right, int n_build_cols, const int *bt, const orc_column *bc, int64_t brow,
                      int n_probe_cols, const int *pt, const orc_column *pc, int64_t prow) {
  for (int k = 0; k < n_conds; k++) {
    cond_operand a = joined_cell(conds[k].lhs_col, outer_is_right, n_build_cols, bt, bc, brow, n_probe_cols, pt, pc, prow), b;
    if (conds[k].rhs_col >= 0) b = joined_cell(conds[k].rhs_col, outer_is_right, n_build_cols, bt, bc, brow, n_probe_cols, pt, pc, prow);
    else { b.type = conds[k].const_type; b.bits = conds[k].const_bits; b.is_null = 0; }
    if (a.is_null || b.is_null) return 0;
    int c;
    if (a.type == ORC_TYPE_FLOAT64) { double x, y; memcpy(&x, &a.bits, 8); memcpy(&y, &b.bits, 8); c = cmp_f64(x, y); }
    else c = cmp_int(a.type == ORC_TYPE_UINT64, b.type == ORC_TYPE_UINT64, (int64_t)a.bits, (int64_t)b.bits);
    if (!cmp_result(conds[k].op, c)) return 0;
  }
  return 1;
}

int orc_hash_join(int join_type, int outer_is_right,
                  int n_build_cols, const int *build_types, const orc_column *build_cols,
                  int n_probe_cols, const int *probe_types, const orc_column *probe_cols,
                  int n_keys, const int *build_key_idx, const int *probe_key_idx,
                  const uint8_t *selected, orc_column *out_cols, int64_t *n_out) {
  return orc_hash_join_cond(join_type, outer_is_right, n_build_cols, build_types, build_cols, n_probe_cols, probe_types, probe_cols, n_keys, build_key_idx,
                            probe_key_idx, selected, 0, NULL, out_cols, n_out);
}

int orc_hash_join_cond(int join_type, int outer_is_right,
                       int n_build_cols, const int *build_types, const orc_column *build_cols,
                       int n_probe_cols, const int *probe_types, const orc_column *probe_cols,
                       int n_keys, const int *build_key_idx, const int *probe_key_idx,
                       const uint8_t *selected, int n_conds, const orc_join_cond *conds, orc_column *out_cols, int64_t *n_out) {
  return orc_hash_join_full(join_type, outer_is_right, n_build_cols, build_types, build_cols, n_probe_cols, probe_types, probe_cols, n_keys, build_key_idx,
                            probe_key_idx, selected, n_conds, conds, NULL, NULL, out_cols, n_out);
}

/* default_bits / default_nn: defaultInner (joiner.go:139-143 initDefaultInner from PhysicalHashJoin.DefaultValues): the inner side of
 * a miss row of an outer join; NULL = all NULL (builder.go:463-465) */
int orc_hash_join_full(int join_type, int outer_is_right,
                       int n_build_cols, const int *build_types, const orc_column *build_cols,
                       int n_probe_cols, const int *probe_types, const orc_column *probe_cols,
                       int n_keys, const int *build_key_idx, const int *probe_key_idx,
                       const uint8_t *selected, int n_conds, const orc_join_cond *conds,
                       const uint64_t *default_bits, const uint8_t *default_nn, orc_column *out_cols, int64_t *n_out) {
  if (join_type < 0 || join_type > 2 || n_keys < 1 || n_conds < 0) return ORC_ERR_INVALID;
  for (int k = 0; k < n_conds; k++) {  /* operands: the 8-byte types, integers with integers / doubles with doubles */
    int nt = n_build_cols + n_probe_cols;
    if (conds[k].op < 0 || conds[k].op > 5 || conds[k].lhs_col < 0 || conds[k].lhs_col >= nt || conds[k].rhs_col >= nt) return ORC_ERR_INVALID;
    int o = conds[k].lhs_col, nf = outer_is_right ? n_build_cols : n_probe_cols;
    int ta = (outer_is_right ? (o < nf) : (o >= nf)) ? build_types[o < nf ? o : o - nf] : probe_types[o < nf ? o : o - nf];
    int tb = conds[k].const_type;
    if (conds[k].rhs_col >= 0) { o = conds[k].rhs_col; tb = (outer_is_right ? (o < nf) : (o >= nf)) ? build_types[o < nf ? o : o - nf] : probe_types[o < nf ? o : o - nf]; }
    if (ta < 1 || ta > 3 || tb < 1 || tb > 3 || ((ta == ORC_TYPE_FLOAT64) != (tb == ORC_TYPE_FLOAT64))) return ORC_ERR_UNSUPPORTED;
  }
  for (int c = 0; c < n_build_cols; c++) if (build_types[c] < 1 || build_types[c] > 5) return ORC_ERR_UNSUPPORTED;
  for (int c = 0; c < n_probe_cols; c++) if (probe_types[c] < 1 || probe_types[c] > 5) return ORC_ERR_UNSUPPORTED;
  /* key columns: every supported chunk type (codec.go:216-236: integers, FLOAT as float64(f), DOUBLE, var-len bytes) */
  int64_t nb = n_build_cols ? build_cols[0].length : 0, np = n_probe_cols ? probe_cols[0].length : 0;

  /* fetchAndBuildHashTable [stub join.go:148] + hashRowContainer.PutChunk (hash_table.go:146-169) */
  orc_rowmap *m = orc_rowmap_new();
  for (int64_t i = 0; i < nb; i++) {
    int has_null;
    uint64_t h = orc_hash_row(n_keys, build_types, build_cols, build_key_idx, i, &has_null);
    if (has_null) continue;                                    /* hash_table.go:161-163 */
    orc_rowmap_put(m, h, (uint32_t)(i >> 32), (uint32_t)i);    /* RowPtr; we pack the global row index */
  }

  int ncols = n_build_cols + n_probe_cols;
  outbuf *obs = (outbuf *)calloc((size_t)ncols, sizeof(outbuf));
  /* output = lhs cols ++ rhs cols (joiner.go:145-150, 361-366); outer_is_right => build side is lhs */
  int build_base = outer_is_right ? 0 : n_probe_cols;
  int probe_base = outer_is_right ? n_build_cols : 0;
  int is_outer = (join_type != 0);
  for (int c = 0; c < n_build_cols; c++) obs[build_base + c].elem = elem_of_type(build_types[c]);
  for (int c = 0; c < n_probe_cols; c++) obs[probe_base + c].elem = elem_of_type(probe_types[c]);

  uint32_t *pairs = NULL; int64_t pairs_cap = 0;
  /* runJoinWorker [stub join.go:243] -> join2Chunk (join.go:325-362) */
  for (int64_t i = 0; i < np; i++) {
    int has_null = 0; uint64_t h = 0;
    int sel = selected ? selected[i] != 0 : 1;
    if (sel) h = orc_hash_row(n_keys, probe_types, probe_cols, probe_key_idx, i, &has_null); /* HashChunkSelected */
    int64_t n_matched = 0;
    if (sel && !has_null) {
      /* GetMatchedRows (hash_table.go:110-134): candidates by hash in insertion order, verified by EqualChunkRow */
      int64_t cnt = orc_rowmap_get(m, h, pairs, pairs_cap);
      if (cnt > pairs_cap) { pairs_cap = cnt * 2; pairs = (uint32_t *)realloc(pairs, 8 * (size_t)pairs_cap); cnt = orc_rowmap_get(m, h, pairs, pairs_cap); }
      for (int64_t c = 0; c < cnt; c++) {
        int64_t brow = ((int64_t)pairs[2 * c] << 32) | pairs[2 * c + 1];
        if (!orc_equal_row(n_keys, build_types, build_cols, build_key_idx, brow, probe_types, probe_cols, probe_key_idx, i)) continue;
        /* tryToMatchInners: makeJoinRowToChunk per inner, then baseJoiner.filter over the joined rows when there are
         * OtherConditions (joiner.go:225-248,288-311,351-378,155-167); `matched` = some joined row survived */
        if (n_conds && !conds_true(n_conds, conds, outer_is_right, n_build_cols, build_types, build_cols, brow, n_probe_cols, probe_types, probe_cols, i)) continue;
        append_row(obs, build_base, n_build_cols, build_cols, brow);
        append_row(obs, probe_base, n_probe_cols, probe_cols, i);
        n_matched++;
      }
    }
    if (n_matched == 0 && is_outer) {                           /* onMissMatch joiner.go:274-277,337-340; inner: :405 */
      for (int c = 0; c < n_build_cols; c++) {                  /* outer ++ defaultInner */
        if (default_nn && default_nn[c] && elem_of_type(build_types[c]) == 8) ob_push(&obs[build_base + c], default_bits[c], 1);
        else ob_push_cell(&obs[build_base + c], &build_cols[c], -1);
      }
      append_row(obs, probe_base, n_probe_cols, probe_cols, i);
    }
  }
  free(pairs);
  orc_rowmap_free(m);
  *n_out = ncols ? obs[0].n : 0;
  for (int c = 0; c < ncols; c++) ob_finish(&obs[c], &out_cols[c]);
  free(obs);
  return ORC_OK;
}

/* ------------------------------------------------------------------ hash aggregation */
enum { AGG_COUNT = 0, AGG_SUM = 1, AGG_AVG = 2, AGG_MAX = 3, AGG_MIN = 4, AGG_FIRSTROW = 5 };

/* one PartialResult (aggfuncs/ sources partialResult4*): a tagged union of the states */
typedef struct {
  int64_t i;      /* count (COUNT, AVG) */
  int64_t si;     /* int sum / int value */
  double sf;      /* float sum / float value */
  uint8_t is_null;   /* SUM/MAX/MIN: no value yet (func_sum.go:40-44) */
  uint8_t got_first; /* FIRSTROW (func_first_row.go:22-28) */
} agg_state;

static void state_alloc(int func, agg_state *s) { /* AllocPartialResult */
  memset(s, 0, sizeof(*s));
  if (func == AGG_SUM || func == AGG_MAX || func == AGG_MIN) s->is_null = 1;
}

/* types.AddInt64 (types/overflow.go:33-40) */
static int add_int64(int64_t a, int64_t b, int64_t *r) {
  if ((a > 0 && b > 0 && INT64_MAX - a < b) || (a < 0 && b < 0 && INT64_MIN - a > b)) return ORC_ERR_OVERFLOW_BIGINT;
  *r = a + b; return ORC_OK;
}

/* Byte strings inside the oracle's aggregation: every distinct cell is interned once (deep copy, like stringutil.Copy in
 * func_max_min.go:352 / func_first_row.go:216) and states / group keys hold the intern id.  Interning is by byte equality. */
typedef struct { uint8_t **str; int64_t *len; int64_t n, cap; int64_t *slots; int64_t n_slots; } str_pool;
static str_pool g_pool;
static void pool_reset(void) {
  for (int64_t i = 0; i < g_pool.n; i++) free(g_pool.str[i]);
  free(g_pool.str); free(g_pool.len); free(g_pool.slots); memset(&g_pool, 0, sizeof(g_pool));
}
static uint64_t pool_hash(const uint8_t *b, int64_t n) { uint64_t h = 14695981039346656037ULL; for (int64_t i = 0; i < n; i++) h = (h ^ b[i]) * 1099511628211ULL; return h; }
static int64_t pool_intern(const uint8_t *b, int64_t n) {
  str_pool *m = &g_pool;
  if ((m->n + 1) * 2 > m->n_slots) {
    m->n_slots = m->n_slots ? m->n_slots * 2 : 1024;
    m->slots = (int64_t *)realloc(m->slots, 8 * (size_t)m->n_slots);
    for (int64_t i = 0; i < m->n_slots; i++) m->slots[i] = -1;
    for (int64_t g = 0; g < m->n; g++) { int64_t s = (int64_t)(pool_hash(m->str[g], m->len[g]) & (uint64_t)(m->n_slots - 1)); while (m->slots[s] >= 0) s = (s + 1) & (m->n_slots - 1); m->slots[s] = g; }
  }
  int64_t s = (int64_t)(pool_hash(b, n) & (uint64_t)(m->n_slots - 1));
  while (m->slots[s] >= 0) { int64_t g = m->slots[s]; if (m->len[g] == n && (n == 0 || !memcmp(m->str[g], b, (size_t)n))) return g; s = (s + 1) & (m->n_slots - 1); }
  if (m->n == m->cap) { m->cap = m->cap ? m->cap * 2 : 1024; m->str = (uint8_t **)realloc(m->str, sizeof(uint8_t *) * (size_t)m->cap); m->len = (int64_t *)realloc(m->len, 8 * (size_t)m->cap); }
  m->str[m->n] = (uint8_t *)malloc((size_t)(n ? n : 1)); if (n) memcpy(m->str[m->n], b, (size_t)n); m->len[m->n] = n;
  m->slots[s] = m->n;
  return m->n++;
}
static int compare_string(const uint8_t *x, int64_t lx, const uint8_t *y, int64_t ly);
/* the value of cell `row` as the 8-byte word the states work on: FLOAT -> float64(f) bits (Column.VecEvalReal widens,
 * expression/column.go:95-110), var-len -> intern id, everything else the raw slot */
static uint64_t cell_word(int type, const orc_column *c, int64_t row) {
  if (type == ORC_TYPE_FLOAT32) { float f; memcpy(&f, c->data + 4 * row, 4); double d = (double)f; uint64_t w; memcpy(&w, &d, 8); return w; }
  if (type == ORC_TYPE_BYTES) return (uint64_t)pool_intern(c->data + c->offsets[row], c->offsets[row + 1] - c->offsets[row]);
  return col_u64(c, row);
}

/* UpdatePartialResult for one input row */
static int state_update(int func, int type, const orc_column *arg, int64_t row, agg_state *s) {
  int isnull = arg ? col_is_null(arg, row) : 0;    /* arg == NULL: constant 1 (COUNT(*) == count(1), parser.y:3258-3262) */
  orc_column wcol; uint64_t wv;
  if (arg && (type == ORC_TYPE_FLOAT32 || type == ORC_TYPE_BYTES)) {
    /* FLOAT arguments are evaluated as float64 (EvalReal), strings by value: re-express the cell as one 8-byte word */
    wv = isnull ? 0 : cell_word(type, arg, row);
    wcol.length = 1; wcol.null_bitmap = NULL; wcol.offsets = NULL; wcol.data = (uint8_t *)&wv;
    uint8_t nb = (uint8_t)(isnull ? 0 : 1); wcol.null_bitmap = &nb;
    if (type == ORC_TYPE_FLOAT32) return state_update(func, ORC_TYPE_FLOAT64, &wcol, 0, s);
    if (func == AGG_COUNT) { if (!isnull) s->i++; return ORC_OK; }                   /* countOriginal4String func_count.go */
    if (func == AGG_FIRSTROW) { if (s->got_first) return ORC_OK; s->got_first = 1; s->is_null = (uint8_t)isnull; s->si = (int64_t)wv; return ORC_OK; }  /* func_first_row.go:206-220 */
    if (func == AGG_MAX || func == AGG_MIN) {                                         /* maxMin4String func_max_min.go:337-361 */
      if (isnull) return ORC_OK;
      if (s->is_null) { s->si = (int64_t)wv; s->is_null = 0; return ORC_OK; }
      int cmp = compare_string(g_pool.str[wv], g_pool.len[wv], g_pool.str[s->si], g_pool.len[s->si]);
      if ((func == AGG_MAX && cmp == 1) || (func == AGG_MIN && cmp == -1)) s->si = (int64_t)wv;
      return ORC_OK;
    }
    return ORC_ERR_UNSUPPORTED;                                                       /* SUM / AVG over strings arrive behind a cast */
  }
  switch (func) {
    case AGG_COUNT: if (!isnull) s->i++; return ORC_OK;                    /* func_count.go:33-49 */
    case AGG_SUM:
      if (isnull) return ORC_OK;
      if (type == ORC_TYPE_FLOAT64) {                                      /* func_sum.go:62-82 */
        double v = arg ? col_f64(arg, row) : 1.0;
        if (s->is_null) { s->sf = v; s->is_null = 0; } else s->sf += v;
      } else {                                                              /* func_sum.go:115-140 */
        int64_t v = arg ? col_i64(arg, row) : 1;
        if (s->is_null) { s->si = v; s->is_null = 0; return ORC_OK; }
        return add_int64(s->si, v, &s->si);
      }
      return ORC_OK;
    case AGG_AVG:
      if (isnull) return ORC_OK;
      if (type == ORC_TYPE_FLOAT64) { s->sf += arg ? col_f64(arg, row) : 1.0; s->i++; return ORC_OK; } /* func_avg.go:172-190 */
      { int rc = add_int64(s->si, arg ? col_i64(arg, row) : 1, &s->si); if (rc) return rc; s->i++; return ORC_OK; } /* :63-83 */
    case AGG_MAX: case AGG_MIN: {
      if (isnull) return ORC_OK;
      int is_max = (func == AGG_MAX);
      if (type == ORC_TYPE_FLOAT64) {                                      /* func_max_min.go:275-295 */
        double v = col_f64(arg, row);
        if (s->is_null) { s->sf = v; s->is_null = 0; }
        else if ((is_max && v > s->sf) || (!is_max && v < s->sf)) s->sf = v;
      } else if (type == ORC_TYPE_UINT64) {                                /* :146-167 */
        uint64_t v = col_u64(arg, row), cur = (uint64_t)s->si;
        if (s->is_null) { s->si = (int64_t)v; s->is_null = 0; }
        else if ((is_max && v > cur) || (!is_max && v < cur)) s->si = (int64_t)v;
      } else {                                                              /* :83-103 */
        int64_t v = col_i64(arg, row);
        if (s->is_null) { s->si = v; s->is_null = 0; }
        else if ((is_max && v > s->si) || (!is_max && v < s->si)) s->si = v;
      }
      return ORC_OK;
    }
    case AGG_FIRSTROW:                                                      /* func_first_row.go:67-81 */
      if (s->got_first) return ORC_OK;
      s->got_first = 1; s->is_null = (uint8_t)isnull;
      if (arg) { s->si = col_i64(arg, row); memcpy(&s->sf, &s->si, 8); } else { s->si = 1; }
      return ORC_OK;
  }
  return ORC_ERR_INVALID;
}

/* MergePartialResult(src, dst) */
static int state_merge(int func, int type, const agg_state *src, agg_state *dst) {
  if (type == ORC_TYPE_FLOAT32) type = ORC_TYPE_FLOAT64;   /* states of FLOAT arguments hold float64(f) */
  switch (func) {
    case AGG_COUNT: dst->i += src->i; return ORC_OK;                       /* func_count.go:115-119 */
    case AGG_SUM:
      if (src->is_null) return ORC_OK;
      if (type == ORC_TYPE_FLOAT64) { dst->sf += src->sf; dst->is_null = 0; return ORC_OK; } /* func_sum.go:84-92 */
      { int rc = add_int64(src->si, dst->si, &dst->si); if (rc) return rc; dst->is_null = 0; return ORC_OK; } /* :142-154 */
    case AGG_AVG:
      if (src->i == 0) return ORC_OK;                                       /* func_avg.go:120-131, 230-238 */
      if (type == ORC_TYPE_FLOAT64) { dst->sf += src->sf; dst->i += src->i; return ORC_OK; }
      { int rc = add_int64(src->si, dst->si, &dst->si); if (rc) return rc; dst->i += src->i; return ORC_OK; }
    case AGG_MAX: case AGG_MIN: {
      if (src->is_null) return ORC_OK;                                      /* func_max_min.go:105-118 */
      if (dst->is_null) { *dst = *src; return ORC_OK; }
      int is_max = (func == AGG_MAX);
      if (type == ORC_TYPE_BYTES) {                                         /* func_max_min.go:363-376 */
        int cmp = compare_string(g_pool.str[src->si], g_pool.len[src->si], g_pool.str[dst->si], g_pool.len[dst->si]);
        if ((is_max && cmp == 1) || (!is_max && cmp == -1)) dst->si = src->si;
        return ORC_OK;
      }
      if (type == ORC_TYPE_FLOAT64) { if ((is_max && src->sf > dst->sf) || (!is_max && src->sf < dst->sf)) dst->sf = src->sf; }
      else if (type == ORC_TYPE_UINT64) { uint64_t a = (uint64_t)src->si, b = (uint64_t)dst->si; if ((is_max && a > b) || (!is_max && a < b)) dst->si = src->si; }
      else { if ((is_max && src->si > dst->si) || (!is_max && src->si < dst->si)) dst->si = src->si; }
      return ORC_OK;
    }
    case AGG_FIRSTROW: if (!dst->got_first) *dst = *src; return ORC_OK;     /* func_first_row.go:83-89 */
  }
  return ORC_ERR_INVALID;
}

/* AppendFinalResult2Chunk */
static void ob_push_str(outbuf *b, int64_t id) { /* AppendString / AppendNull (id < 0) of a var-len result column */
  orc_column c; int64_t off[2] = {0, 0}; uint8_t nb = 1;
  c.length = 1; c.null_bitmap = &nb; c.offsets = off; c.data = NULL;
  if (id >= 0) { off[1] = g_pool.len[id]; c.data = g_pool.str[id]; ob_push_cell(b, &c, 0); } else ob_push_cell(b, &c, -1);
}
static void state_final(int func, int type, const agg_state *s, outbuf *ob) {
  uint64_t bits;
  if (type == ORC_TYPE_BYTES && func != AGG_COUNT) {   /* maxMin4String / firstRow4String AppendFinalResult2Chunk */
    int isnull = (func == AGG_FIRSTROW) ? (s->is_null || !s->got_first) : s->is_null;
    ob_push_str(ob, isnull ? -1 : s->si);
    return;
  }
  if (type == ORC_TYPE_FLOAT32 && (func == AGG_MAX || func == AGG_MIN || func == AGG_FIRSTROW)) {
    /* maxMin4Float32 / firstRow4Float32 keep a float32 and AppendFloat32 it (func_max_min.go:214-271, func_first_row.go:101-146);
     * the state above holds float64(f), which narrows back exactly */
    int isnull = (func == AGG_FIRSTROW) ? (s->is_null || !s->got_first) : s->is_null;
    double d; if (func == AGG_FIRSTROW) memcpy(&d, &s->si, 8); else d = s->sf;
    float f = (float)d; uint32_t w; memcpy(&w, &f, 4);
    ob_push(ob, isnull ? 0 : w, !isnull);
    return;
  }
  if (type == ORC_TYPE_FLOAT32) type = ORC_TYPE_FLOAT64;
  switch (func) {
    case AGG_COUNT: ob_push(ob, (uint64_t)s->i, 1); return;                /* func_count.go:23-27 */
    case AGG_SUM: case AGG_MAX: case AGG_MIN:
      if (s->is_null) { ob_push(ob, 0, 0); return; }                        /* func_sum.go:53-60 */
      if (type == ORC_TYPE_FLOAT64) { memcpy(&bits, &s->sf, 8); ob_push(ob, bits, 1); } else ob_push(ob, (uint64_t)s->si, 1);
      return;
    case AGG_AVG:
      if (s->i == 0) { ob_push(ob, 0, 0); return; }                         /* func_avg.go:47-55,159-167 */
      if (type == ORC_TYPE_FLOAT64) { double r = s->sf / (double)s->i; memcpy(&bits, &r, 8); ob_push(ob, bits, 1); }
      else ob_push(ob, (uint64_t)(s->si / s->i), 1);                        /* Go truncating int division */
      return;
    case AGG_FIRSTROW:
      if (s->is_null || !s->got_first) { ob_push(ob, 0, 0); return; }       /* func_first_row.go:91-99 */
      ob_push(ob, (uint64_t)s->si, 1); return;
  }
}

/* Group key = HashGroupKey bytes (util/codec/codec.go:713-746).  The varint / cmp-float encodings
 * are injective on (is_null, 8 raw bytes), so the oracle keys on exactly that pair per GROUP BY item. */
typedef struct { uint64_t *keys; /* n_gb*2 words per group: isnull, bits */ agg_state *states; int64_t n, cap;
                 int64_t *slots; int64_t n_slots; int n_gb, n_funcs; } agg_map;

static void amap_init(agg_map *m, int n_gb, int n_funcs) {
  memset(m, 0, sizeof(*m)); m->n_gb = n_gb; m->n_funcs = n_funcs; m->n_slots = 1024;
  m->slots = (int64_t *)malloc(8 * (size_t)m->n_slots); for (int64_t i = 0; i < m->n_slots; i++) m->slots[i] = -1;
}
static uint64_t akey_hash(const uint64_t *k, int nw) { uint64_t h = 1469598103934665603ULL; for (int i = 0; i < nw; i++) { h ^= k[i]; h *= 0x100000001B3ULL; h ^= h >> 29; } return h; }
static int64_t amap_get(agg_map *m, const uint64_t *key, const int *funcs) { /* getPartialResult aggregate.go:396-410 */
  int nw = m->n_gb * 2;
  if ((m->n + 1) * 2 > m->n_slots) {
    m->n_slots *= 2; m->slots = (int64_t *)realloc(m->slots, 8 * (size_t)m->n_slots);
    for (int64_t i = 0; i < m->n_slots; i++) m->slots[i] = -1;
    for (int64_t g = 0; g < m->n; g++) { int64_t s = (int64_t)(akey_hash(m->keys + g * nw, nw) & (uint64_t)(m->n_slots - 1)); while (m->slots[s] >= 0) s = (s + 1) & (m->n_slots - 1); m->slots[s] = g; }
  }
  int64_t s = (int64_t)(akey_hash(key, nw) & (uint64_t)(m->n_slots - 1));
  while (m->slots[s] >= 0) { if (nw == 0 || !memcmp(m->keys + m->slots[s] * nw, key, 8 * (size_t)nw)) return m->slots[s]; s = (s + 1) & (m->n_slots - 1); }
  if (m->n == m->cap) { m->cap = m->cap ? m->cap * 2 : 1024; m->keys = (uint64_t *)realloc(m->keys, 8 * (size_t)(nw ? nw : 1) * (size_t)m->cap); m->states = (agg_state *)realloc(m->states, sizeof(agg_state) * (size_t)(m->n_funcs ? m->n_funcs : 1) * (size_t)m->cap); }
  if (nw) memcpy(m->keys + m->n * nw, key, 8 * (size_t)nw);
  for (int f = 0; f < m->n_funcs; f++) state_alloc(funcs[f], &m->states[m->n * m->n_funcs + f]);
  m->slots[s] = m->n;
  return m->n++;
}
static void amap_free(agg_map *m) { free(m->keys); free(m->states); free(m->slots); }

int orc_hash_agg(int n_input_cols, const int *types, const orc_column *cols, int64_t n_rows,
                 int n_group_by, const int *group_by_cols, int n_funcs, const orc_agg_func *funcs,
                 int n_partial_workers, orc_column *out_cols, int64_t *n_out) {
  if (n_partial_workers < 1) n_partial_workers = 1;
  for (int c = 0; c < n_input_cols; c++) if (types[c] < 1 || types[c] > 5) return ORC_ERR_UNSUPPORTED;
  for (int f = 0; f < n_funcs; f++)
    if (funcs[f].arg_col >= 0 && types[funcs[f].arg_col] == ORC_TYPE_BYTES && (funcs[f].func == AGG_SUM || funcs[f].func == AGG_AVG)) return ORC_ERR_UNSUPPORTED;
  pool_reset();
  int *fn = (int *)malloc(sizeof(int) * (size_t)(n_funcs ? n_funcs : 1));
  int *ft = (int *)malloc(sizeof(int) * (size_t)(n_funcs ? n_funcs : 1));
  for (int f = 0; f < n_funcs; f++) { fn[f] = funcs[f].func; ft[f] = funcs[f].arg_col >= 0 ? types[funcs[f].arg_col] : ORC_TYPE_INT64; }
  agg_map *partial = (agg_map *)malloc(sizeof(agg_map) * (size_t)n_partial_workers);
  for (int w = 0; w < n_partial_workers; w++) amap_init(&partial[w], n_group_by, n_funcs);
  uint64_t key[64];
  int rc = ORC_OK;
  /* fetchChildData deals chunks to partial workers (aggregate.go:487-522); updatePartialResult (:332-350) */
  for (int64_t i = 0; i < n_rows && rc == ORC_OK; i++) {
    int w = (int)((i / 1024) % n_partial_workers);
    for (int g = 0; g < n_group_by; g++) {
      const orc_column *c = &cols[group_by_cols[g]];
      int isnull = col_is_null(c, i);
      /* NilFlag: NULL is its own group; FLOAT items are evaluated as float64 (getGroupKey -> VecEvalReal), strings by their bytes */
      key[2 * g] = (uint64_t)isnull; key[2 * g + 1] = isnull ? 0 : cell_word(types[group_by_cols[g]], c, i);
    }
    int64_t gi = amap_get(&partial[w], key, fn);
    for (int f = 0; f < n_funcs && rc == ORC_OK; f++)
      rc = state_update(fn[f], ft[f], funcs[f].arg_col >= 0 ? &cols[funcs[f].arg_col] : NULL, i, &partial[w].states[gi * n_funcs + f]);
  }
  /* shuffleIntermData [stub :354] + consumeIntermData [stub :424]: every group reaches exactly one
   * final worker and is merged there with MergePartialResult; one final map is result-equivalent. */
  agg_map fin; amap_init(&fin, n_group_by, n_funcs);
  for (int w = 0; w < n_partial_workers && rc == ORC_OK; w++)
    for (int64_t g = 0; g < partial[w].n && rc == ORC_OK; g++) {
      int64_t gi = amap_get(&fin, partial[w].keys + g * n_group_by * 2, fn);
      for (int f = 0; f < n_funcs && rc == ORC_OK; f++)
        rc = state_merge(fn[f], ft[f], &partial[w].states[g * n_funcs + f], &fin.states[gi * n_funcs + f]);
    }
  outbuf *obs = (outbuf *)calloc((size_t)(n_funcs ? n_funcs : 1), sizeof(outbuf));
  for (int f = 0; f < n_funcs; f++) {
    int sel = (fn[f] == AGG_MAX || fn[f] == AGG_MIN || fn[f] == AGG_FIRSTROW);
    obs[f].elem = (sel && ft[f] == ORC_TYPE_BYTES) ? 0 : ((sel && ft[f] == ORC_TYPE_FLOAT32) ? 4 : 8);
  }
  if (rc == ORC_OK) {
    if (fin.n == 0 && n_group_by == 0) {
      /* empty input, no GROUP BY: defaultVal row (aggregate.go:572-574, builder.go:517-540):
       * COUNT -> 0, everything else NULL.  (all-FIRSTROW aggregates produce no row.) */
      int all_first = 1; for (int f = 0; f < n_funcs; f++) if (fn[f] != AGG_FIRSTROW) all_first = 0;
      if (!all_first) for (int f = 0; f < n_funcs; f++) { if (fn[f] == AGG_COUNT) ob_push(&obs[f], 0, 1); else if (obs[f].elem == 0) ob_push_str(&obs[f], -1); else ob_push(&obs[f], 0, 0); }
    } else {
      for (int64_t g = 0; g < fin.n; g++)              /* getFinalResult aggregate.go:429-457 */
        for (int f = 0; f < n_funcs; f++) state_final(fn[f], ft[f], &fin.states[g * n_funcs + f], &obs[f]);
    }
  }
  *n_out = n_funcs ? obs[0].n : 0;
  for (int f = 0; f < n_funcs; f++) ob_finish(&obs[f], &out_cols[f]);
  free(obs);
  for (int w = 0; w < n_partial_workers; w++) amap_free(&partial[w]);
  amap_free(&fin); free(partial); free(fn); free(ft);
  pool_reset();
  return rc;
}

/* ------------------------------------------------------------------ pushed-down partial aggregation + FinalMode HashAgg (SURVEY §8 f4)
 * orc_cop_partial_agg restates the coprocessor's hashAggExec (store/mockstore/mocktikv/aggregate.go:66-182): ONE map, groups
 * in first-seen order (:159-163), Update per row (:166-172), and per group one output row = the GetPartialResult datums of
 * every function (:98-107; expression/aggregation/{count,sum,avg,max_min,first_row}.go GetPartialResult — COUNT: count;
 * SUM: value or NULL; AVG: count, value; MAX / MIN / FIRSTROW: the datum in the argument's own type) followed by the GROUP BY
 * values of the group's first row (:108, :118-147).  calculateSum (aggregation/util.go:57-91) adds BIGINT arguments as int64
 * (ComputePlus: overflow error) and everything else as float64 — exactly what state_update's SUM / AVG cases do. */
static void state_partial_out(int func, int type, const agg_state *s, outbuf *obs, int *oc) {
  uint64_t bits;
  int ft = type == ORC_TYPE_FLOAT32 ? ORC_TYPE_FLOAT64 : type;
  switch (func) {
    case AGG_COUNT: ob_push(&obs[(*oc)++], (uint64_t)s->i, 1); return;
    case AGG_AVG:
      ob_push(&obs[(*oc)++], (uint64_t)s->i, 1);          /* types.NewIntDatum(evalCtx.Count), avg.go:79-81 */
      if (s->i == 0) { ob_push(&obs[(*oc)++], 0, 0); return; }   /* evalCtx.Value is still the NULL datum */
      if (ft == ORC_TYPE_FLOAT64) { memcpy(&bits, &s->sf, 8); ob_push(&obs[(*oc)++], bits, 1); } else ob_push(&obs[(*oc)++], (uint64_t)s->si, 1);
      return;
    default:
      state_final(func, type, s, &obs[(*oc)++]);           /* SUM / MAX / MIN / FIRSTROW: GetResult == the final value */
      return;
  }
}
static int partial_out_type(int func, int type) {   /* column type of a partial VALUE column */
  if (func == AGG_COUNT) return ORC_TYPE_INT64;
  if (func == AGG_SUM || func == AGG_AVG) return (type == ORC_TYPE_FLOAT64 || type == ORC_TYPE_FLOAT32) ? ORC_TYPE_FLOAT64 : ORC_TYPE_INT64;
  return type;
}
int orc_cop_partial_agg(int n_input_cols, const int *types, const orc_column *cols, int64_t n_rows,
                        int n_group_by, const int *group_by_cols, int n_funcs, const orc_agg_func *funcs,
                        orc_column *out_cols, int *out_types, int64_t *n_out) {
  for (int c = 0; c < n_input_cols; c++) if (types[c] < 1 || types[c] > 5) return ORC_ERR_UNSUPPORTED;
  for (int f = 0; f < n_funcs; f++)
    if (funcs[f].arg_col >= 0 && types[funcs[f].arg_col] == ORC_TYPE_BYTES && (funcs[f].func == AGG_SUM || funcs[f].func == AGG_AVG)) return ORC_ERR_UNSUPPORTED;
  pool_reset();
  int *fn = (int *)malloc(sizeof(int) * (size_t)(n_funcs ? n_funcs : 1));
  int *ft = (int *)malloc(sizeof(int) * (size_t)(n_funcs ? n_funcs : 1));
  int n_outc = n_group_by;
  for (int f = 0; f < n_funcs; f++) { fn[f] = funcs[f].func; ft[f] = funcs[f].arg_col >= 0 ? types[funcs[f].arg_col] : ORC_TYPE_INT64; n_outc += fn[f] == AGG_AVG ? 2 : 1; }
  agg_map m; amap_init(&m, n_group_by, n_funcs);
  int64_t *first_row = NULL; int64_t fr_cap = 0;
  uint64_t key[64];
  int rc = ORC_OK;
  for (int64_t i = 0; i < n_rows && rc == ORC_OK; i++) {
    for (int g = 0; g < n_group_by; g++) {
      const orc_column *c = &cols[group_by_cols[g]];
      int isnull = col_is_null(c, i);
      key[2 * g] = (uint64_t)isnull; key[2 * g + 1] = isnull ? 0 : cell_word(types[group_by_cols[g]], c, i);
    }
    int64_t before = m.n;
    int64_t gi = amap_get(&m, key, fn);
    if (m.n != before) {   /* a new group: remember the row its GROUP BY values are taken from (groupKeyRows, :159-163) */
      if (m.n > fr_cap) { fr_cap = fr_cap ? fr_cap * 2 : 1024; while (fr_cap < m.n) fr_cap *= 2; first_row = (int64_t *)realloc(first_row, 8 * (size_t)fr_cap); }
      first_row[gi] = i;
    }
    for (int f = 0; f < n_funcs && rc == ORC_OK; f++)
      rc = state_update(fn[f], ft[f], funcs[f].arg_col >= 0 ? &cols[funcs[f].arg_col] : NULL, i, &m.states[gi * n_funcs + f]);
  }
  outbuf *obs = (outbuf *)calloc((size_t)(n_outc ? n_outc : 1), sizeof(outbuf));
  int oc = 0;
  for (int f = 0; f < n_funcs; f++) {
    if (fn[f] == AGG_AVG) { out_types[oc] = ORC_TYPE_INT64; obs[oc++].elem = 8; }
    out_types[oc] = partial_out_type(fn[f], ft[f]); obs[oc].elem = elem_of_type(out_types[oc]); oc++;
  }
  for (int g = 0; g < n_group_by; g++) { out_types[oc] = types[group_by_cols[g]]; obs[oc].elem = elem_of_type(out_types[oc]); oc++; }
  if (rc == ORC_OK)
    for (int64_t g = 0; g < m.n; g++) {
      oc = 0;
      for (int f = 0; f < n_funcs; f++) state_partial_out(fn[f], ft[f], &m.states[g * n_funcs + f], obs, &oc);
      for (int k = 0; k < n_group_by; k++) ob_push_cell(&obs[oc++], &cols[group_by_cols[k]], first_row[g]);
    }
  *n_out = n_outc ? obs[0].n : 0;
  for (int c = 0; c < n_outc; c++) ob_finish(&obs[c], &out_cols[c]);
  free(obs); free(first_row); amap_free(&m); free(fn); free(ft);
  pool_reset();
  return rc;
}

/* HashAggExec in FinalMode over partial rows (executor/aggregate.go with AggFuncDesc.Mode == FinalMode; the functions
 * aggfuncs/builder.go builds for Partial2Mode / FinalMode):
 *   COUNT  -> countPartial.UpdatePartialResult   func_count.go:99-113   (adds the partial counts, NULL skipped)
 *   AVG    -> avgPartial4Int64 / avgPartial4Float64   func_avg.go:86-113, 200-227   (args[0] = count, args[1] = sum; a row whose
 *             sum or count is NULL is skipped)
 *   SUM / MAX / MIN / FIRSTROW -> the ordinary functions over the partial value column (builder.go:66-80,112-175)
 * One partial worker / one final worker is result-equivalent (see orc_hash_agg). */
int orc_hash_agg_final(int n_input_cols, const int *types, const orc_column *cols, int64_t n_rows,
                       int n_group_by, const int *group_by_cols, int n_funcs, const orc_agg_final_func *funcs,
                       orc_column *out_cols, int64_t *n_out) {
  for (int c = 0; c < n_input_cols; c++) if (types[c] < 1 || types[c] > 5) return ORC_ERR_UNSUPPORTED;
  pool_reset();
  int *fn = (int *)malloc(sizeof(int) * (size_t)(n_funcs ? n_funcs : 1));
  int *ft = (int *)malloc(sizeof(int) * (size_t)(n_funcs ? n_funcs : 1));
  for (int f = 0; f < n_funcs; f++) {
    fn[f] = funcs[f].func;
    ft[f] = fn[f] == AGG_AVG ? types[funcs[f].arg_col2] : (fn[f] == AGG_COUNT ? ORC_TYPE_INT64 : types[funcs[f].arg_col]);
  }
  agg_map m; amap_init(&m, n_group_by, n_funcs);
  uint64_t key[64];
  int rc = ORC_OK;
  for (int64_t i = 0; i < n_rows && rc == ORC_OK; i++) {
    for (int g = 0; g < n_group_by; g++) {
      const orc_column *c = &cols[group_by_cols[g]];
      int isnull = col_is_null(c, i);
      key[2 * g] = (uint64_t)isnull; key[2 * g + 1] = isnull ? 0 : cell_word(types[group_by_cols[g]], c, i);
    }
    int64_t gi = amap_get(&m, key, fn);
    for (int f = 0; f < n_funcs && rc == ORC_OK; f++) {
      agg_state *st = &m.states[gi * n_funcs + f];
      const orc_column *a = &cols[funcs[f].arg_col];
      if (fn[f] == AGG_COUNT) { if (!col_is_null(a, i)) st->i += col_i64(a, i); }
      else if (fn[f] == AGG_AVG) {
        const orc_column *sc = &cols[funcs[f].arg_col2];
        if (col_is_null(sc, i) || col_is_null(a, i)) continue;
        if (ft[f] == ORC_TYPE_FLOAT64) { st->sf += col_f64(sc, i); st->i += col_i64(a, i); }
        else { rc = add_int64(st->si, col_i64(sc, i), &st->si); if (rc == ORC_OK) st->i += col_i64(a, i); }
      } else rc = state_update(fn[f], ft[f], a, i, st);
    }
  }
  outbuf *obs = (outbuf *)calloc((size_t)(n_funcs ? n_funcs : 1), sizeof(outbuf));
  for (int f = 0; f < n_funcs; f++) {
    int sel = (fn[f] == AGG_MAX || fn[f] == AGG_MIN || fn[f] == AGG_FIRSTROW);
    obs[f].elem = (sel && ft[f] == ORC_TYPE_BYTES) ? 0 : ((sel && ft[f] == ORC_TYPE_FLOAT32) ? 4 : 8);
  }
  if (rc == ORC_OK) {
    if (m.n == 0 && n_group_by == 0) {   /* the default row of a scalar aggregate over empty input, as in orc_hash_agg */
      int all_first = 1; for (int f = 0; f < n_funcs; f++) if (fn[f] != AGG_FIRSTROW) all_first = 0;
      if (!all_first) for (int f = 0; f < n_funcs; f++) { if (fn[f] == AGG_COUNT) ob_push(&obs[f], 0, 1); else if (obs[f].elem == 0) ob_push_str(&obs[f], -1); else ob_push(&obs[f], 0, 0); }
    } else {
      for (int64_t g = 0; g < m.n; g++)
        for (int f = 0; f < n_funcs; f++) state_final(fn[f], ft[f], &m.states[g * n_funcs + f], &obs[f]);
    }
  }
  *n_out = n_funcs ? obs[0].n : 0;
  for (int f = 0; f < n_funcs; f++) ob_finish(&obs[f], &out_cols[f]);
  free(obs); amap_free(&m); free(fn); free(ft);
  pool_reset();
  return rc;
}

/* ------------------------------------------------------------------ vectorized builtins */
/* types/compare.go:44-100 VecCompare{UU,II,UI,IU} -> -1/0/1 */
static int cmp_int(int ua, int ub, int64_t x, int64_t y) {
  if (ua && ub) { uint64_t a = (uint64_t)x, b = (uint64_t)y; return a < b ? -1 : (a == b ? 0 : 1); }
  if (!ua && !ub) return x < y ? -1 : (x == y ? 0 : 1);
  if (ua && !ub) { /* VecCompareUI :72-85 */
    if (y < 0 || (uint64_t)x > (uint64_t)INT64_MAX) return 1;
    return x < y ? -1 : (x == y ? 0 : 1);
  }
  /* VecCompareIU :88-100 */
  if (x < 0 || (uint64_t)y > (uint64_t)INT64_MAX) return -1;
  return x < y ? -1 : (x == y ? 0 : 1);
}
static int64_t cmp_result(int op, int c) { /* vecResOf{LT,LE,GT,GE,EQ,NE} builtin_compare_vec.go:214-279 */
  switch (op) { case 0: return c < 0; case 1: return c <= 0; case 2: return c > 0; case 3: return c >= 0; case 4: return c == 0; default: return c != 0; }
}

int orc_vec_compare_int(int op, int64_t n, const orc_column *a, int ua, const orc_column *b, int ub, orc_column *out) {
  if (op < 0 || op > 5) return ORC_ERR_INVALID;
  out_init(out, n);                                   /* result.ResizeInt64(n, false)  builtin_compare_vec.go:207 */
  int64_t *r = (int64_t *)out->data;
  for (int64_t i = 0; i < n; i++) r[i] = cmp_result(op, cmp_int(ua, ub, col_i64(a, i), col_i64(b, i))); /* all rows, NULL or not */
  merge_nulls(out, a, n); merge_nulls(out, b, n);     /* result.MergeNulls(buf0, buf1) :209 */
  return ORC_OK;
}

/* types.CompareFloat64 (types/compare.go): x<y -> -1; x==y -> 0; else 1 (NaN compares as 1) */
static int cmp_f64(double x, double y) { return x < y ? -1 : (x == y ? 0 : 1); }
int orc_vec_compare_real(int op, int64_t n, const orc_column *a, const orc_column *b, orc_column *out) {
  if (op < 0 || op > 5) return ORC_ERR_INVALID;
  out_init(out, n); merge_nulls(out, a, n); merge_nulls(out, b, n);   /* builtin_compare_vec_generated.go:44-45 */
  int64_t *r = (int64_t *)out->data;
  for (int64_t i = 0; i < n; i++) {
    if (col_is_null(out, i)) { r[i] = 0; continue; }               /* `continue`: slot is don't-care; we pin it to 0 */
    r[i] = cmp_result(op, cmp_f64(col_f64(a, i), col_f64(b, i)));
  }
  return ORC_OK;
}

int orc_vec_arith_int(int op, int64_t n, const orc_column *a, int ua, const orc_column *b, int ub, orc_column *out) {
  if (op < 0 || op > 2) return ORC_ERR_INVALID;
  out_init(out, n); merge_nulls(out, a, n); merge_nulls(out, b, n);
  int64_t *r = (int64_t *)out->data;
  for (int64_t i = 0; i < n; i++) {
    if (col_is_null(out, i)) { r[i] = 0; continue; }                /* `if result.IsNull(i) continue` — slot don't-care, pinned 0 */
    int64_t lh = col_i64(a, i), rh = col_i64(b, i);
    if (op == 0) {                                                   /* builtin_arithmetic_vec.go:431-495 */
      if (ua && ub) { if ((uint64_t)lh > UINT64_MAX - (uint64_t)rh) return ORC_ERR_OVERFLOW_BIGINT_UNSIGNED; }        /* plusUU :437 */
      else if (ua && !ub) {                                          /* plusUS :448-459 (second test restated verbatim: lh twice) */
        if (rh < 0 && (uint64_t)(-rh) > (uint64_t)lh) return ORC_ERR_OVERFLOW_BIGINT_UNSIGNED;
        if (rh > 0 && (uint64_t)lh > UINT64_MAX - (uint64_t)lh) return ORC_ERR_OVERFLOW_BIGINT_UNSIGNED;
      } else if (!ua && ub) {                                        /* plusSU :464-476 */
        if (lh < 0 && (uint64_t)(-lh) > (uint64_t)rh) return ORC_ERR_OVERFLOW_BIGINT_UNSIGNED;
        if (lh > 0 && (uint64_t)rh > UINT64_MAX - (uint64_t)lh) return ORC_ERR_OVERFLOW_BIGINT_UNSIGNED;
      } else {                                                       /* plusSS :481-495 */
        if ((lh > 0 && rh > INT64_MAX - lh) || (lh < 0 && rh < INT64_MIN - lh)) return ORC_ERR_OVERFLOW_BIGINT;
      }
      r[i] = lh + rh;
    } else if (op == 1) {                                            /* Minus, forceToSigned == false (default SQL mode) :130-139 */
      if (ua && ub) { if ((uint64_t)lh < (uint64_t)rh) return ORC_ERR_OVERFLOW_BIGINT_UNSIGNED; }                      /* minusUU :208 */
      else if (ua && !ub) {                                          /* minusUS :224-229 */
        if (rh >= 0 && (uint64_t)lh < (uint64_t)rh) return ORC_ERR_OVERFLOW_BIGINT_UNSIGNED;
        if (rh < 0 && (uint64_t)lh > UINT64_MAX - (uint64_t)(-rh)) return ORC_ERR_OVERFLOW_BIGINT_UNSIGNED;
      } else if (!ua && ub) {                                        /* minusSU :245 */
        if ((uint64_t)(lh - INT64_MIN) < (uint64_t)rh) return ORC_ERR_OVERFLOW_BIGINT_UNSIGNED;
      } else {                                                       /* minusSS :260 */
        if ((lh > 0 && -rh > INT64_MAX - lh) || (lh < 0 && -rh < INT64_MIN - lh)) return ORC_ERR_OVERFLOW_BIGINT;
      }
      r[i] = lh - rh;
    } else {
      if (ua || ub) {                                                /* MultiplyIntUnsigned :521-529 — chosen when EITHER side is unsigned (builtin_arithmetic.go:344-348) */
        uint64_t x = (uint64_t)lh, y = (uint64_t)rh, res = x * y;
        if (x != 0 && res / x != y) return ORC_ERR_OVERFLOW_BIGINT_UNSIGNED;
        r[i] = (int64_t)res;
      } else {                                                       /* MultiplyInt :332-338 */
        int64_t tmp = lh * rh;
        /* Go's wrapping quotient: MinInt64 / -1 == MinInt64 (no trap) */
        int64_t q = (lh == -1 && tmp == INT64_MIN) ? INT64_MIN : (lh != 0 ? tmp / lh : 0);
        if (lh != 0 && q != rh) return ORC_ERR_OVERFLOW_BIGINT;
        r[i] = tmp;
      }
    }
  }
  return ORC_OK;
}

int orc_vec_arith_real(int op, int64_t n, const orc_column *a, const orc_column *b, orc_column *out, int64_t *div_by_zero) {
  if (op < 0 || op > 3) return ORC_ERR_INVALID;
  out_init(out, n); merge_nulls(out, a, n); merge_nulls(out, b, n);
  double *r = (double *)out->data;
  int64_t dz = 0;
  for (int64_t i = 0; i < n; i++) {
    if (col_is_null(out, i)) { r[i] = 0; continue; }
    double x = col_f64(a, i), y = col_f64(b, i);
    switch (op) {
      case 0: if ((x > 0 && y > DBL_MAX_ - x) || (x < 0 && y < -DBL_MAX_ - x)) return ORC_ERR_OVERFLOW_DOUBLE; r[i] = x + y; break;   /* :302-305 */
      case 1: if ((x > 0 && -y > DBL_MAX_ - x) || (x < 0 && -y < -DBL_MAX_ - x)) return ORC_ERR_OVERFLOW_DOUBLE; r[i] = x - y; break; /* :80-83 */
      case 2: r[i] = x * y; if (isinf(r[i])) return ORC_ERR_OVERFLOW_DOUBLE; break;                                                  /* :49-52 */
      case 3:                                                                                                                        /* :368-381 */
        if (y == 0) { dz++; col_set_null(out, i, 1); r[i] = 0; break; }
        r[i] = x / y; if (isinf(r[i])) return ORC_ERR_OVERFLOW_DOUBLE; break;
    }
  }
  if (div_by_zero) *div_by_zero = dz;
  return ORC_OK;
}

int orc_vec_logic(int op, int64_t n, const orc_column *a, const orc_column *b, orc_column *out) {
  out_init(out, n);
  int64_t *r = (int64_t *)out->data;
  for (int64_t i = 0; i < n; i++) {
    int n0 = col_is_null(a, i), n1 = col_is_null(b, i);
    int64_t v0 = col_i64(a, i), v1 = col_i64(b, i);
    if (op == 0) {                                                   /* LogicAnd builtin_op_vec.go:192-211 */
      if (!n0 && v0 == 0) { r[i] = 0; }
      else if (!n1 && v1 == 0) { r[i] = 0; }
      else if (n0 || n1) { r[i] = 0; col_set_null(out, i, 1); }
      else r[i] = 1;
    } else if (op == 1) {                                            /* LogicOr :46-66 */
      if ((!n0 && v0 != 0) || (!n1 && v1 != 0)) r[i] = 1;
      else if (n0 || n1) { r[i] = 0; col_set_null(out, i, 1); }
      else r[i] = 0;
    } else return ORC_ERR_INVALID;
  }
  return ORC_OK;
}

int orc_vec_unary(int op, int64_t n, const orc_column *a, int ua, orc_column *out) {
  out_init(out, n);
  int64_t *r = (int64_t *)out->data; double *rf = (double *)out->data;
  for (int64_t i = 0; i < n; i++) {
    int isn = col_is_null(a, i);
    switch (op) {
      case 0: if (isn) { col_set_null(out, i, 1); r[i] = 0; } else r[i] = (col_i64(a, i) == 0); break;        /* UnaryNotInt :255-265 */
      case 1: if (isn) { col_set_null(out, i, 1); r[i] = 0; } else r[i] = (col_f64(a, i) == 0); break;        /* UnaryNotReal :152-165 */
      case 2: {                                                                                              /* UnaryMinusInt :221-243 — no NULL test in the loops; NULL slots are don't-care in the column contract, so the oracle skips them */
        if (isn) { col_set_null(out, i, 1); r[i] = 0; break; }
        int64_t v = col_i64(a, i);
        if (ua) { if ((uint64_t)v > (uint64_t)INT64_MAX + 1ULL) return ORC_ERR_OVERFLOW_BIGINT; }
        else if (v == INT64_MIN) return ORC_ERR_OVERFLOW_BIGINT;
        r[i] = -v; break;
      }
      case 3: if (isn) { col_set_null(out, i, 1); rf[i] = 0; } else rf[i] = -col_f64(a, i); break;           /* UnaryMinusReal :74-86 */
      case 4: r[i] = isn ? 1 : 0; break;                                                                     /* IsNull :98-106: never NULL */
      default: return ORC_ERR_INVALID;
    }
  }
  return ORC_OK;
}

int orc_vec_if(int64_t n, const orc_column *c, const orc_column *a, const orc_column *b, orc_column *out) {
  out_init(out, n);
  uint64_t *r = (uint64_t *)out->data;
  for (int64_t i = 0; i < n; i++) {                    /* builtin_control_vec_generated.go:141-156 */
    const orc_column *src = (col_is_null(c, i) || col_i64(c, i) == 0) ? b : a;
    if (col_is_null(src, i)) { col_set_null(out, i, 1); r[i] = 0; } else r[i] = col_u64(src, i);
  }
  return ORC_OK;
}
int orc_vec_ifnull(int64_t n, const orc_column *a, const orc_column *b, orc_column *out) {
  out_init(out, n);
  uint64_t *r = (uint64_t *)out->data;
  for (int64_t i = 0; i < n; i++) {                    /* builtin_control_vec_generated.go:38-45 */
    const orc_column *src = col_is_null(a, i) ? b : a;
    if (col_is_null(src, i)) { col_set_null(out, i, 1); r[i] = 0; } else r[i] = col_u64(src, i);
  }
  return ORC_OK;
}
int orc_vec_in_int(int64_t n, const orc_column *a, int ua, int n_list, const orc_column *list, const int *lu, orc_column *out) {
  out_init(out, n);
  int64_t *r = (int64_t *)out->data;
  for (int64_t i = 0; i < n; i++) {                    /* builtin_other_vec_generated.go:42-94 */
    int has_null = 0, found = 0;
    for (int j = 0; j < n_list; j++) {
      if (col_is_null(&list[j], i) || col_is_null(a, i)) { has_null = 1; continue; }  /* buf1.MergeNulls(buf0) */
      int64_t x = col_i64(a, i), y = col_i64(&list[j], i);
      int eq;
      if ((ua && lu[j]) || (!ua && !lu[j])) eq = (x == y);
      else if (!ua && lu[j]) eq = (x >= 0 && y == x);
      else eq = (y >= 0 && y == x);
      if (eq) found = 1;
    }
    if (found) r[i] = 1; else { r[i] = 0; if (has_null) col_set_null(out, i, 1); }
  }
  return ORC_OK;
}
int orc_vec_filter_int(int64_t n, const orc_column *a, uint8_t *selected) {
  /* VectorizedFilter over one int column: VecEvalBool + toBool (expression/expression.go:205-326):
   * selected = !isNull && value != 0 */
  for (int64_t i = 0; i < n; i++) selected[i] = (uint8_t)(!col_is_null(a, i) && col_i64(a, i) != 0);
  return ORC_OK;
}

/* ------------------------------------------------------------------ string builtins */
/* types.CompareString (types/compare.go:115-123): Go string order = unsigned byte order, shorter first on a tie */
static int compare_string(const uint8_t *x, int64_t lx, const uint8_t *y, int64_t ly) {
  int64_t m = lx < ly ? lx : ly;
  int c = m ? memcmp(x, y, (size_t)m) : 0;
  if (c) return c < 0 ? -1 : 1;
  return lx < ly ? -1 : (lx > ly ? 1 : 0);
}
/* builtin{LT..NE}StringSig.vecEvalInt (builtin_compare_vec_generated.go:65-555): MergeNulls, then per non-NULL row
 * val = CompareString(a, b) mapped through the operator; op 6 = builtinStrcmpSig (builtin_string_vec.go:52-83). */
int orc_vec_compare_string(int op, int64_t n, const orc_column *a, const orc_column *b, orc_column *out) {
  if (op < 0 || op > 6) return ORC_ERR_INVALID;
  int64_t *o = (int64_t *)out->data;
  out->length = n;
  memset(out->null_bitmap, 0, (size_t)((n + 7) >> 3));
  for (int64_t i = 0; i < n; i++) {
    o[i] = 0;
    if (col_is_null(a, i) || col_is_null(b, i)) continue;
    out->null_bitmap[i >> 3] |= (uint8_t)(1u << (i & 7));
    int c = compare_string(a->data + a->offsets[i], a->offsets[i + 1] - a->offsets[i], b->data + b->offsets[i], b->offsets[i + 1] - b->offsets[i]);
    switch (op) {
      case 0: o[i] = c < 0; break;
      case 1: o[i] = c <= 0; break;
      case 2: o[i] = c > 0; break;
      case 3: o[i] = c >= 0; break;
      case 4: o[i] = c == 0; break;
      case 5: o[i] = c != 0; break;
      default: o[i] = c; break;
    }
  }
  return ORC_OK;
}
/* op 0: builtinLengthSig.evalInt per row — int64(len([]byte(val))), NULL in, NULL out (builtin_string.go:75-81);
 * op 1: builtinStringIsNullSig.vecEvalInt (builtin_string_vec.go:21-42) */
int orc_vec_string_unary(int op, int64_t n, const orc_column *a, orc_column *out) {
  if (op < 0 || op > 1) return ORC_ERR_INVALID;
  int64_t *o = (int64_t *)out->data;
  out->length = n;
  memset(out->null_bitmap, 0, (size_t)((n + 7) >> 3));
  for (int64_t i = 0; i < n; i++) {
    int isnull = col_is_null(a, i);
    if (op == 0) {
      o[i] = isnull ? 0 : a->offsets[i + 1] - a->offsets[i];
      if (!isnull) out->null_bitmap[i >> 3] |= (uint8_t)(1u << (i & 7));
    } else {
      o[i] = isnull ? 1 : 0;
      out->null_bitmap[i >> 3] |= (uint8_t)(1u << (i & 7));
    }
  }
  return ORC_OK;
}

/* builtinInRealSig.vecEvalInt (expression/builtin_other_vec_generated.go:151-204): like IN over ints with types.CompareFloat64 */
int orc_vec_in_real(int64_t n, const orc_column *a, int n_list, const orc_column *list, orc_column *out) {
  out_init(out, n);
  int64_t *r = (int64_t *)out->data;
  for (int64_t i = 0; i < n; i++) {
    int has_null = 0, found = 0;
    for (int j = 0; j < n_list; j++) {
      if (col_is_null(a, i) || col_is_null(&list[j], i)) { has_null = 1; continue; }   /* buf1.MergeNulls(buf0) :185 */
      double x = col_f64(a, i), y = col_f64(&list[j], i);
      if (cmp_f64(x, y) == 0) found = 1;                                             /* :193-197 */
    }
    r[i] = found;
    col_set_null(out, i, !found && has_null);                                        /* :199-203 */
  }
  return ORC_OK;
}

/* builtinInStringSig.vecEvalInt (builtin_other_vec_generated.go:97-149) */
int orc_vec_in_string(int64_t n, const orc_column *a, int n_list, const orc_column *list, orc_column *out) {
  out_init(out, n);
  int64_t *r = (int64_t *)out->data;
  for (int64_t i = 0; i < n; i++) {
    int has_null = 0, found = 0;
    for (int j = 0; j < n_list; j++) {
      if (col_is_null(a, i) || col_is_null(&list[j], i)) { has_null = 1; continue; }
      const orc_column *b = &list[j];
      if (compare_string(a->data + a->offsets[i], a->offsets[i + 1] - a->offsets[i], b->data + b->offsets[i], b->offsets[i + 1] - b->offsets[i]) == 0) found = 1;
    }
    r[i] = found;
    col_set_null(out, i, !found && has_null);
  }
  return ORC_OK;
}

/* builtinIfStringSig (builtin_control_vec_generated.go:209-262, mode 0) / builtinIfNullStringSig (:81-112, mode 1): the result
 * column is malloc'ed here (free with orc_free_columns) */
int orc_vec_pick_string(int mode, int64_t n, const orc_column *cond, const orc_column *a, const orc_column *b, orc_column *out) {
  outbuf ob; memset(&ob, 0, sizeof(ob)); ob.elem = 0;
  for (int64_t i = 0; i < n; i++) {
    const orc_column *src;
    if (mode == 0) src = (col_is_null(cond, i) || col_i64(cond, i) == 0) ? b : a;
    else src = !col_is_null(a, i) ? a : b;
    ob_push_cell(&ob, src, col_is_null(src, i) ? -1 : i);
  }
  ob_finish(&ob, out);
  return ORC_OK;
}

/* toBool for ETReal (expression/expression.go:296-307): zero iff types.RoundFloat(f) == 0 (types/helper.go:28-34) */
int orc_vec_filter_real(int64_t n, const orc_column *a, uint8_t *selected) {
  for (int64_t i = 0; i < n; i++) {
    double f = col_f64(a, i), rf;
    if (fabs(f) < 0.5) rf = 0; else rf = trunc(f + copysign(0.5, f));
    selected[i] = (uint8_t)(!col_is_null(a, i) && !(rf == 0));
  }
  return ORC_OK;
}

/* ------------------------------------------------------------------ SortExec / TopNExec / MergeJoinExec (SURVEY §8 f3)
 * chunk.GetCompareFunc (util/chunk/compare.go:27-110): cmpNull first, then the type's comparison.  kind: the column type. */
static int cmp_cell(int type, const orc_column *a, int64_t ra, const orc_column *b, int64_t rb) {
  int an = col_is_null(a, ra), bn = col_is_null(b, rb);
  if (an || bn) return (an && bn) ? 0 : (an ? -1 : 1);                       /* cmpNull :45-53 */
  switch (type) {
    case ORC_TYPE_INT64: { int64_t x = col_i64(a, ra), y = col_i64(b, rb); return x < y ? -1 : (x == y ? 0 : 1); }      /* cmpInt64 :55-61 */
    case ORC_TYPE_UINT64: { uint64_t x = col_u64(a, ra), y = col_u64(b, rb); return x < y ? -1 : (x == y ? 0 : 1); }    /* cmpUint64 :63-69 */
    case ORC_TYPE_FLOAT64: return cmp_f64(col_f64(a, ra), col_f64(b, rb));                                                /* cmpFloat64 :87-93 */
    case ORC_TYPE_FLOAT32: { float x, y; memcpy(&x, a->data + 4 * ra, 4); memcpy(&y, b->data + 4 * rb, 4); return cmp_f64((double)x, (double)y); } /* cmpFloat32 :79-85 */
    default: return compare_string(a->data + a->offsets[ra], a->offsets[ra + 1] - a->offsets[ra],
                                   b->data + b->offsets[rb], b->offsets[rb + 1] - b->offsets[rb]);                       /* cmpString :71-77 */
  }
}

/* SortExec.Next / keyColumnsLess / lessRow (executor/sort.go:58-129) and TopNExec (:159-318).  The reference sorts row
 * pointers with sort.Slice, which leaves rows that compare equal in an unspecified order; the oracle fixes ONE of the
 * allowed outcomes — ties stay in child order (a bottom-up merge sort) — and the tests state that contract.  TopNExec keeps
 * the totalLimit = Offset + Count smallest rows in a heap and emits them from Offset on (:210-214, :262-279): the rows
 * [Offset, Offset + Count) of the full order.  limit_count < 0: SortExec. */
typedef struct { int n_by; const int *by_cols, *by_desc, *types; const orc_column *cols; } sort_ctx;
static int sort_less_eq(const sort_ctx *c, int64_t i, int64_t j) {   /* !lessRow(j, i) */
  for (int k = 0; k < c->n_by; k++) {
    int col = c->by_cols[k];
    int cmp = cmp_cell(c->types[col], &c->cols[col], j, &c->cols[col], i);
    if (c->by_desc[k]) cmp = -cmp;                                            /* sort.go:120-122 */
    if (cmp < 0) return 0;                                                    /* row j sorts before row i */
    if (cmp > 0) return 1;
  }
  return 1;
}
int orc_sort(int n_cols, const int *types, const orc_column *cols, int64_t n_rows, int n_by, const int *by_cols, const int *by_desc,
             int64_t limit_offset, int64_t limit_count, orc_column *out_cols, int64_t *n_out) {
  for (int c = 0; c < n_cols; c++) if (types[c] < 1 || types[c] > 5) return ORC_ERR_UNSUPPORTED;
  for (int k = 0; k < n_by; k++) if (by_cols[k] < 0 || by_cols[k] >= n_cols) return ORC_ERR_INVALID;
  sort_ctx ctx = {n_by, by_cols, by_desc, types, cols};
  int64_t *ptr = (int64_t *)malloc(8 * (size_t)(n_rows ? n_rows : 1)), *tmp = (int64_t *)malloc(8 * (size_t)(n_rows ? n_rows : 1));
  for (int64_t i = 0; i < n_rows; i++) ptr[i] = i;                            /* initPointers :88-97 */
  for (int64_t w = 1; w < n_rows; w *= 2) {
    for (int64_t lo = 0; lo < n_rows; lo += 2 * w) {
      int64_t mid = lo + w < n_rows ? lo + w : n_rows, hi = lo + 2 * w < n_rows ? lo + 2 * w : n_rows;
      int64_t a = lo, b = mid, o = lo;
      while (a < mid && b < hi) tmp[o++] = sort_less_eq(&ctx, ptr[a], ptr[b]) ? ptr[a++] : ptr[b++];
      while (a < mid) tmp[o++] = ptr[a++];
      while (b < hi) tmp[o++] = ptr[b++];
    }
    int64_t *t = ptr; ptr = tmp; tmp = t;
  }
  int64_t lo = limit_offset < n_rows ? limit_offset : n_rows, hi = n_rows;
  if (limit_count >= 0) hi = (limit_count < n_rows - lo) ? lo + limit_count : n_rows;
  outbuf *obs = (outbuf *)calloc((size_t)(n_cols ? n_cols : 1), sizeof(outbuf));
  for (int c = 0; c < n_cols; c++) obs[c].elem = elem_of_type(types[c]);
  for (int64_t i = lo; i < hi; i++) append_row(obs, 0, n_cols, cols, ptr[i]);   /* req.AppendRow(e.rowChunks.GetRow(rowPtr)) :71-75 */
  *n_out = hi - lo;
  for (int c = 0; c < n_cols; c++) ob_finish(&obs[c], &out_cols[c]);
  free(obs); free(ptr); free(tmp);
  return ORC_OK;
}

/* MergeJoinExec (executor/merge_join.go).  Children sorted ascending by their keys.  compare() (:323-337) uses the
 * expression CompareFuncs: NULL outer key -> compareNull = -1 (a miss); integers by CompareInt incl. mixed unsigned flags
 * (builtin_compare.go:525-560), reals by CompareFloat64 (FLOAT columns evaluate as float64), strings by CompareString. */
static int mj_cmp_key(int to, const orc_column *o, int64_t ro, int ti, const orc_column *i, int64_t ri) {
  if (col_is_null(o, ro)) return -1;                                          /* the inner row never has a NULL key (:154-162) */
  if (to == ORC_TYPE_BYTES) return compare_string(o->data + o->offsets[ro], o->offsets[ro + 1] - o->offsets[ro], i->data + i->offsets[ri], i->offsets[ri + 1] - i->offsets[ri]);
  if (to == ORC_TYPE_FLOAT64 || to == ORC_TYPE_FLOAT32) {
    uint64_t a = cell_word(to, o, ro), b = cell_word(ti, i, ri); double x, y; memcpy(&x, &a, 8); memcpy(&y, &b, 8);
    return cmp_f64(x, y);
  }
  return cmp_int(to == ORC_TYPE_UINT64, ti == ORC_TYPE_UINT64, col_i64(o, ro), col_i64(i, ri));
}
/* mergeJoinInnerTable: nextRow (:127-152) skips rows with a NULL join key; rowsWithSameKey (:96-125) returns the next run of
 * rows whose keys compare equal to the run's first row */
typedef struct { int n_keys; const int *keys, *types; const orc_column *cols; int64_t n, ip; int64_t *grp; int64_t g_n; } mj_inner;
static int mj_inner_null_key(const mj_inner *t, int64_t r) {
  for (int k = 0; k < t->n_keys; k++) if (col_is_null(&t->cols[t->keys[k]], r)) return 1;
  return 0;
}
static void mj_fetch_group(mj_inner *t) {
  t->g_n = 0;
  while (t->ip < t->n && mj_inner_null_key(t, t->ip)) t->ip++;
  if (t->ip >= t->n) return;
  int64_t first = t->ip;
  t->grp[t->g_n++] = t->ip++;
  for (;;) {
    while (t->ip < t->n && mj_inner_null_key(t, t->ip)) t->ip++;
    if (t->ip >= t->n) return;
    for (int k = 0; k < t->n_keys; k++)
      if (cmp_cell(t->types[t->keys[k]], &t->cols[t->keys[k]], t->ip, &t->cols[t->keys[k]], first) != 0) return;   /* compareChunkRow != 0 */
    t->grp[t->g_n++] = t->ip++;
  }
}
int orc_merge_join(int join_type, int outer_is_right,
                   int n_inner_cols, const int *inner_types, const orc_column *inner_cols,
                   int n_outer_cols, const int *outer_types, const orc_column *outer_cols,
                   int n_keys, const int *inner_keys, const int *outer_keys, const uint8_t *selected,
                   int n_conds, const orc_join_cond *conds,
                   const uint64_t *default_bits, const uint8_t *default_nn, orc_column *out_cols, int64_t *n_out) {
  if (join_type < 0 || join_type > 2 || n_keys < 0 || n_conds < 0) return ORC_ERR_INVALID;
  for (int c = 0; c < n_inner_cols; c++) if (inner_types[c] < 1 || inner_types[c] > 5) return ORC_ERR_UNSUPPORTED;
  for (int c = 0; c < n_outer_cols; c++) if (outer_types[c] < 1 || outer_types[c] > 5) return ORC_ERR_UNSUPPORTED;
  int64_t ni = n_inner_cols ? inner_cols[0].length : 0, no = n_outer_cols ? outer_cols[0].length : 0;
  int ncols = n_inner_cols + n_outer_cols;
  outbuf *obs = (outbuf *)calloc((size_t)ncols, sizeof(outbuf));
  int inner_base = outer_is_right ? 0 : n_outer_cols, outer_base = outer_is_right ? n_inner_cols : 0;
  for (int c = 0; c < n_inner_cols; c++) obs[inner_base + c].elem = elem_of_type(inner_types[c]);
  for (int c = 0; c < n_outer_cols; c++) obs[outer_base + c].elem = elem_of_type(outer_types[c]);
  int is_outer = join_type != 0;
  mj_inner in = {n_keys, inner_keys, inner_types, inner_cols, ni, 0, (int64_t *)malloc(8 * (size_t)(ni ? ni : 1)), 0};
  mj_fetch_group(&in);                           /* prepare -> fetchNextInnerRows (:217-223) */
  int64_t o = 0;
  while (o < no) {                               /* joinToChunk (:246-321) */
    int cmp = -1;
    if ((selected ? selected[o] != 0 : 1) && in.g_n > 0) {
      cmp = 0;
      for (int k = 0; k < n_keys && cmp == 0; k++)
        cmp = mj_cmp_key(outer_types[outer_keys[k]], &outer_cols[outer_keys[k]], o, inner_types[inner_keys[k]], &inner_cols[inner_keys[k]], in.grp[0]);
    }
    if (cmp > 0) { mj_fetch_group(&in); continue; }    /* :267-272 */
    if (cmp < 0) {                               /* onMissMatch (:274-288) */
      if (is_outer) {
        for (int c = 0; c < n_inner_cols; c++) {
          if (default_nn && default_nn[c] && elem_of_type(inner_types[c]) == 8) ob_push(&obs[inner_base + c], default_bits[c], 1);
          else ob_push_cell(&obs[inner_base + c], &inner_cols[c], -1);
        }
        append_row(obs, outer_base, n_outer_cols, outer_cols, o);
      }
      o++;
      continue;
    }
    int has_match = 0;
    for (int64_t g = 0; g < in.g_n; g++) {      /* tryToMatchInners over the whole group (:290-305): makeJoinRowToChunk + baseJoiner.filter */
      if (n_conds && !conds_true(n_conds, conds, outer_is_right, n_inner_cols, inner_types, inner_cols, in.grp[g], n_outer_cols, outer_types, outer_cols, o)) continue;
      append_row(obs, inner_base, n_inner_cols, inner_cols, in.grp[g]);
      append_row(obs, outer_base, n_outer_cols, outer_cols, o);
      has_match = 1;
    }
    if (!has_match && is_outer) {                /* :300-304 every joined row was filtered: onMissMatch */
      for (int c = 0; c < n_inner_cols; c++) {
        if (default_nn && default_nn[c] && elem_of_type(inner_types[c]) == 8) ob_push(&obs[inner_base + c], default_bits[c], 1);
        else ob_push_cell(&obs[inner_base + c], &inner_cols[c], -1);
      }
      append_row(obs, outer_base, n_outer_cols, outer_cols, o);
    }
    o++;
  }
  free(in.grp);
  *n_out = ncols ? obs[0].n : 0;
  for (int c = 0; c < ncols; c++) ob_finish(&obs[c], &out_cols[c]);
  free(obs);
  return ORC_OK;
}

/* ------------------------------------------------------------------ toBool for ETString (expression/expression.go:308-322)
 * isZero = (types.StrToInt(sc, s) == 0), and the error VecEvalBool sees is the err of the LAST non-NULL row (`err = err1`
 * inside the loop).  StrToInt (types/convert.go:224-232) in a SELECT statement (InSelectStmt, truncation is a warning,
 * CastStrToIntStrict == false): TrimSpace -> getValidFloatPrefix (:430-475) -> floatStrToIntStr (:318-405) -> strconv.ParseInt;
 * a ParseInt failure (syntax or range) is reported as ErrOverflow("BIGINT").  Restated LITERALLY — the intermediate strings are
 * built exactly as the Go code builds them — so that it is independent of the streaming form the device kernel uses.
 * strings.TrimSpace: the ASCII white space characters (the Unicode ones, U+0085 / U+00A0 / U+2000..., are not trimmed here
 * or on the device: documented deviation). */
typedef struct { char *p; int64_t n; } gostr;
static gostr gs_make(const char *p, int64_t n) { gostr s; s.p = (char *)malloc((size_t)(n + 1)); if (n) memcpy(s.p, p, (size_t)n); s.p[n] = 0; s.n = n; return s; }
static int is_digit_b(char c) { return c >= '0' && c <= '9'; }
/* strconv.ParseInt(s, 10, 64): returns 0 ok, 1 syntax error (value 0), 2 range error (value = max / min) */
static int go_parse_int(const char *s, int64_t n, int64_t *out) {
  *out = 0;
  if (n == 0) return 1;
  int neg = 0; int64_t i = 0;
  if (s[0] == '+') i = 1; else if (s[0] == '-') { neg = 1; i = 1; }
  if (i == n) return 1;
  uint64_t un = 0; int range = 0;
  for (; i < n; i++) {
    if (!is_digit_b(s[i])) return 1;
    uint64_t d = (uint64_t)(s[i] - '0');
    if (un > (UINT64_MAX - d) / 10) { range = 1; un = UINT64_MAX; } else if (!range) un = un * 10 + d;
  }
  if (!neg && (range || un > (uint64_t)INT64_MAX)) { *out = INT64_MAX; return 2; }
  if (neg && (range || un > (uint64_t)INT64_MAX + 1)) { *out = INT64_MIN; return 2; }
  *out = neg ? (int64_t)(0 - un) : (int64_t)un;
  return 0;
}
/* strconv.Atoi for the exponent: 0 ok, 1 error */
static int go_atoi(const char *s, int64_t n, int64_t *out) { int rc = go_parse_int(s, n, out); return rc != 0; }
/* roundIntStr (types/convert.go:283-311) */
static gostr round_int_str(char next, gostr in) {
  if (next < '5') return in;
  gostr r = gs_make(in.p, in.n + 1); r.n = in.n;   /* room for one appended '0' */
  int64_t idx = in.n - 1;
  for (; idx >= 1; idx--) { if (r.p[idx] != '9') { r.p[idx]++; break; } r.p[idx] = '0'; }
  if (idx == 0) {
    if (in.p[0] == '9') { r.p[0] = '1'; r.p[r.n++] = '0'; }
    else if (is_digit_b(in.p[0])) r.p[0]++;
    else { r.p[1] = '1'; r.p[r.n++] = '0'; }
  }
  r.p[r.n] = 0;
  free(in.p);
  return r;
}
int orc_str_to_int(const uint8_t *bytes, int64_t len, int64_t *ival, int *overflow_err) {
  const char *s = (const char *)bytes;
  int64_t n = len;
  while (n > 0 && (s[0] == ' ' || (s[0] >= '\t' && s[0] <= '\r'))) { s++; n--; }            /* strings.TrimSpace */
  while (n > 0 && (s[n - 1] == ' ' || (s[n - 1] >= '\t' && s[n - 1] <= '\r'))) n--;
  /* getValidFloatPrefix */
  gostr valid;
  if (n == 0) valid = gs_make("0", 1);                                                        /* InSelectStmt && s == "" */
  else {
    int saw_dot = 0, saw_digit = 0; int64_t valid_len = 0, e_idx = 0;
    for (int64_t i = 0; i < n; i++) {
      char c = s[i];
      if (c == '+' || c == '-') { if (i != 0 && i != e_idx + 1) break; }
      else if (c == '.') { if (saw_dot || e_idx > 0) break; saw_dot = 1; if (saw_digit) valid_len = i + 1; }
      else if (c == 'e' || c == 'E') { if (!saw_digit) break; if (e_idx != 0) break; e_idx = i; }
      else if (c < '0' || c > '9') break;
      else { saw_digit = 1; valid_len = i + 1; }
    }
    valid = valid_len ? gs_make(s, valid_len) : gs_make("0", 1);
  }
  /* floatStrToIntStr(validFloat) */
  gostr vf = valid, int_str;
  int64_t dot = -1, eidx = -1;
  for (int64_t i = 0; i < vf.n; i++) { if (vf.p[i] == '.') dot = i; else if (vf.p[i] == 'e' || vf.p[i] == 'E') eidx = i; }
  if (eidx == -1) {
    if (dot == -1) int_str = gs_make(vf.p, vf.n);
    else {
      const char *digits = vf.p; int64_t dl = vf.n;
      if (vf.p[0] == '-' || vf.p[0] == '+') { dot--; digits = vf.p + 1; dl = vf.n - 1; }
      int_str = dot == 0 ? gs_make("0", 1) : gs_make(digits, dot);
      if (dl > dot + 1) int_str = round_int_str(digits[dot + 1], int_str);
      if ((int_str.n > 1 || int_str.p[0] != '0') && vf.p[0] == '-') {
        gostr t = gs_make("-", 1); t.p = (char *)realloc(t.p, (size_t)(int_str.n + 2)); memcpy(t.p + 1, int_str.p, (size_t)int_str.n + 1); t.n = int_str.n + 1;
        free(int_str.p); int_str = t;
      }
    }
  } else {
    gostr digits = gs_make("", 0); digits.p = (char *)realloc(digits.p, (size_t)(vf.n + 1));
    int64_t int_cnt;
    if (dot == -1) { memcpy(digits.p, vf.p, (size_t)eidx); digits.n = eidx; int_cnt = eidx; }
    else { memcpy(digits.p, vf.p, (size_t)dot); int_cnt = dot; memcpy(digits.p + dot, vf.p + dot + 1, (size_t)(eidx - dot - 1)); digits.n = dot + (eidx - dot - 1); }
    digits.p[digits.n] = 0;
    int64_t exp = 0;
    if (go_atoi(vf.p + eidx + 1, vf.n - eidx - 1, &exp)) int_str = gs_make(vf.p, vf.n);     /* return validFloat, err */
    else {
      int_cnt = (int64_t)((uint64_t)int_cnt + (uint64_t)exp);                                 /* Go int addition wraps */
      if (exp >= 0 && (int_cnt > 21 || int_cnt < 0)) int_str = gs_make(vf.p, eidx);            /* + an overflow WARNING */
      else if (int_cnt <= 0) {
        int_str = gs_make("0", 1);
        if (int_cnt == 0 && digits.n > 0 && is_digit_b(digits.p[0])) int_str = round_int_str(digits.p[0], int_str);
      } else if (int_cnt == 1 && (digits.p[0] == '-' || digits.p[0] == '+')) {
        int_str = gs_make("0", 1);
        if (digits.n > 1) int_str = round_int_str(digits.p[1], int_str);
        if (int_str.p[0] == '1') { gostr t = gs_make(digits.p, 1); t.p = (char *)realloc(t.p, (size_t)(int_str.n + 2)); memcpy(t.p + 1, int_str.p, (size_t)int_str.n + 1); t.n = int_str.n + 1; free(int_str.p); int_str = t; }
      } else if (int_cnt <= digits.n) {
        int_str = gs_make(digits.p, int_cnt);
        if (int_cnt < digits.n) int_str = round_int_str(digits.p[int_cnt], int_str);
      } else {
        int64_t extra = int_cnt - digits.n;
        int_str = gs_make(digits.p, digits.n); int_str.p = (char *)realloc(int_str.p, (size_t)(digits.n + extra + 1));
        memset(int_str.p + digits.n, '0', (size_t)extra); int_str.n = digits.n + extra; int_str.p[int_str.n] = 0;
      }
    }
    free(digits.p);
  }
  int rc = go_parse_int(int_str.p, int_str.n, ival);                                          /* StrToInt :227-231 */
  *overflow_err = rc != 0;
  free(int_str.p); free(vf.p);
  return ORC_OK;
}
/* the valid int string itself, for the reference's floatStrToIntStr / getValidIntPrefix vectors (tests only) */
int orc_vec_filter_string(int64_t n, const orc_column *a, uint8_t *selected, int *err_overflow) {
  *err_overflow = 0;
  for (int64_t i = 0; i < n; i++) {
    if (col_is_null(a, i)) { selected[i] = 0; continue; }                                     /* isZero = -1 */
    int64_t v; int e;
    orc_str_to_int(a->data + a->offsets[i], a->offsets[i + 1] - a->offsets[i], &v, &e);
    *err_overflow = e;                                                                         /* err = err1: the last row wins */
    selected[i] = (uint8_t)(v != 0);
  }
  return ORC_OK;
}
