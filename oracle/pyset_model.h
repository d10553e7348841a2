/*
 * pyset_model.h — ORACLE (test infrastructure, never shipped in the product path).
 *
 * A restatement of the two pieces of CPython the reference's hot path depends
 * on for its tie-breaks (SURVEY.md appendix B):
 *   - the tuple hash of CPython >= 3.8 (Objects/tupleobject.c, tuplehash), and
 *   - the open-addressing table of `set` (Objects/setobject.c: set_add_entry,
 *     set_insert_clean, set_table_resize, set_intersection, iteration order).
 * CPython is not part of the reference; the algorithm is the published one of
 * CPython 3.8 .. 3.12 and is pinned against the running interpreter (3.12.3) by
 * tests/test_pyset_model.py.
 *
 * The reference uses sets at nhd/Matcher.py:113,129,141 (GPU tuples),
 * :175,212,220 (CPU tuples), :349,365 (intersection) and
 * nhd/NHDScheduler.py:302 (claimed NIC indices).
 *
 * Keys are small tuples of small non-negative ints (or single ints); a key is
 * carried as an opaque 64-bit id plus its Python hash.
 */
#ifndef NHD_ORACLE_PYSET_MODEL_H
#define NHD_ORACLE_PYSET_MODEL_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PYSET_MINSIZE 8
#define PYSET_MAX_SLOTS 4096

typedef struct {
    uint64_t key;    /* opaque key id, valid iff live */
    uint64_t hash;   /* Py_hash_t reinterpreted as unsigned */
    int live;
} pyset_entry;

typedef struct {
    pyset_entry slots[PYSET_MAX_SLOTS];
    size_t mask;     /* table size - 1 */
    size_t fill;     /* live + dummy (no deletions here, so == used) */
    size_t used;
} pyset;

/* hash(int) for 0 <= v < 2^61-1 */
uint64_t py_hash_int(int64_t v);
/* hash(tuple of small non-negative ints) */
uint64_t py_hash_tuple(const int* items, int len);

void pyset_init(pyset* s);
/* s.add(key); returns 1 when inserted, 0 when already present */
int  pyset_add(pyset* s, uint64_t key, uint64_t hash);
int  pyset_contains(const pyset* s, uint64_t key, uint64_t hash);
/* list(s): writes keys in iteration (slot) order, returns count */
size_t pyset_list(const pyset* s, uint64_t* keys_out, uint64_t* hashes_out);
/* out = a & b, with CPython's operand-swap rule */
void pyset_intersection(const pyset* a, const pyset* b, pyset* out);

/* tuple <-> key id helpers: id = len in the top byte, items base-16 below */
uint64_t pyset_tuple_key(const int* items, int len);
void     pyset_key_tuple(uint64_t key, int* items_out, int* len_out);

#ifdef __cplusplus
}
#endif
#endif
