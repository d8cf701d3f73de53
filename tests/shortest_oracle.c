// shortest() without weights restated line by line: query/shortest.go expandOut :141-273 and shortestPath's Dijkstra
// loop :457-618, with numpaths 1, no facets (getCost returns 1 for every edge) and no maxfrontiersize.
// TEST INFRASTRUCTURE ONLY: the checker of dgx_path_search in tests/ and the CPU leg of tools/bench_ops.py C16.
//
// Go's maps become hash tables with last-writer semantics, container/heap becomes a binary heap with its sift rules
// (up / down / Fix exactly as in the Go standard library), and the random order of `for toUID := range neighbours`
// becomes a seeded shuffle of the neighbour list, so different seeds stand for different map iteration orders.
// ProcessGraph is restated for a child with a uid predicate and an optional filter: row i is the predicate's sorted
// adjacency of SrcUIDs[i], DestUIDs is the merge of the rows, intersected with the filter's allowed uids.
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef struct {
    uint64_t* key;  // pairs (a, b); a == 0 marks a free slot (uid 0 is never a node)
    int64_t* val;
    size_t cap, n;
} Map;

static uint64_t mix(uint64_t a, uint64_t b) {
    uint64_t h = a * 0x9E3779B97F4A7C15ull ^ (b + 0x632BE59BD9B4E019ull + (a << 6) + (a >> 2));
    h ^= h >> 31;
    h *= 0xBF58476D1CE4E5B9ull;
    return h ^ (h >> 29);
}

static int map_init(Map* m, size_t cap) {
    m->cap = cap;
    m->n = 0;
    m->key = calloc(2 * cap, sizeof(uint64_t));
    m->val = calloc(cap, sizeof(int64_t));
    return m->key && m->val ? 0 : -1;
}

static void map_free(Map* m) {
    free(m->key);
    free(m->val);
}

static size_t map_slot(const Map* m, uint64_t a, uint64_t b) {
    size_t i = mix(a, b) & (m->cap - 1);
    while (m->key[2 * i] && (m->key[2 * i] != a || m->key[2 * i + 1] != b)) i = (i + 1) & (m->cap - 1);
    return i;
}

static int64_t* map_get(const Map* m, uint64_t a, uint64_t b) {
    const size_t i = map_slot(m, a, b);
    return m->key[2 * i] ? &m->val[i] : NULL;
}

// Inserts or overwrites (last writer wins); *fresh tells which.
static int map_put(Map* m, uint64_t a, uint64_t b, int64_t v, int* fresh) {
    if (2 * (m->n + 1) > m->cap) {
        Map g;
        if (map_init(&g, 2 * m->cap)) return -1;
        for (size_t i = 0; i < m->cap; ++i)
            if (m->key[2 * i]) {
                const size_t j = map_slot(&g, m->key[2 * i], m->key[2 * i + 1]);
                g.key[2 * j] = m->key[2 * i];
                g.key[2 * j + 1] = m->key[2 * i + 1];
                g.val[j] = m->val[i];
            }
        g.n = m->n;
        map_free(m);
        *m = g;
    }
    const size_t i = map_slot(m, a, b);
    *fresh = !m->key[2 * i];
    if (*fresh) {
        m->key[2 * i] = a;
        m->key[2 * i + 1] = b;
        m->n++;
    }
    m->val[i] = v;
    return 0;
}

typedef struct {
    uint64_t* a;
    size_t n, cap;
} Vec;

static int vec_push(Vec* v, uint64_t x) {
    if (v->n == v->cap) {
        const size_t c = v->cap ? 2 * v->cap : 16;
        uint64_t* p = realloc(v->a, c * sizeof(uint64_t));
        if (!p) return -1;
        v->a = p;
        v->cap = c;
    }
    v->a[v->n++] = x;
    return 0;
}

// ---- the graph and ProcessGraph --------------------------------------------------------------------------------------
typedef struct {
    int npred;
    const uint64_t* const* off;  // pred p, node u: adj[p][off[p][u] .. off[p][u+1]), ascending
    const uint64_t* const* adj;
    uint64_t nnodes;
    int nchild;
    const int* child_pred;
    const uint64_t* const* allow;  // child c's filter: allowed uids, ascending; NULL: no filter
    const uint64_t* nallow;
} Graph;

typedef struct {
    int child;
    Vec src;
    Vec* rows;  // uidMatrix, one per src
    Vec dest;   // DestUIDs
} Sg;

static int has(const uint64_t* a, uint64_t n, uint64_t x) {
    uint64_t lo = 0, hi = n;
    while (lo < hi) {
        const uint64_t mid = (lo + hi) / 2;
        if (a[mid] < x) lo = mid + 1; else hi = mid;
    }
    return lo < n && a[lo] == x;
}

static int cmp_u64(const void* x, const void* y) {
    const uint64_t a = *(const uint64_t*)x, b = *(const uint64_t*)y;
    return a < b ? -1 : a > b;
}

// ProcessGraph for one child sg, then updateUidMatrix (:194): rows intersected with DestUIDs.
static int process(const Graph* G, Sg* sg) {
    const int p = G->child_pred[sg->child];
    sg->rows = calloc(sg->src.n ? sg->src.n : 1, sizeof(Vec));
    if (!sg->rows) return -1;
    Vec all = {0};
    for (size_t i = 0; i < sg->src.n; ++i) {
        const uint64_t u = sg->src.a[i];
        if (u >= G->nnodes) continue;
        for (uint64_t k = G->off[p][u]; k < G->off[p][u + 1]; ++k)
            if (vec_push(&sg->rows[i], G->adj[p][k]) || vec_push(&all, G->adj[p][k])) return -1;
    }
    qsort(all.a, all.n, sizeof(uint64_t), cmp_u64);
    for (size_t i = 0; i < all.n; ++i) {
        if (i && all.a[i] == all.a[i - 1]) continue;
        if (G->allow[sg->child] && !has(G->allow[sg->child], G->nallow[sg->child], all.a[i])) continue;
        if (vec_push(&sg->dest, all.a[i])) return -1;
    }
    free(all.a);
    for (size_t i = 0; i < sg->src.n; ++i) {  // algo.IntersectWith(l, sg.DestUIDs, l)
        size_t w = 0;
        for (size_t k = 0; k < sg->rows[i].n; ++k)
            if (has(sg->dest.a, sg->dest.n, sg->rows[i].a[k])) sg->rows[i].a[w++] = sg->rows[i].a[k];
        sg->rows[i].n = w;
    }
    return 0;
}

static void sg_free(Sg* sg) {
    if (sg->rows)
        for (size_t i = 0; i < sg->src.n; ++i) free(sg->rows[i].a);
    free(sg->rows);
    free(sg->src.a);
    free(sg->dest.a);
}

// ---- expandOut ------------------------------------------------------------------------------------------------------
typedef struct {
    const Graph* G;
    Sg* exec;
    size_t nexec;
    Map adj_attr;  // (from, to) -> attr: adjacencyMap[from][to].attr
    Map adj_keys;  // (from, 0) -> index into nbr: adjacencyMap's keys
    Vec* nbr;      // the neighbour list of each key, in insertion order
    size_t nnbr, nbr_cap;
    uint64_t num_edges;
} Expand;

enum { EX_NEXT = 0, EX_STOP = 1, EX_OOM = -1 };

// One level (:158-271): returns EX_NEXT, EX_STOP (errStop) or EX_OOM.
static int expand_level(Expand* E) {
    for (size_t e = 0; e < E->nexec; ++e)
        if (process(E->G, &E->exec[e])) return EX_OOM;
    for (size_t e = 0; e < E->nexec; ++e) {
        Sg* sg = &E->exec[e];
        for (size_t m = 0; m < sg->src.n; ++m) {
            const uint64_t from = sg->src.a[m];
            for (size_t l = 0; l < sg->rows[m].n; ++l) {
                const uint64_t to = sg->rows[m].a[l];
                int fresh;
                if (!map_get(&E->adj_keys, from, 0)) {  // adjacencyMap[fromUID] = make(map[uint64]mapItem)
                    if (E->nnbr == E->nbr_cap) {
                        const size_t c = E->nbr_cap ? 2 * E->nbr_cap : 64;
                        Vec* p = realloc(E->nbr, c * sizeof(Vec));
                        if (!p) return EX_OOM;
                        memset(p + E->nbr_cap, 0, (c - E->nbr_cap) * sizeof(Vec));
                        E->nbr = p;
                        E->nbr_cap = c;
                    }
                    if (map_put(&E->adj_keys, from, 0, (int64_t)E->nnbr++, &fresh)) return EX_OOM;
                }
                if (map_put(&E->adj_attr, from, to, sg->child, &fresh)) return EX_OOM;  // the last writer wins (:220)
                if (fresh && vec_push(&E->nbr[*map_get(&E->adj_keys, from, 0)], to)) return EX_OOM;
                E->num_edges++;
            }
        }
    }
    Vec out_child = {0};  // the next exec list: (child, index of the sg whose DestUIDs it takes)
    for (size_t e = 0; e < E->nexec; ++e) {
        Sg* sg = &E->exec[e];
        if (sg->dest.n == 0) continue;
        size_t w = 0;  // algo.ApplyFilter(temp.SrcUIDs, !adjacencyMap[uid]), in place on the shared DestUIDs
        for (size_t k = 0; k < sg->dest.n; ++k)
            if (!map_get(&E->adj_keys, sg->dest.a[k], 0)) sg->dest.a[w++] = sg->dest.a[k];
        sg->dest.n = w;
        for (int c = 0; c < E->G->nchild; ++c)
            if (vec_push(&out_child, ((uint64_t)e << 16) | (uint64_t)c)) return EX_OOM;
    }
    Sg* next = calloc(out_child.n ? out_child.n : 1, sizeof(Sg));
    if (!next) return EX_OOM;
    for (size_t i = 0; i < out_child.n; ++i) {
        const Sg* from = &E->exec[out_child.a[i] >> 16];
        next[i].child = (int)(out_child.a[i] & 0xffff);
        for (size_t k = 0; k < from->dest.n; ++k)
            if (vec_push(&next[i].src, from->dest.a[k])) return EX_OOM;
    }
    for (size_t e = 0; e < E->nexec; ++e) sg_free(&E->exec[e]);
    free(E->exec);
    E->exec = next;
    E->nexec = out_child.n;
    free(out_child.a);
    return E->nexec == 0 ? EX_STOP : EX_NEXT;
}

// ---- shortestPath's Dijkstra loop -----------------------------------------------------------------------------------
typedef struct {
    uint64_t uid;
    int64_t cost, hop, index;
} Item;

typedef struct {
    Item** h;
    size_t n, cap;
} Heap;

static int less(const Heap* q, size_t i, size_t j) { return q->h[i]->cost < q->h[j]->cost; }
static void swap(Heap* q, size_t i, size_t j) {
    Item* t = q->h[i];
    q->h[i] = q->h[j];
    q->h[j] = t;
    q->h[i]->index = (int64_t)i;
    q->h[j]->index = (int64_t)j;
}
static void up(Heap* q, size_t j) {
    for (;;) {
        if (j == 0) break;  // i := (j - 1) / 2; i == j
        const size_t i = (j - 1) / 2;
        if (!less(q, j, i)) break;
        swap(q, i, j);
        j = i;
    }
}
static int down(Heap* q, size_t i0, size_t n) {
    size_t i = i0;
    for (;;) {
        const size_t j1 = 2 * i + 1;
        if (j1 >= n) break;
        size_t j = j1;
        if (j1 + 1 < n && less(q, j1 + 1, j1)) j = j1 + 1;
        if (!less(q, j, i)) break;
        swap(q, i, j);
        i = j;
    }
    return i > i0;
}
static int heap_push(Heap* q, Item* it) {
    if (q->n == q->cap) {
        const size_t c = q->cap ? 2 * q->cap : 64;
        Item** p = realloc(q->h, c * sizeof(Item*));
        if (!p) return -1;
        q->h = p;
        q->cap = c;
    }
    it->index = (int64_t)q->n;
    q->h[q->n++] = it;
    up(q, q->n - 1);
    return 0;
}
static Item* heap_pop(Heap* q) {
    const size_t n = q->n - 1;
    swap(q, 0, n);
    down(q, 0, n);
    Item* it = q->h[--q->n];
    it->index = -1;
    return it;
}
static void heap_fix(Heap* q, size_t i) {
    if (!down(q, i, q->n)) up(q, i);
}

static uint64_t rng_next(uint64_t* s) {
    *s ^= *s << 13;
    *s ^= *s >> 7;
    *s ^= *s << 17;
    return *s;
}

// Returns the number of levels expandOut ran, or -1 when out of memory.  Per level: numEdges added, exec sgs.  dist as
// (uid, hop, parent, attr) in no particular order, the adjacency as (from, to, attr), and Go's path (path_len 0 when
// To was not reached).  Output arrays must hold nnodes dist entries, every edge of every predicate, and nnodes path
// uids; level arrays max_levels.
int64_t orc_shortest(int npred, const uint64_t* const* off, const uint64_t* const* adj, uint64_t nnodes, int nchild,
                     const int* child_pred, const uint64_t* const* allow, const uint64_t* nallow, uint64_t from,
                     uint64_t to, int64_t max_hops, uint64_t seed, uint64_t* level_edges, uint64_t* level_sgs,
                     size_t max_levels, uint64_t* d_uid, int64_t* d_hop, uint64_t* d_par, int64_t* d_attr,
                     size_t* nd, uint64_t* a_from, uint64_t* a_to, int64_t* a_attr, size_t* na, uint64_t* path,
                     size_t* path_len) {
    const Graph G = {npred, off, adj, nnodes, nchild, child_pred, allow, nallow};
    Expand E = {0};
    E.G = &G;
    int64_t levels = 0, rc = 0;
    Map dist = {0};  // uid -> index into items (the node), with the mapItem fields alongside
    Vec items_par = {0}, items_attr = {0};
    Item** items = NULL;
    size_t nitems = 0, items_cap = 0;
    Heap pq = {0};
    Vec order = {0};
    *path_len = 0;
    *nd = 0;
    *na = 0;
    if (map_init(&E.adj_attr, 1024) || map_init(&E.adj_keys, 1024) || map_init(&dist, 1024)) { rc = -1; goto done; }
    // exec: one sg per child over SrcUIDs = {From} (:147-155)
    E.exec = calloc(nchild ? nchild : 1, sizeof(Sg));
    if (!E.exec) { rc = -1; goto done; }
    E.nexec = nchild;
    for (int c = 0; c < nchild; ++c) {
        E.exec[c].child = c;
        if (vec_push(&E.exec[c].src, from)) { rc = -1; goto done; }
    }
    if (max_hops == 0) goto done;
#define NEW_ITEM(u, c, hp, par, at)                                                                                    \
    do {                                                                                                               \
        if (nitems == items_cap) {                                                                                     \
            items_cap = items_cap ? 2 * items_cap : 64;                                                                \
            Item** p_ = realloc(items, items_cap * sizeof(Item*));                                                     \
            if (!p_) { rc = -1; goto done; }                                                                           \
            items = p_;                                                                                                \
        }                                                                                                              \
        items[nitems] = calloc(1, sizeof(Item));                                                                       \
        if (!items[nitems]) { rc = -1; goto done; }                                                                    \
        items[nitems]->uid = (u);                                                                                      \
        items[nitems]->cost = (c);                                                                                     \
        items[nitems]->hop = (hp);                                                                                     \
        if (vec_push(&items_par, (par)) || vec_push(&items_attr, (uint64_t)(at))) { rc = -1; goto done; }              \
        int f_;                                                                                                        \
        if (map_put(&dist, (u), 0, (int64_t)nitems, &f_)) { rc = -1; goto done; }                                      \
        nitems++;                                                                                                      \
    } while (0)
    NEW_ITEM(from, 0, 0, 0, -1);
    if (heap_push(&pq, items[0])) { rc = -1; goto done; }
    int64_t num_hops = 0;
    int stop_expansion = 0;
    while (pq.n > 0) {
        Item* item = heap_pop(&pq);
        if (item->uid == to) break;
        if (num_hops < max_hops && item->hop > num_hops - 1) {
            if (!stop_expansion) {
                const uint64_t before = E.num_edges;
                const size_t nsg = E.nexec;
                const int r = expand_level(&E);
                if (r == EX_OOM) { rc = -1; goto done; }
                if ((size_t)levels < max_levels) {
                    level_edges[levels] = E.num_edges - before;
                    level_sgs[levels] = nsg;
                }
                levels++;
                if (r == EX_STOP) stop_expansion = 1;
                num_hops++;
            }
        }
        const int64_t* key = map_get(&E.adj_keys, item->uid, 0);
        if (!key) continue;
        const Vec* nb = &E.nbr[*key];
        order.n = 0;
        for (size_t k = 0; k < nb->n; ++k)
            if (vec_push(&order, nb->a[k])) { rc = -1; goto done; }
        for (size_t k = order.n; k > 1; --k) {  // the map's iteration order
            const size_t j = rng_next(&seed) % k;
            const uint64_t t = order.a[k - 1];
            order.a[k - 1] = order.a[j];
            order.a[j] = t;
        }
        for (size_t k = 0; k < order.n; ++k) {
            const uint64_t to_uid = order.a[k];
            const int64_t attr = *map_get(&E.adj_attr, item->uid, to_uid);
            const int64_t* d = map_get(&dist, to_uid, 0);
            const int64_t node_cost = item->cost + 1;
            if (d && items[*d]->cost <= node_cost) continue;
            if (!d) {
                NEW_ITEM(to_uid, node_cost, item->hop + 1, item->uid, attr);
                if (heap_push(&pq, items[nitems - 1])) { rc = -1; goto done; }
            } else {
                Item* node = items[*d];
                node->cost = node_cost;
                node->hop = item->hop + 1;
                heap_fix(&pq, (size_t)node->index);
                items_par.a[*d] = item->uid;
                items_attr.a[*d] = (uint64_t)attr;
            }
        }
    }
    // the path: parents from To while dist has entries (:596-606)
    {
        const int64_t* dt = map_get(&dist, to, 0);
        uint64_t cur = to;
        size_t n = 0;
        for (size_t k = 0; k < nitems; ++k) {
            path[n++] = cur;
            if (cur == from) break;
            const int64_t* d = map_get(&dist, cur, 0);
            cur = d ? items_par.a[*d] : 0;
        }
        if (dt && cur == from) {
            for (size_t i = 0; i < n / 2; ++i) {
                const uint64_t t = path[i];
                path[i] = path[n - 1 - i];
                path[n - 1 - i] = t;
            }
            *path_len = n;
        }
    }
    for (size_t k = 0; k < nitems; ++k) {
        d_uid[k] = items[k]->uid;
        d_hop[k] = items[k]->hop;
        d_par[k] = items_par.a[k];
        d_attr[k] = (int64_t)items_attr.a[k];
    }
    *nd = nitems;
    {
        size_t n = 0;
        for (size_t i = 0; i < E.adj_attr.cap; ++i)
            if (E.adj_attr.key[2 * i]) {
                a_from[n] = E.adj_attr.key[2 * i];
                a_to[n] = E.adj_attr.key[2 * i + 1];
                a_attr[n++] = E.adj_attr.val[i];
            }
        *na = n;
    }
    rc = levels;
done:
    for (size_t e = 0; e < E.nexec; ++e) sg_free(&E.exec[e]);
    free(E.exec);
    for (size_t k = 0; k < E.nnbr; ++k) free(E.nbr[k].a);
    free(E.nbr);
    map_free(&E.adj_attr);
    map_free(&E.adj_keys);
    map_free(&dist);
    for (size_t k = 0; k < nitems; ++k) free(items[k]);
    free(items);
    free(items_par.a);
    free(items_attr.a);
    free(pq.h);
    free(order.a);
    return rc;
}
