/*
 * spread_oracle.c -- CPU ORACLE for the failure-domain ranked lists (DESIGN.md 3.12); test infrastructure, NOT product code.
 *
 * Restates the definition, not the kernels: rank_r(k) is the policy's placement of k over the live set minus every node whose
 * domain is the domain of one of rank_1(k) .. rank_{r-1}(k), NONE once that set is empty.  Every rank is one more masked single
 * assignment per object with the oracle's own routines of oracle/rio_oracle.c (included whole): the flat policy scans every node
 * with a per-object exclusion mask (hrw_one), HRW2 rebuilds the member list and its prefix sums without the excluded nodes and walks
 * that (h2_range).  A node labelled ORC_NONE is a domain of its own.
 */
#include "../oracle/rio_oracle.c"

static int same_domain(const uint32_t *dom, uint32_t a, uint32_t b) {
    return a == b || (dom[a] != ORC_NONE && dom[a] == dom[b]);
}

typedef struct { const uint64_t *keys, *seed; const uint32_t *dom; node_tab t; uint32_t M, R; uint32_t *out; } sp_hrw_ctx;

static void sp_hrw_range(void *p, size_t lo, size_t hi) {
    sp_hrw_ctx *c = (sp_hrw_ctx *)p;
    uint32_t words = (c->M + 31) / 32;
    uint32_t *mask = (uint32_t *)calloc(words ? words : 1, 4);
    for (size_t i = lo; i < hi; i++) {
        uint32_t *row = c->out + i * c->R;
        for (uint32_t r = 0; r < c->R; r++) {
            uint32_t j = hrw_one(c->keys[i], c->seed, c->t.seed2, c->t.invw, mask, c->M, NULL, NULL);
            row[r] = j;
            if (j == ORC_NONE) continue;
            for (uint32_t q = 0; q < c->M; q++) if (same_domain(c->dom, q, j)) mask[q >> 5] |= 1u << (q & 31);
        }
        memset(mask, 0, 4 * (size_t)(words ? words : 1));
    }
    free(mask);
}

/* out is n x R row-major; weight[j] == 0 means node j is not live; dom[j] is node j's label */
void orc_assign_spread_hrw(const uint64_t *keys, size_t n, const uint64_t *seed, const uint32_t *weight, const uint32_t *dom, uint32_t M,
                           uint32_t R, uint32_t *out, int threads) {
    sp_hrw_ctx c = { keys, seed, dom, make_tab(seed, weight, M), M, R, out };
    par_for(n, threads, sp_hrw_range, &c);
    free(c.t.seed2); free(c.t.invw);
}

typedef struct { const uint64_t *keys; const h2_member *mem; const uint32_t *dom; uint32_t c, bits, R; uint32_t *out; } sp_h2_ctx;

static void sp_h2_range(void *p, size_t lo, size_t hi) {
    sp_h2_ctx *c = (sp_h2_ctx *)p;
    h2_member *sub = (h2_member *)malloc(sizeof(h2_member) * (c->c ? c->c : 1));
    uint64_t *pre = (uint64_t *)malloc(8 * ((size_t)c->c + 1));
    for (size_t i = lo; i < hi; i++) {
        uint32_t *row = c->out + i * c->R;
        for (uint32_t r = 0; r < c->R; r++) {
            uint32_t m = 0;
            for (uint32_t q = 0; q < c->c; q++) {
                int excluded = 0;
                for (uint32_t x = 0; x < r; x++) excluded |= row[x] != ORC_NONE && same_domain(c->dom, row[x], c->mem[q].j);
                if (!excluded) sub[m++] = c->mem[q];
            }
            pre[0] = 0;
            for (uint32_t q = 0; q < m; q++) pre[q + 1] = pre[q] + sub[q].w;
            h2_ctx one = { c->keys + i, sub, pre, m, c->bits, row + r };
            h2_range(&one, 0, 1);   /* NONE when no member is left */
        }
    }
    free(sub); free(pre);
}

void orc_assign_spread_hrw2(const uint64_t *keys, size_t n, const uint64_t *seed, const uint32_t *weight, const uint32_t *dom, uint32_t M,
                            uint32_t bits, uint32_t R, uint32_t *out, int threads) {
    h2_member *mem = (h2_member *)malloc(sizeof(h2_member) * (M ? M : 1));
    uint32_t c = 0;
    for (uint32_t j = 0; j < M; j++) {
        if (!weight[j]) continue;
        mem[c].pos = orc_hrw2_pos(seed[j]); mem[c].seed = seed[j]; mem[c].j = j; mem[c].w = weight[j]; c++;
    }
    qsort(mem, c, sizeof(h2_member), h2_cmp);
    sp_h2_ctx ctx = { keys, mem, dom, c, bits, R, out };
    par_for(n, threads, sp_h2_range, &ctx);
    free(mem);
}
