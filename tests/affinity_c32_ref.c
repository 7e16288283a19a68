/* affinity_c32_ref.c -- TEST INFRASTRUCTURE: the exact fp32 affinity cost c32 of DESIGN.md 3.6 / 3.15 and the lists it defines,
 * written from DESIGN.md alone (no header shared with the CUDA sources, as in oracle/).
 *
 *   c32(f, F_j) = -acc,  acc = fmaf(f[k], F_j[k], acc) for k = 0..K-1 from 0.f
 *
 * C99 fmaf is correctly rounded, so with denormals kept (no fast-math, -ffp-contract=off) this is the device's fmaf bit for bit.
 * Lists compare costs with float `<`: -0 == +0, and equal costs go to the lower node index.
 *
 * Mode 0 is c32.  Modes 1..7 are MUTANTS: plausible ways a kernel could be subtly wrong, used only to prove that the fixtures of
 * tests/test_gpu_affinity_c32.py would notice.  Mode 8 is the six-term bf16 split of the tensor-core path with its accumulation
 * done exactly (fp64, every term is exact there) and rounded once: the split itself, with no accumulation error. */
#include <math.h>
#include <pthread.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

enum {
    M_C32 = 0,
    M_SEPARATE = 1,   /* p = f*F rounded, then acc + p rounded */
    M_REVERSED = 2,   /* fmaf over k = K-1..0 */
    M_FP64 = 3,       /* fp64 dot rounded to fp32 */
    M_PAIRWISE = 4,   /* fp32 products summed as a binary tree */
    M_INTIMAGE = 5,   /* c32, but ordered by the integer image of the float: -0 before +0 */
    M_BF16 = 6,       /* fmaf chain over bf16(f) * bf16(F): one term of the split */
    M_SPLIT5 = 7,     /* the split without the hl term */
    M_SPLIT6 = 8      /* the six-term split, exact accumulation */
};

#define NONE 0xFFFFFFFFu

static float bf16(float x) {   /* round to nearest even, to 8 significant bits */
    uint32_t u;
    memcpy(&u, &x, 4);
    u += 0x7FFFu + ((u >> 16) & 1u);
    u &= 0xFFFF0000u;
    memcpy(&x, &u, 4);
    return x;
}

static void split3(float a, float *h, float *m, float *l) {
    *h = bf16(a);
    const float r1 = a - *h;
    *m = bf16(r1);
    *l = bf16(r1 - *m);
}

static float pairwise(const float *p, uint32_t n) {
    if (n == 1) return p[0];
    const uint32_t h = n / 2;
    const float a = pairwise(p, h), b = pairwise(p + h, n - h);
    return a + b;
}

static float cost(const float *f, const float *g, uint32_t K, int mode) {
    float acc = 0.f;
    switch (mode) {
        case M_SEPARATE:
            for (uint32_t k = 0; k < K; k++) { const float p = f[k] * g[k]; acc = acc + p; }
            return -acc;
        case M_REVERSED:
            for (uint32_t k = K; k-- > 0;) acc = fmaf(f[k], g[k], acc);
            return -acc;
        case M_FP64: {
            double s = 0.0;
            for (uint32_t k = 0; k < K; k++) s += (double)f[k] * (double)g[k];
            return (float)-s;
        }
        case M_PAIRWISE: {
            float p[256];
            for (uint32_t k = 0; k < K; k++) p[k] = f[k] * g[k];
            return -pairwise(p, K);
        }
        case M_BF16:
            for (uint32_t k = 0; k < K; k++) acc = fmaf(bf16(f[k]), bf16(g[k]), acc);
            return -acc;
        case M_SPLIT5:
        case M_SPLIT6: {
            double s = 0.0;
            for (uint32_t k = 0; k < K; k++) {
                float a[3], b[3];
                split3(f[k], &a[0], &a[1], &a[2]);
                split3(g[k], &b[0], &b[1], &b[2]);
                /* hh, hm, mh, mm, hl, lh (0 = h, 1 = m, 2 = l) */
                s += (double)a[0] * b[0] + (double)a[0] * b[1] + (double)a[1] * b[0] + (double)a[1] * b[1] + (double)a[2] * b[0];
                if (mode == M_SPLIT6) s += (double)a[0] * b[2];
            }
            return (float)-s;
        }
        default:
            for (uint32_t k = 0; k < K; k++) acc = fmaf(f[k], g[k], acc);
            return -acc;
    }
}

static int32_t image(float c) {
    uint32_t b;
    memcpy(&b, &c, 4);
    return (int32_t)(b ^ ((uint32_t)((int32_t)b >> 31) & 0x7FFFFFFFu));
}

/* (c, j) strictly before (c2, j2) */
static int before(float c, uint32_t j, float c2, uint32_t j2, int mode) {
    if (mode == M_INTIMAGE) {
        const int32_t a = image(c), b = image(c2);
        return a < b || (a == b && j < j2);
    }
    return c < c2 || (c == c2 && j < j2);
}

typedef struct {
    const float *fo, *fn;
    uint64_t n;
    uint32_t M, K, R;
    const uint8_t *live;
    const uint32_t *dom;   /* NULL: ranked; else failure-domain lists, NONE = a domain of its own */
    int mode;
    float *costs;          /* n x M */
    double *S;             /* n x M */
    uint32_t *out;         /* n x R */
    uint64_t next;
    pthread_mutex_t mu;
} job;

static void row(job *J, uint64_t i, float *c) {
    const float *f = J->fo + i * J->K;
    if (J->costs || J->out)
        for (uint32_t j = 0; j < J->M; j++) c[j] = cost(f, J->fn + (size_t)j * J->K, J->K, J->mode);
    if (J->costs) memcpy(J->costs + i * J->M, c, (size_t)J->M * 4);
    if (J->S)
        for (uint32_t j = 0; j < J->M; j++) {
            double s = 0.0;
            for (uint32_t k = 0; k < J->K; k++) s += fabs((double)f[k] * (double)J->fn[(size_t)j * J->K + k]);
            J->S[i * J->M + j] = s;
        }
    if (!J->out) return;
    /* rank by rank: the first (c, j) among live nodes not listed (ranked) or outside every listed domain (failure-domain) */
    uint32_t *o = J->out + i * J->R;
    for (uint32_t r = 0; r < J->R; r++) {
        uint32_t best = NONE;
        for (uint32_t j = 0; j < J->M; j++) {
            if (!J->live[j]) continue;
            int excluded = 0;
            for (uint32_t x = 0; x < r && !excluded; x++)
                excluded = o[x] == j || (J->dom && J->dom[j] != NONE && J->dom[o[x]] == J->dom[j]);
            if (excluded) continue;
            if (best == NONE || before(c[j], j, c[best], best, J->mode)) best = j;
        }
        o[r] = best;
    }
}

static void *worker(void *arg) {
    job *J = (job *)arg;
    float *c = (float *)malloc((size_t)(J->M ? J->M : 1) * 4);
    for (;;) {
        pthread_mutex_lock(&J->mu);
        const uint64_t lo = J->next;
        J->next += 64;
        pthread_mutex_unlock(&J->mu);
        if (lo >= J->n) break;
        const uint64_t hi = lo + 64 < J->n ? lo + 64 : J->n;
        for (uint64_t i = lo; i < hi; i++) row(J, i, c);
    }
    free(c);
    return NULL;
}

static void run(job *J, int threads) {
    pthread_t t[64];
    if (threads < 1) threads = 1;
    if (threads > 64) threads = 64;
    J->next = 0;
    pthread_mutex_init(&J->mu, NULL);
    for (int x = 0; x < threads; x++) pthread_create(&t[x], NULL, worker, J);
    for (int x = 0; x < threads; x++) pthread_join(t[x], NULL);
    pthread_mutex_destroy(&J->mu);
}

/* n x M costs under `mode` and (when S is not NULL) n x M sums sum_k |f_k F_jk| in fp64 */
void c32_costs(const float *fo, uint64_t n, const float *fn, uint32_t M, uint32_t K, int mode, float *costs, double *S, int threads) {
    job J = {fo, fn, n, M, K, 0, NULL, NULL, mode, costs, S, NULL, 0, {{0}}};
    run(&J, threads);
}

/* n x R lists: the first R live nodes in (cost, j) order, or with dom the best R domain representatives; NONE past the live set */
void c32_lists(const float *fo, uint64_t n, const float *fn, uint32_t M, uint32_t K, const uint8_t *live, const uint32_t *dom, uint32_t R, int mode,
               uint32_t *out, int threads) {
    job J = {fo, fn, n, M, K, R, live, dom, mode, NULL, NULL, out, 0, {{0}}};
    run(&J, threads);
}
