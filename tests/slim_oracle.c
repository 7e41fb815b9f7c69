/*
 * slim_oracle.c — SLIM / fsSLIM column training restated from its contract, one statement per step, for the
 * tests and the CPU arm of tools/slim_bench.py.  Build with -O2 -ffp-contract=off -fopenmp: every f32 operation
 * is a separate IEEE operation, as in the reference's Rust (which never contracts into FMAs).
 *
 * For target item i with users U_i = IU row i in stored order:
 *   1. resid[u] = 1 for u in U_i, 0 elsewhere;
 *   2. active: the items j != i of the UI rows of U_i, walked in stored order, in first-encounter order; pc[j]
 *      counts the encounters;
 *   3. fsSLIM (0 <= k < |active|): stable sort by the f64 key -(pc[j]) / (sqrt(|U_i|) * sqrt(|U_j|)), keep k;
 *   4. up to max_iters rounds: for j in active: upd = 0; upd += (resid[u] + W[j]) for u in U_j;
 *      new = upd >= l1 ? (upd - l1) / ((float)|U_j| + l2) : 0; diff = new - W[j]; W[j] = new;
 *      resid[u] -= diff for u in U_j; the round's max |diff| <= 1e-3f ends the descent;
 *   5. output: every j ascending with W[j] >= 1e-12f.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef struct {
    double key;
    int32_t pos;
    int32_t item;
} slim_key;

static int key_cmp(const void *pa, const void *pb)
{
    const slim_key *a = pa, *b = pb;
    if (a->key < b->key) return -1;
    if (a->key > b->key) return 1;
    return (a->pos > b->pos) - (a->pos < b->pos);  /* a stable sort keeps first-encounter order on ties */
}

typedef struct {
    int32_t n_cols;
    int64_t *count;    /* [n_cols] */
    int32_t **items;   /* [n_cols] */
    float **values;    /* [n_cols] */
} slim_result;

static void train_column(int32_t item, int32_t n_users, int32_t n_items, const int64_t *ui_ptr,
                         const int32_t *ui_cols, const int64_t *iu_ptr, const int32_t *iu_cols, float l1, float l2,
                         int32_t max_iters, int64_t max_nbrs, float *resid, float *w, int32_t *pc, int32_t *active,
                         slim_key *keys, int64_t *count, int32_t **items, float **values)
{
    (void)n_users;
    const int64_t i0 = iu_ptr[item], ni = iu_ptr[item + 1] - i0;

    /* 1 and 2 */
    int64_t n_act = 0;
    for (int64_t p = i0; p < i0 + ni; p++) {
        const int32_t u = iu_cols[p];
        resid[u] = 1.0f;
        for (int64_t q = ui_ptr[u]; q < ui_ptr[u + 1]; q++) {
            const int32_t j = ui_cols[q];
            if (j != item) {
                if (pc[j] == 0) active[n_act++] = j;
                pc[j] += 1;
            }
        }
    }

    /* 3 */
    int64_t n_cd = n_act;
    if (max_nbrs >= 0 && max_nbrs < n_act) {
        const double i_norm = sqrt((double)ni);
        for (int64_t c = 0; c < n_act; c++) {
            const int32_t j = active[c];
            const double j_norm = sqrt((double)(iu_ptr[j + 1] - iu_ptr[j]));
            keys[c].key = -(double)pc[j] / (i_norm * j_norm);
            keys[c].pos = (int32_t)c;
            keys[c].item = j;
        }
        qsort(keys, (size_t)n_act, sizeof(slim_key), key_cmp);
        for (int64_t c = 0; c < max_nbrs; c++) active[c] = keys[c].item;
        n_cd = max_nbrs;
    }

    /* 4 */
    for (int32_t it = 0; it < max_iters; it++) {
        float dmax = 0.0f;
        for (int64_t c = 0; c < n_cd; c++) {
            const int32_t j = active[c];
            const float cur = w[j];
            float upd = 0.0f;
            for (int64_t p = iu_ptr[j]; p < iu_ptr[j + 1]; p++) {
                const float t = resid[iu_cols[p]] + cur;
                upd = upd + t;
            }
            float nw = 0.0f;
            if (upd >= l1) {
                const float num = upd - l1;
                const float den = (float)(iu_ptr[j + 1] - iu_ptr[j]) + l2;
                nw = num / den;
            }
            const float diff = nw - cur;
            w[j] = nw;
            for (int64_t p = iu_ptr[j]; p < iu_ptr[j + 1]; p++) resid[iu_cols[p]] -= diff;
            const float ad = fabsf(diff);
            if (ad > dmax) dmax = ad;
        }
        if (dmax <= 1e-3f) break;
    }

    /* 5 */
    int64_t n_out = 0;
    for (int32_t j = 0; j < n_items; j++)
        if (w[j] >= 1.0e-12f) n_out++;
    *count = n_out;
    *items = malloc(sizeof(int32_t) * (size_t)(n_out ? n_out : 1));
    *values = malloc(sizeof(float) * (size_t)(n_out ? n_out : 1));
    n_out = 0;
    for (int32_t j = 0; j < n_items; j++) {
        if (w[j] >= 1.0e-12f) {
            (*items)[n_out] = j;
            (*values)[n_out] = w[j];
            n_out++;
        }
    }

    /* reset the scratch for the next column */
    for (int64_t c = 0; c < n_cd; c++) {
        const int32_t j = active[c];
        w[j] = 0.0f;
        for (int64_t p = iu_ptr[j]; p < iu_ptr[j + 1]; p++) resid[iu_cols[p]] = 0.0f;
    }
    for (int64_t p = i0; p < i0 + ni; p++) resid[iu_cols[p]] = 0.0f;
    memset(pc, 0, sizeof(int32_t) * (size_t)n_items);
}

/* Train the columns `columns[0 .. n_cols)`; returns a handle for slim_counts / slim_fetch / slim_free. */
slim_result *slim_train(int32_t n_users, int32_t n_items, const int64_t *ui_ptr, const int32_t *ui_cols,
                        const int64_t *iu_ptr, const int32_t *iu_cols, float l1, float l2, int32_t max_iters,
                        int64_t max_nbrs, const int32_t *columns, int32_t n_cols)
{
    slim_result *r = calloc(1, sizeof(slim_result));
    r->n_cols = n_cols;
    r->count = calloc((size_t)(n_cols ? n_cols : 1), sizeof(int64_t));
    r->items = calloc((size_t)(n_cols ? n_cols : 1), sizeof(int32_t *));
    r->values = calloc((size_t)(n_cols ? n_cols : 1), sizeof(float *));
#pragma omp parallel
    {
        float *resid = calloc((size_t)(n_users ? n_users : 1), sizeof(float));
        float *w = calloc((size_t)n_items, sizeof(float));
        int32_t *pc = calloc((size_t)n_items, sizeof(int32_t));
        int32_t *active = malloc(sizeof(int32_t) * (size_t)n_items);
        slim_key *keys = malloc(sizeof(slim_key) * (size_t)n_items);
#pragma omp for schedule(dynamic, 1)
        for (int32_t c = 0; c < n_cols; c++)
            train_column(columns[c], n_users, n_items, ui_ptr, ui_cols, iu_ptr, iu_cols, l1, l2, max_iters, max_nbrs,
                         resid, w, pc, active, keys, &r->count[c], &r->items[c], &r->values[c]);
        free(resid);
        free(w);
        free(pc);
        free(active);
        free(keys);
    }
    return r;
}

void slim_counts(const slim_result *r, int64_t *count)
{
    memcpy(count, r->count, sizeof(int64_t) * (size_t)r->n_cols);
}

/* the columns' entries one after the other, in the order they were given */
void slim_fetch(const slim_result *r, int32_t *items, float *values)
{
    int64_t at = 0;
    for (int32_t c = 0; c < r->n_cols; c++) {
        memcpy(items + at, r->items[c], sizeof(int32_t) * (size_t)r->count[c]);
        memcpy(values + at, r->values[c], sizeof(float) * (size_t)r->count[c]);
        at += r->count[c];
    }
}

void slim_free(slim_result *r)
{
    for (int32_t c = 0; c < r->n_cols; c++) {
        free(r->items[c]);
        free(r->values[c]);
    }
    free(r->count);
    free(r->items);
    free(r->values);
    free(r);
}
