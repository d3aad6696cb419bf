/* Load for the name recycling race test (tests/_name_recycling_cases.py): threads call Histogram / Counter through
 * the mirror's C entry points over a window of names that the collecting thread slides forward, so ids are retired,
 * freed and handed to new names while samples are in flight.
 *
 * The window only moves once every thread has finished a call that read the current position, so an in-flight
 * call uses the position or the one before it.  The collector moves it at most once per collection, so names used
 * in any three consecutive intervals number at most window + 3, whatever the scheduler does, and a table of that
 * size never drops a sample. */
#include <pthread.h>
#include <stdatomic.h>
#include <stdint.h>
#include <stdlib.h>
#include <time.h>

typedef void (*hist_fn)(void *ms, const char *name, double value);
typedef void (*ctr_fn)(void *ms, const char *name, uint64_t amount);

typedef struct race race;
typedef struct {
    race *r;
    int index;
    pthread_t tid;
} worker;

struct race {
    void *ms;
    hist_fn hist;
    ctr_fn ctr;
    const char *const *hnames, *const *cnames;
    const double *values;
    const uint64_t *amounts;
    uint32_t nnames, window;
    int threads;
    _Atomic uint32_t base;     /* lowest name of the window */
    _Atomic uint32_t *acks;    /* per thread: the position its last completed call read */
    uint64_t *hcalls, *ccalls; /* [threads][nnames] */
    worker *workers;
};

static uint64_t next_rand(uint64_t *s) {
    *s ^= *s << 13;
    *s ^= *s >> 7;
    *s ^= *s << 17;
    return *s;
}

static void *run(void *arg) {
    worker *w = arg;
    race *r = w->r;
    uint64_t rng = 0x9E3779B97F4A7C15ull * (uint64_t)(w->index + 1);
    uint64_t *hc = r->hcalls + (size_t)w->index * r->nnames, *cc = r->ccalls + (size_t)w->index * r->nnames;
    for (uint64_t k = 1;; k++) {
        const uint32_t b = atomic_load(&r->base);
        if (b + r->window > r->nnames) break;
        const uint64_t x = next_rand(&rng);
        const uint32_t i = b + (uint32_t)(x % r->window);
        if (x >> 63) {
            r->hist(r->ms, r->hnames[i], r->values[i]);
            hc[i]++;
        } else {
            r->ctr(r->ms, r->cnames[i], r->amounts[i]);
            cc[i]++;
        }
        atomic_store(&r->acks[w->index], b);
        if (k % 32 == 0) { /* keep the sample volume modest; calls still overlap every collection */
            struct timespec ts = {0, 20000};
            nanosleep(&ts, NULL);
        }
    }
    return NULL;
}

void *race_start(void *ms, hist_fn hist, ctr_fn ctr, const char *const *hnames, const char *const *cnames,
                 const double *values, const uint64_t *amounts, uint32_t nnames, uint32_t window, int threads) {
    race *r = calloc(1, sizeof *r);
    r->ms = ms; r->hist = hist; r->ctr = ctr;
    r->hnames = hnames; r->cnames = cnames; r->values = values; r->amounts = amounts;
    r->nnames = nnames; r->window = window; r->threads = threads;
    r->acks = calloc((size_t)threads, sizeof *r->acks);
    r->hcalls = calloc((size_t)threads * nnames, sizeof *r->hcalls);
    r->ccalls = calloc((size_t)threads * nnames, sizeof *r->ccalls);
    r->workers = calloc((size_t)threads, sizeof *r->workers);
    for (int t = 0; t < threads; t++) {
        r->workers[t].r = r;
        r->workers[t].index = t;
        pthread_create(&r->workers[t].tid, NULL, run, &r->workers[t]);
    }
    return r;
}

/* Moves the window one name forward if every thread has caught up with it; returns 1 once the threads are done. */
int race_advance(void *h) {
    race *r = h;
    const uint32_t b = atomic_load(&r->base);
    if (b + r->window > r->nnames) return 1;
    for (int t = 0; t < r->threads; t++)
        if (atomic_load(&r->acks[t]) < b) return 0;
    atomic_store(&r->base, b + 1);
    return 0;
}

/* Stops the threads (at once, if the window has not reached the end), joins them and returns the calls they made
 * per name. */
void race_finish(void *h, uint64_t *hcalls, uint64_t *ccalls) {
    race *r = h;
    atomic_store(&r->base, r->nnames);
    for (int t = 0; t < r->threads; t++) pthread_join(r->workers[t].tid, NULL);
    for (uint32_t i = 0; i < r->nnames; i++) {
        hcalls[i] = ccalls[i] = 0;
        for (int t = 0; t < r->threads; t++) {
            hcalls[i] += r->hcalls[(size_t)t * r->nnames + i];
            ccalls[i] += r->ccalls[(size_t)t * r->nnames + i];
        }
    }
    free(r->acks); free(r->hcalls); free(r->ccalls); free(r->workers); free(r);
}
