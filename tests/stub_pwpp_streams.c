/* TEST-ONLY stand-in for libpwpp_b200.so with the stream table: what tests/stub_pwpp.c offers plus
 * pwpp_estimate_host_streams, for the several-streams form of examples/pwpp_sequence.cpp in the GPU-less build container
 * (tests/test_examples_streams.py). "Ground" = points with z < -1.5.
 * pwpp_estimate_host labels frame 0 of a call; pwpp_estimate_host_streams labels every frame of the call, keeps the results
 * by call position and counts the frames each stream was given (the stub's "height" of a stream is 1.723 + that count). */
#include <stdlib.h>
#include <string.h>
#include "pwpp.h"
struct stub_frame { int32_t* g; int32_t* ng; int64_t ngr, nng; };
struct pwpp_ctx { int nf, cap, ns; struct stub_frame* fr; int64_t* seen; double h; };
static void stub_reset(pwpp_ctx* c, int nf) {
  for (int f = 0; f < c->cap; ++f) { free(c->fr[f].g); free(c->fr[f].ng); }
  free(c->fr);
  c->fr = calloc((size_t) nf, sizeof(struct stub_frame));
  c->cap = c->nf = nf;
}
static void stub_label(struct stub_frame* o, const float* p, int64_t n, int64_t rs, int64_t cs) {
  o->g = malloc(sizeof(int32_t) * (size_t) (n + 1)); o->ng = malloc(sizeof(int32_t) * (size_t) (n + 1));
  o->ngr = o->nng = 0;
  for (int64_t i = 0; i < n; ++i) { if (p[i * rs + 2 * cs] < -1.5f) o->g[o->ngr++] = (int32_t) i; else o->ng[o->nng++] = (int32_t) i; }
}
void pwpp_params_default(pwpp_params* p) { memset(p, 0, sizeof *p); p->num_zones = 4; }
int pwpp_create(const pwpp_params* p, int device, int ns, int64_t m, pwpp_ctx** out) {
  (void) p; (void) device; (void) m;
  *out = calloc(1, sizeof(pwpp_ctx)); (*out)->h = 1.723; (*out)->ns = ns; (*out)->seen = calloc((size_t) (ns > 0 ? ns : 1), sizeof(int64_t));
  return 0;
}
void pwpp_destroy(pwpp_ctx* c) { if (c) { stub_reset(c, 0); free(c->seen); free(c); } }
const char* pwpp_last_error(void) { return "stub"; }
void* pwpp_host_alloc(size_t b) { return malloc(b ? b : 1); }
void pwpp_host_free(void* p) { free(p); }
int pwpp_estimate_host(pwpp_ctx* c, int nf, const float* const* pts, const int64_t* n, int cols, int64_t rs, int64_t cs) {
  (void) nf; (void) cols;
  stub_reset(c, 1);
  stub_label(&c->fr[0], pts[0], n[0], rs, cs);
  return 0;
}
int pwpp_estimate_host_streams(pwpp_ctx* c, int nf, const int32_t* streams, const float* const* pts, const int64_t* n, int cols, int64_t rs,
                               int64_t cs) {
  (void) cols;
  if (!streams || nf < 1) return PWPP_ERR_INVALID_ARG;
  for (int f = 0; f < nf; ++f) if (streams[f] < 0 || streams[f] >= c->ns) return PWPP_ERR_INVALID_ARG;
  stub_reset(c, nf);
  for (int f = 0; f < nf; ++f) { stub_label(&c->fr[f], pts[f], n[f], rs, cs); ++c->seen[streams[f]]; }
  return 0;
}
int64_t pwpp_num_ground(pwpp_ctx* c, int f) { return c->fr[f].ngr; }
int64_t pwpp_num_nonground(pwpp_ctx* c, int f) { return c->fr[f].nng; }
int pwpp_copy_ground_indices(pwpp_ctx* c, int f, int32_t* d) { memcpy(d, c->fr[f].g, sizeof(int32_t) * (size_t) c->fr[f].ngr); return 0; }
int pwpp_copy_nonground_indices(pwpp_ctx* c, int f, int32_t* d) { memcpy(d, c->fr[f].ng, sizeof(int32_t) * (size_t) c->fr[f].nng); return 0; }
int pwpp_copy_ground_xyz(pwpp_ctx* c, int f, float* d) { (void) c; (void) f; (void) d; return 0; }
int pwpp_copy_nonground_xyz(pwpp_ctx* c, int f, float* d) { (void) c; (void) f; (void) d; return 0; }
int pwpp_num_patches(pwpp_ctx* c, int f) { (void) c; (void) f; return 2; }
int pwpp_copy_centers(pwpp_ctx* c, int f, float* d) { (void) c; (void) f; memset(d, 0, 24); return 0; }
int pwpp_copy_normals(pwpp_ctx* c, int f, float* d) { (void) c; (void) f; memset(d, 0, 24); return 0; }
double pwpp_height(pwpp_ctx* c, int f) { return (f >= 0 && f < c->ns) ? c->h + (double) c->seen[f] : c->h; }
double pwpp_time_us(pwpp_ctx* c) { (void) c; return 1000.0; }
int pwpp_set_output_order(pwpp_ctx* c, int order) { (void) c; (void) order; return 0; }
int pwpp_device_synchronize(pwpp_ctx* c) { (void) c; return 0; }
int pwpp_estimate_device(pwpp_ctx* c, int nf, const void* d, const int64_t* o, int hi, void* s) { (void) c; (void) nf; (void) d; (void) o; (void) hi; (void) s; return -1; }
int pwpp_estimate_device_streams(pwpp_ctx* c, int nf, const int32_t* st, const void* d, const int64_t* o, int hi, void* s) {
  (void) c; (void) nf; (void) st; (void) d; (void) o; (void) hi; (void) s; return -1;
}
int pwpp_estimate_device_xyz(pwpp_ctx* c, int nf, const void* d, const int64_t* o, void* s) { (void) c; (void) nf; (void) d; (void) o; (void) s; return -1; }
int pwpp_device_results(pwpp_ctx* c, const int32_t** a, const int32_t** b) { (void) c; if (a) *a = 0; if (b) *b = 0; return 0; }
