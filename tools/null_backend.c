/* tools/null_backend.c — MEASUREMENT AID, not a back end: the subset of the libb200av1 C ABI the dav1d hooks bind
 * (integration/dav1d/b200_hooks.c), with a frame job that does nothing. Decoding a stream through the hooked dav1d with
 * this library (`stream.HookedDecoder(backend=".../libnull.so")`, output pictures are garbage) times the host side alone:
 * dav1d's front end + the record emitters + frame completion. DESIGN.md 5b quotes it next to stock dav1d.
 *     gcc -O2 -shared -fPIC -o /tmp/libnull.so tools/null_backend.c */
#include <stdlib.h>
#include <stdint.h>
#include <string.h>
#include "../include/b200av1.h"
const char *b200_last_error(void) { return ""; }
void *b200_dev_alloc(size_t n) { return malloc(n ? n : 1); }
void b200_dev_free(void *p) { free(p); }
void *b200_host_alloc(size_t n) { return malloc(n ? n : 1); }
void b200_host_free(void *p) { free(p); }
void *b200_stream_create(void) { return (void *)1; }
void b200_stream_destroy(void *s) { (void)s; }
size_t b200_intra_scratch_bytes(const B200IntraFrame *f) { (void)f; return 1 << 20; }
int b200_frame_run_host(const B200FrameJob *j, const B200Xfer *u, int nu, const B200Xfer *d, int nd, void *s) { (void)j; (void)u; (void)nu; (void)d; (void)nd; (void)s; return 0; }
int b200_frame_submit_host(const B200FrameJob *j, const B200Xfer *u, int nu, const B200Xfer *d, int nd, void *s) { (void)j; (void)u; (void)nu; (void)d; (void)nd; (void)s; return 0; }
int b200_frame_wait(void *s) { (void)s; return 0; }
int b200_copy_async(void *d, const void *src, size_t n, void *s) { (void)d; (void)src; (void)n; (void)s; return 0; }
void *b200_event_create(void) { return (void *)1; }
void b200_event_destroy(void *e) { (void)e; }
int b200_event_record(void *e, void *s) { (void)e; (void)s; return 0; }
int b200_stream_wait_event(void *s, void *e) { (void)s; (void)e; return 0; }
int b200_struct_size(int w) { switch (w) { case 9: return sizeof(B200FrameJob); case 14: return sizeof(B200IntraTx); case 10: return sizeof(B200Av1Filter); case 11: return sizeof(B200Av1Restoration); case 22: return sizeof(B200ExportJob); case 23: return sizeof(B200TensorJob); case 24: return sizeof(B200ToneMap); case 25: return sizeof(B200ColorJitter); } return -1; }
int b200_event_sync(void *e) { (void)e; return 0; }
int b200_export_picture(const B200ExportJob *j, void *s) { (void)j; (void)s; return 0; }
int b200_export_tensor(const B200TensorJob *j, void *s) { (void)j; (void)s; return 0; }
int b200_export_tensor_batch(const B200TensorJob *j, int n, void *s) { (void)j; (void)n; (void)s; return 0; }
int b200_export_tensor_tone_batch(const B200TensorJob *j, const B200ToneMap *const *t, int n, void *s) { (void)j; (void)t; (void)n; (void)s; return 0; }
int b200_export_tensor_jitter_batch(const B200TensorJob *j, const B200ToneMap *const *t, const B200ColorJitter *const *c, int n, void *s) { (void)j; (void)t; (void)c; (void)n; (void)s; return 0; }
