/* TEST INFRASTRUCTURE: the lazy allocations of stereo rectification in the emulated library (tests/test_rectify_lifetime.py builds both
 * with -fsanitize=address): the fixed-point maps and their float staging (rgbl_set_stereo_rectification) and the raw planes (the first
 * stereo upload, array or PNG, with rectification on).  For each path it fails the k-th allocation of those calls for each k
 * (emu_fail_allocation) and checks that the call reports RGBL_E_CUDA and that a retry on the same context gives the outputs of a fresh
 * context: level 0 of the left slot and the stereo frame (keypoints, descriptors, mvDepth, mvuRight).  LeakSanitizer checks at exit that nothing leaks.
 * Exit 0: every check passed.                                                                                                           */
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <zlib.h>

#include "rgbl_b200.h"

int emu_fail_allocation(int nth);

enum { W = 128, H = 96 };

static int g_failures = 0;
#define CHECK(cond, ...) do { if (!(cond)) { fprintf(stderr, "FAIL %s:%d: ", __FILE__, __LINE__); fprintf(stderr, __VA_ARGS__); fputc('\n', stderr); ++g_failures; } } while (0)

static uint8_t g_left[W * H], g_right[W * H];
static float g_mx[W * H], g_my[W * H];
static uint8_t* g_png[2]; static size_t g_png_n[2];

static rgbl_ctx* new_ctx(void) {
    rgbl_config cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.width = W; cfg.height = H; cfg.max_batch = 2;
    cfg.orb.nfeatures = 100; cfg.orb.scale_factor = 1.2f; cfg.orb.nlevels = 2; cfg.orb.ini_th_fast = 20; cfg.orb.min_th_fast = 7;
    rgbl_ctx* c = NULL;
    if (rgbl_create(&cfg, &c)) { fprintf(stderr, "rgbl_create: %s\n", rgbl_last_error(NULL)); exit(2); }
    rgbl_set_host_quadtree(c, 1);
    return c;
}

static uint8_t* encode_png(const uint8_t* gray, size_t* n_out) {       /* 8-bit gray, filter type 0 */
    const size_t row = W + 1, raw_n = row * H;
    uint8_t* raw = (uint8_t*)calloc(raw_n, 1);
    for (int y = 0; y < H; ++y) memcpy(raw + y * row + 1, gray + (size_t)y * W, W);
    uLongf z_n = compressBound(raw_n);
    uint8_t* z = (uint8_t*)malloc(z_n);
    compress(z, &z_n, raw, raw_n);
    uint8_t* png = (uint8_t*)malloc(8 + 25 + 12 + z_n + 12);
    static const uint8_t sig[8] = {137, 'P', 'N', 'G', 13, 10, 26, 10};
    const uint8_t ihdr[13] = {0, 0, W >> 8, W & 255, 0, 0, H >> 8, H & 255, 8, 0, 0, 0, 0};
    const char* types[3] = {"IHDR", "IDAT", "IEND"};
    const uint8_t* data[3] = {ihdr, z, NULL};
    const uint32_t lens[3] = {13, (uint32_t)z_n, 0};
    size_t n = 8;
    memcpy(png, sig, 8);
    for (int i = 0; i < 3; ++i) {
        uint8_t* o = png + n;
        o[0] = lens[i] >> 24; o[1] = lens[i] >> 16; o[2] = lens[i] >> 8; o[3] = lens[i];
        memcpy(o + 4, types[i], 4);
        if (lens[i]) memcpy(o + 8, data[i], lens[i]);
        const uint32_t crc = (uint32_t)crc32(crc32(0L, Z_NULL, 0), o + 4, lens[i] + 4);
        o[8 + lens[i]] = crc >> 24; o[9 + lens[i]] = crc >> 16; o[10 + lens[i]] = crc >> 8; o[11 + lens[i]] = crc;
        n += 12 + lens[i];
    }
    free(raw); free(z);
    *n_out = n;
    return png;
}

static void make_inputs(void) {
    for (int y = 0; y < H; ++y)
        for (int x = 0; x < W; ++x) {
            const int u = x + 4;
            g_left[y * W + x] = (uint8_t)((((x / 12) ^ (y / 12)) & 1) ? 200 - (x % 12) * 9 : 40 + (y % 12) * 7);
            g_right[y * W + x] = (uint8_t)((((u / 12) ^ (y / 12)) & 1) ? 200 - (u % 12) * 9 : 40 + (y % 12) * 7);
            /* a barrel lens around the centre, the map of initUndistortRectifyMap(K, D, I, K) */
            const float xn = (x - 64.f) / 120.f, yn = (y - 48.f) / 120.f, r2 = xn * xn + yn * yn, k = 1.f - 0.25f * r2;
            g_mx[y * W + x] = 64.f + 120.f * xn * k; g_my[y * W + x] = 48.f + 120.f * yn * k;
        }
    g_png[0] = encode_png(g_left, &g_png_n[0]);
    g_png[1] = encode_png(g_right, &g_png_n[1]);
}

typedef struct { uint8_t* p; size_t n; } Bytes;
static void put(Bytes* o, const void* p, size_t n) { o->p = (uint8_t*)realloc(o->p, o->n + n); memcpy(o->p + o->n, p, n); o->n += n; }

/* process the uploaded pair -> level 0 of the left slot and the left frame */
static int process_and_put(rgbl_ctx* c, Bytes* o) {
    int rc = rgbl_resident_process_stereo(c, 0.5f, 75.f, NULL);
    if (rc) return rc;
    uint8_t l0[W * H];
    rc = rgbl_orb_get_level(c, 0, 0, l0, W, NULL, NULL);
    if (rc) return rc;
    put(o, l0, sizeof(l0));
    const int cap = rgbl_keypoint_capacity(c);
    rgbl_keypoint* k = (rgbl_keypoint*)calloc((size_t)cap, sizeof(rgbl_keypoint));
    uint8_t* d = (uint8_t*)calloc((size_t)cap, 32);
    float* dep = (float*)calloc((size_t)cap, sizeof(float)); float* ur = (float*)calloc((size_t)cap, sizeof(float));
    int n = 0;
    rc = rgbl_resident_download(c, k, d, dep, ur, cap, &n);
    if (!rc) { put(o, &n, sizeof(n)); put(o, k, n * sizeof(rgbl_keypoint)); put(o, d, (size_t)n * 32); put(o, dep, n * sizeof(float)); put(o, ur, n * sizeof(float)); }
    free(k); free(d); free(dep); free(ur);
    return rc;
}

/* the rectification setting and the upload of one pair: the calls whose allocations fail in turn */
static int prepare_arrays(rgbl_ctx* c) {
    const uint8_t* l[1] = {g_left}; const uint8_t* r[1] = {g_right};
    const int rc = rgbl_set_stereo_rectification(c, g_mx, g_my, g_mx, g_my, W);
    return rc ? rc : rgbl_resident_upload_stereo(c, 1, l, r, W, H, W);
}

static int prepare_png(rgbl_ctx* c) {
    const uint8_t* l[1] = {g_png[0]}; const uint8_t* r[1] = {g_png[1]};
    size_t ln[1] = {g_png_n[0]}, rn[1] = {g_png_n[1]};
    const int rc = rgbl_set_stereo_rectification(c, g_mx, g_my, g_mx, g_my, W);
    return rc ? rc : rgbl_resident_upload_stereo_png(c, 1, l, ln, r, rn, 0);
}

/* the PNG staging is not the rectification's: allocated beforehand by a plain decode, so that only the rectification's allocations fail */
static void prime_png(rgbl_ctx* c) {
    uint8_t out[W * H]; uint8_t* o[1] = {out};
    const uint8_t* p[1] = {g_png[0]}; size_t n[1] = {g_png_n[0]};
    if (rgbl_decode_png_gray(c, 1, p, n, 0, o, W)) { fprintf(stderr, "PNG decode: %s\n", rgbl_last_error(c)); exit(2); }
}

typedef int (*Prepare)(rgbl_ctx*);

/* `prepare` + process on a fresh context; then for k = 1, 2, ... a fresh context whose k-th allocation fails inside `prepare`: until k
 * passes the number of allocations it makes, RGBL_E_CUDA, then a retry on the same context whose processed outputs are the first's.
 * Frame construction is slow under emulation, so only the retries are processed. */
static void check_path(const char* name, Prepare prepare, int png) {
    Bytes want = {NULL, 0};
    rgbl_ctx* c = new_ctx();
    if (png) prime_png(c);
    int rc = prepare(c);
    if (!rc) rc = process_and_put(c, &want);
    CHECK(rc == RGBL_OK, "%s: %d (%s)", name, rc, rgbl_last_error(c));
    rgbl_destroy(c);
    for (int k = 1;; ++k) {
        c = new_ctx();
        if (png) prime_png(c);
        Bytes got = {NULL, 0};
        emu_fail_allocation(k);
        rc = prepare(c);
        const int fired = emu_fail_allocation(-1) == -1;
        if (!fired) {
            CHECK(rc == RGBL_OK, "%s: %d (%s)", name, rc, rgbl_last_error(c));
            rgbl_destroy(c);
            printf("%s: %d allocations\n", name, k - 1);
            break;
        }
        CHECK(rc == RGBL_E_CUDA, "%s, allocation %d failed: returned %d", name, k, rc);
        CHECK(rgbl_last_error(c)[0] != 0, "%s, allocation %d failed: no message", name, k);
        rc = prepare(c);
        if (!rc) rc = process_and_put(c, &got);
        CHECK(rc == RGBL_OK, "%s, retry after allocation %d failed: %d (%s)", name, k, rc, rgbl_last_error(c));
        CHECK(got.n == want.n && (want.n == 0 || memcmp(got.p, want.p, want.n) == 0), "%s, retry after allocation %d failed: outputs differ", name, k);
        rgbl_destroy(c); free(got.p);
    }
    free(want.p);
}

int main(void) {
    make_inputs();
    check_path("rectified stereo from arrays", prepare_arrays, 0);
    check_path("rectified stereo from PNG bytes", prepare_png, 1);
    free(g_png[0]); free(g_png[1]);
    printf("%d failed checks\n", g_failures);
    return g_failures ? 1 : 0;
}
