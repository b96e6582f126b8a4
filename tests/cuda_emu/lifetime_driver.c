/* TEST INFRASTRUCTURE: resource lifetime of the emulated library (tests/test_ctx_lifetime.py builds both with -fsanitize=address).
 * Creates and destroys contexts and runs every lazily allocating entry point.  For rgbl_create and the PNG, RGB-D, stage, tracking,
 * BoW and mapping paths it fails the k-th allocation for each k (emu_fail_allocation, cuda_runtime.h in this directory) and checks
 * that the failed call reports RGBL_E_CUDA and that a retry on the same context succeeds with the outputs of a fresh context.
 * LeakSanitizer checks at exit that nothing leaks.  PoseOptimization and the tracking chain are not emulated, so nothing here
 * reaches them.  Frame construction is slow under emulation: the RGB-D path is the one that runs it.
 * Exit 0: every check passed.                                                                                                   */
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <zlib.h>

#include "rgbl_b200.h"

int emu_fail_allocation(int nth);

enum { W = 160, H = 120, NF = 2, NPTS = 2000 };

static int g_failures = 0;
#define CHECK(cond, ...) do { if (!(cond)) { fprintf(stderr, "FAIL %s:%d: ", __FILE__, __LINE__); fprintf(stderr, __VA_ARGS__); fputc('\n', stderr); ++g_failures; } } while (0)

static rgbl_config config(int max_points) {
    rgbl_config cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.width = W; cfg.height = H; cfg.max_batch = NF; cfg.max_points = max_points;
    cfg.orb.nfeatures = 200; cfg.orb.scale_factor = 1.2f; cfg.orb.nlevels = 4; cfg.orb.ini_th_fast = 20; cfg.orb.min_th_fast = 7;
    return cfg;
}

static rgbl_ctx* new_ctx(void) {
    rgbl_config cfg = config(NPTS);
    rgbl_ctx* c = NULL;
    const int rc = rgbl_create(&cfg, &c);
    if (rc) { fprintf(stderr, "rgbl_create: %d (%s)\n", rc, rgbl_last_error(NULL)); exit(2); }
    rgbl_set_host_quadtree(c, 1);          /* the quicker of the two under emulation; it allocates nothing */
    return c;
}

/* ---- inputs: textured images, planar clouds, 16-bit depth, and both as PNG files (filter type 0) ---- */
static uint8_t g_gray[NF][W * H];
static uint16_t g_depth[NF][W * H];
static float g_pts[NF][4 * NPTS], g_xyzr[NF][4 * NPTS];
static uint8_t* g_png[NF]; static size_t g_png_n[NF];
static uint8_t* g_png16[NF]; static size_t g_png16_n[NF];

static size_t put_chunk(uint8_t* out, const char* type, const uint8_t* data, uint32_t len) {
    out[0] = len >> 24; out[1] = len >> 16; out[2] = len >> 8; out[3] = len;
    memcpy(out + 4, type, 4);
    if (len) memcpy(out + 8, data, len);
    const uint32_t crc = (uint32_t)crc32(crc32(0L, Z_NULL, 0), out + 4, len + 4);
    uint8_t* t = out + 8 + len;
    t[0] = crc >> 24; t[1] = crc >> 16; t[2] = crc >> 8; t[3] = crc;
    return 12 + (size_t)len;
}

static uint8_t* encode_png(const uint8_t* samples, int bytes_per_px, size_t* n_out) {
    const size_t row = (size_t)W * bytes_per_px + 1, raw_n = row * H;
    uint8_t* raw = (uint8_t*)calloc(raw_n, 1);
    for (int y = 0; y < H; ++y) memcpy(raw + y * row + 1, samples + (size_t)y * W * bytes_per_px, (size_t)W * bytes_per_px);
    uLongf z_n = compressBound(raw_n);
    uint8_t* z = (uint8_t*)malloc(z_n);
    compress(z, &z_n, raw, raw_n);
    uint8_t* png = (uint8_t*)malloc(8 + 25 + 12 + z_n + 12);
    static const uint8_t sig[8] = {137, 'P', 'N', 'G', 13, 10, 26, 10};
    const uint8_t ihdr[13] = {0, 0, W >> 8, W & 255, 0, 0, H >> 8, H & 255, (uint8_t)(bytes_per_px == 2 ? 16 : 8), 0, 0, 0, 0};
    size_t n = 8;
    memcpy(png, sig, 8);
    n += put_chunk(png + n, "IHDR", ihdr, 13);
    n += put_chunk(png + n, "IDAT", z, (uint32_t)z_n);
    n += put_chunk(png + n, "IEND", NULL, 0);
    free(raw); free(z);
    *n_out = n;
    return png;
}

static void make_inputs(void) {
    for (int f = 0; f < NF; ++f) {
        uint8_t be16[W * H * 2];
        for (int y = 0; y < H; ++y)
            for (int x = 0; x < W; ++x) {
                const int u = x + 3 * f;
                g_gray[f][y * W + x] = (uint8_t)((((u / 12) ^ (y / 12)) & 1) ? 200 - (u % 12) * 9 : 40 + (y % 12) * 7);
                const uint16_t d = (uint16_t)(2000 + 7 * x + 5 * y + 300 * f);
                g_depth[f][y * W + x] = (x % 17 == 3) ? 0 : d;          /* a few holes */
                be16[2 * (y * W + x)] = d >> 8; be16[2 * (y * W + x) + 1] = d & 255;
            }
        for (int i = 0; i < NPTS; ++i) {
            const float px = -4.f + 8.f * (float)(i % 50) / 50.f, py = -3.f + 6.f * (float)(i / 50) / 40.f, pz = 10.f + 0.1f * f;
            g_pts[f][i] = px; g_pts[f][NPTS + i] = py; g_pts[f][2 * NPTS + i] = pz; g_pts[f][3 * NPTS + i] = 1.f;
            g_xyzr[f][4 * i] = px; g_xyzr[f][4 * i + 1] = py; g_xyzr[f][4 * i + 2] = pz; g_xyzr[f][4 * i + 3] = 0.5f;
        }
        g_png[f] = encode_png(g_gray[f], 1, &g_png_n[f]);
        g_png16[f] = encode_png(be16, 2, &g_png16_n[f]);
    }
}

/* ---- the entry points under test: each runs one lazily allocating call (+ what makes its result visible) into `out` ---- */
typedef struct { uint8_t* p; size_t n; } Bytes;

static void put(Bytes* o, const void* p, size_t n) { o->p = (uint8_t*)realloc(o->p, o->n + n); memcpy(o->p + o->n, p, n); o->n += n; }

/* the frame-construction outputs of the last process call */
static int put_frames(rgbl_ctx* c, Bytes* o) {
    const int cap = rgbl_keypoint_capacity(c);
    rgbl_keypoint* k = (rgbl_keypoint*)calloc((size_t)NF * cap, sizeof(rgbl_keypoint));
    uint8_t* d = (uint8_t*)calloc((size_t)NF * cap, 32);
    float* dep = (float*)calloc((size_t)NF * cap, sizeof(float)); float* ur = (float*)calloc((size_t)NF * cap, sizeof(float));
    int n[NF] = {0};
    const int rc = rgbl_resident_download(c, k, d, dep, ur, cap, n);
    if (!rc) {
        put(o, n, sizeof(n));
        for (int f = 0; f < NF; ++f) {
            put(o, k + (size_t)f * cap, n[f] * sizeof(rgbl_keypoint)); put(o, d + (size_t)f * cap * 32, (size_t)n[f] * 32);
            put(o, dep + (size_t)f * cap, n[f] * sizeof(float)); put(o, ur + (size_t)f * cap, n[f] * sizeof(float));
        }
    }
    free(k); free(d); free(dep); free(ur);
    return rc;
}

static const uint8_t* gray_ptrs[NF] = {g_gray[0], g_gray[1]};
static const uint16_t* depth_ptrs[NF] = {g_depth[0], g_depth[1]};
static const float* pts_ptrs[NF] = {g_pts[0], g_pts[1]};
static const float* xyzr_ptrs[NF] = {g_xyzr[0], g_xyzr[1]};
static const int n_pts[NF] = {NPTS, NPTS - 100};

/* uploads whose frames only a frame construction would show (slow under emulation): the call's status is what is checked */
static int run_kitti_bin(rgbl_ctx* c, Bytes* o) {
    (void)o;
    return rgbl_resident_upload_kitti(c, NF, gray_ptrs, W, H, W, xyzr_ptrs, n_pts);
}

static int run_kitti_png(rgbl_ctx* c, Bytes* o) {
    (void)o;
    return rgbl_resident_upload_kitti_png(c, NF, (const uint8_t* const*)g_png, g_png_n, 0, xyzr_ptrs, n_pts);
}

static int run_rgbd_png(rgbl_ctx* c, Bytes* o) {
    (void)o;
    return rgbl_resident_upload_rgbd_png(c, NF, (const uint8_t* const*)g_png, g_png_n, 0, (const uint8_t* const*)g_png16, g_png16_n);
}

static int run_decode_gray(rgbl_ctx* c, Bytes* o) {
    static uint8_t out[NF][W * H];
    uint8_t* outs[NF] = {out[0], out[1]};
    const int rc = rgbl_decode_png_gray(c, NF, (const uint8_t* const*)g_png, g_png_n, 0, outs, W);
    if (!rc) put(o, out, sizeof(out));
    return rc;
}

static int run_decode_depth16(rgbl_ctx* c, Bytes* o) {
    static uint16_t out[NF][W * H];
    uint16_t* outs[NF] = {out[0], out[1]};
    const int rc = rgbl_decode_png_depth16(c, NF, (const uint8_t* const*)g_png16, g_png16_n, outs, W);
    if (!rc) put(o, out, sizeof(out));
    return rc;
}

/* RGB-D frame construction with a distorted camera (UndistortKeyPoints): mvKeys, descriptors, depths, mvKeysUn */
static int run_rgbd(rgbl_ctx* c, Bytes* o) {
    const float dist[4] = {-0.25f, 0.08f, 0.001f, -0.002f};
    float bounds[4];
    int rc = rgbl_set_camera_distortion(c, 200.f, 200.f, 80.f, 60.f, dist, 4, bounds);
    if (!rc) rc = rgbl_resident_upload_rgbd(c, NF, gray_ptrs, W, H, W, depth_ptrs, W);
    if (!rc) rc = rgbl_resident_process_rgbd(c, 1.f / 5000.f, 40.f, NULL);
    if (!rc) rc = put_frames(c, o);
    if (rc) return rc;
    const int cap = rgbl_keypoint_capacity(c);
    rgbl_keypoint* k = (rgbl_keypoint*)calloc((size_t)NF * cap, sizeof(rgbl_keypoint));
    int n[NF];
    rc = rgbl_resident_download_keys_un(c, k, cap, n);
    if (!rc) { put(o, bounds, sizeof(bounds)); put(o, k, (size_t)NF * cap * sizeof(rgbl_keypoint)); }
    free(k);
    return rc;
}

/* staged slots have no output of their own short of the tracking chain: the call's status is what is checked */
static int run_stage(rgbl_ctx* c, Bytes* o) {
    (void)o;
    return rgbl_resident_stage(c, 1, NF, gray_ptrs, W, H, W, pts_ptrs, n_pts);
}

static int run_stage_rgbd(rgbl_ctx* c, Bytes* o) {
    (void)o;
    return rgbl_resident_stage_rgbd(c, 2, NF, gray_ptrs, W, H, W, depth_ptrs, W);
}

/* Frame::isInFrustum grows the tracking scratch */
static int run_frustum(rgbl_ctx* c, Bytes* o) {
    enum { N = 300 };
    static float xw[3 * N], normal[3 * N], dmin[N], dmax[N], px[N], py[N], pxr[N], td[N], vc[N];
    static uint8_t in_view[N]; static int32_t level[N];
    for (int i = 0; i < N; ++i) {
        xw[3 * i] = -3.f + 0.02f * i; xw[3 * i + 1] = 1.f - 0.007f * i; xw[3 * i + 2] = 8.f + 0.01f * i;
        normal[3 * i] = 0.f; normal[3 * i + 1] = 0.f; normal[3 * i + 2] = -1.f; dmin[i] = 1.f; dmax[i] = 50.f;
    }
    const float scale[4] = {1.f, 1.2f, 1.44f, 1.728f};
    rgbl_frame_view v;
    memset(&v, 0, sizeof(v));
    v.min_x = 0.f; v.max_x = W; v.min_y = 0.f; v.max_y = H; v.n_levels = 4; v.scale_factors = scale;
    v.fx = 200.f; v.fy = 200.f; v.cx = 80.f; v.cy = 60.f; v.bf = 40.f; v.log_scale_factor = logf(1.2f);
    const float R[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}, t[3] = {0, 0, 0}, Ow[3] = {0, 0, 0};
    const int rc = rgbl_is_in_frustum(c, &v, R, t, Ow, N, xw, normal, dmin, dmax, 0.5f, in_view, px, py, pxr, td, level, vc);
    if (!rc) { put(o, in_view, sizeof(in_view)); put(o, px, sizeof(px)); put(o, py, sizeof(py)); put(o, level, sizeof(level)); }
    return rc;
}

/* a one-level DBoW2 vocabulary of 4 words: create, ComputeBoW (grows the BoW scratch), destroy */
static int run_bow(rgbl_ctx* c, Bytes* o) {
    enum { NN = 5, ND = 40 };
    const int32_t child_begin[NN + 1] = {0, 4, 4, 4, 4, 4}, child_index[4] = {1, 2, 3, 4}, word_id[NN] = {-1, 0, 1, 2, 3};
    uint8_t node_desc[NN * 32], desc[ND * 32];
    const double weight[NN] = {0.0, 0.5, 1.0, 1.5, 2.0};
    for (int i = 0; i < NN * 32; ++i) node_desc[i] = (uint8_t)(i * 37 + 11);
    for (int i = 0; i < ND * 32; ++i) desc[i] = (uint8_t)(i * 53 + (i >> 5) * 7);
    rgbl_vocabulary* voc = NULL;
    int rc = rgbl_vocabulary_create(c, NN, child_begin, child_index, node_desc, weight, word_id, 1, 0, 0, &voc);
    if (rc) return rc;
    int32_t bow_word[ND], fv_node[ND], fv_start[ND + 1], fv_feature[ND];
    double bow_value[ND];
    int n_words = 0, n_fv = 0;
    rc = rgbl_compute_bow(c, voc, ND, desc, 0, bow_word, bow_value, &n_words, fv_node, fv_start, fv_feature, &n_fv);
    rgbl_vocabulary_destroy(voc);
    if (!rc) { put(o, &n_words, sizeof(int)); put(o, bow_word, n_words * sizeof(int32_t)); put(o, bow_value, n_words * sizeof(double)); put(o, fv_feature, ND * sizeof(int32_t)); }
    return rc;
}

/* LocalMapping's ComputeDistinctiveDescriptors: the mapping arena */
static int run_distinctive(rgbl_ctx* c, Bytes* o) {
    enum { NP = 30, NO = 4 };
    int32_t obs_start[NP + 1], best[NP];
    uint8_t desc[NP * NO * 32];
    for (int p = 0; p <= NP; ++p) obs_start[p] = p * NO;
    for (int i = 0; i < NP * NO * 32; ++i) desc[i] = (uint8_t)(i * 29 + (i >> 7));
    const int rc = rgbl_distinctive_descriptors(c, NP, obs_start, desc, best);
    if (!rc) put(o, best, sizeof(best));
    return rc;
}

typedef int (*Path)(rgbl_ctx*, Bytes*);

/* `run` on a fresh context; with_failures: then for k = 1, 2, ... a fresh context whose k-th allocation fails inside `run`.  Until k
 * passes the number of allocations `run` makes: RGBL_E_CUDA, then a retry on the same context that succeeds with the outputs of
 * the first context. */
static void check_path(const char* name, Path run, int with_failures) {
    Bytes want = {NULL, 0};
    rgbl_ctx* c = new_ctx();
    int rc = run(c, &want);
    CHECK(rc == RGBL_OK, "%s: %d (%s)", name, rc, rgbl_last_error(c));
    rgbl_destroy(c);
    for (int k = 1; with_failures; ++k) {
        c = new_ctx();
        Bytes got = {NULL, 0}, discard = {NULL, 0};
        emu_fail_allocation(k);
        rc = run(c, &discard);
        const int fired = emu_fail_allocation(-1) == -1;
        if (!fired) {                  /* the call made fewer than k allocations */
            CHECK(rc == RGBL_OK, "%s: %d (%s)", name, rc, rgbl_last_error(c));
            rgbl_destroy(c); free(discard.p);
            printf("%s: %d allocations\n", name, k - 1);
            break;
        }
        CHECK(rc == RGBL_E_CUDA, "%s, allocation %d failed: returned %d", name, k, rc);
        CHECK(rgbl_last_error(c)[0] != 0, "%s, allocation %d failed: no message", name, k);
        rc = run(c, &got);
        CHECK(rc == RGBL_OK, "%s, retry after allocation %d failed: %d (%s)", name, k, rc, rgbl_last_error(c));
        CHECK(got.n == want.n && (want.n == 0 || memcmp(got.p, want.p, want.n) == 0), "%s, retry after allocation %d failed: outputs differ", name, k);
        rgbl_destroy(c); free(got.p); free(discard.p);
    }
    free(want.p);
}

int main(void) {
    make_inputs();
    rgbl_config cfg = config(NPTS);
    rgbl_ctx* c = NULL;
    /* create / destroy, max_points = 0, an invalid configuration, destroy(NULL) */
    CHECK(rgbl_create(&cfg, &c) == RGBL_OK, "create");
    rgbl_destroy(c);
    cfg = config(0);
    c = NULL;
    CHECK(rgbl_create(&cfg, &c) == RGBL_OK, "create with max_points = 0");
    rgbl_destroy(c);
    cfg = config(NPTS);
    cfg.width = 0;
    c = NULL;
    CHECK(rgbl_create(&cfg, &c) == RGBL_E_INVALID && c == NULL, "invalid configuration");
    rgbl_destroy(NULL);
    /* every allocation of rgbl_create in turn */
    cfg = config(NPTS);
    for (int k = 1;; ++k) {
        c = NULL;
        emu_fail_allocation(k);
        const int rc = rgbl_create(&cfg, &c);
        const int fired = emu_fail_allocation(-1) == -1;
        if (!fired) { CHECK(rc == RGBL_OK, "create: %d", rc); rgbl_destroy(c); printf("rgbl_create: %d allocations\n", k - 1); break; }
        CHECK(rc == RGBL_E_CUDA && c == NULL, "create, allocation %d failed: returned %d", k, rc);
        CHECK(rgbl_last_error(NULL)[0] != 0, "create, allocation %d failed: no message", k);
    }
    /* the PNG staging and the depth planes fail inside the decode calls (the uploads share them), the raw point records once */
    check_path("rgbl_decode_png_gray", run_decode_gray, 1);
    check_path("rgbl_decode_png_depth16", run_decode_depth16, 1);
    check_path("rgbl_resident_upload_rgbd + distorted-camera frame construction", run_rgbd, 1);
    check_path("rgbl_resident_stage", run_stage, 1);
    check_path("rgbl_resident_stage_rgbd", run_stage_rgbd, 1);
    check_path("rgbl_is_in_frustum", run_frustum, 1);
    check_path("rgbl_vocabulary_create + rgbl_compute_bow", run_bow, 1);
    check_path("rgbl_distinctive_descriptors", run_distinctive, 1);
    check_path("rgbl_resident_upload_kitti", run_kitti_bin, 0);
    check_path("rgbl_resident_upload_kitti_png", run_kitti_png, 0);
    check_path("rgbl_resident_upload_rgbd_png", run_rgbd_png, 0);
    for (int f = 0; f < NF; ++f) { free(g_png[f]); free(g_png16[f]); }
    printf("%d failed checks\n", g_failures);
    return g_failures ? 1 : 0;
}
