/*
 * rtx.h -- C ABI of the H100-native (sm_90a) sequential geometric ray-trace engine.
 *
 * This is the drop-in boundary for ONE hot path of quartiq/rayopt: the
 * per-surface  transfer -> intercept -> clip -> refract  loop
 *
 *     GeometricTrace.propagate      rayopt/geometric_trace.py:72-80
 *       System.propagate            rayopt/system.py:459-464
 *         TransformMixin.to_normal  rayopt/elements.py:174 (156-163)
 *         Interface.propagate       rayopt/elements.py:306-315
 *           Spheroid.intercept      rayopt/elements.py:477-501
 *           Interface.intercept     rayopt/elements.py:333-349 (Newton, aspheres)
 *           Element.clip            rayopt/elements.py:206-209
 *           Interface.refract       rayopt/elements.py:351-369
 *           Spheroid.surface_normal rayopt/elements.py:457-475
 *           Spheroid.surface_sag    rayopt/elements.py:440-455
 *         TransformMixin.from_normal rayopt/elements.py:171
 *
 * The reference has no FFI layer (pure numpy); the boundary it would bind is
 * "one call per GeometricTrace.propagate()": a table of per-surface POD
 * records (what System.propagate reads off each Element for one wavelength)
 * plus the launch rays, returning the (S, N, 3) / (S, N) result arrays the
 * reference stores into GeometricTrace.y/u/i/t (geometric_trace.py:80).
 *
 * Plain C, plain pointers and sizes.  No torch types.  Every function returns
 * 0 on success, a NEGATIVE rtx error (RTX_E_*) for argument errors, or a
 * POSITIVE cudaError_t for CUDA failures.  Numerical failure (missed surface,
 * total internal reflection, vignetting, Newton non-convergence) is NOT an
 * error: it is NaN in the data, exactly where the reference puts it
 * (elements.py:208, 347-348, 367, 496).  With RTX_EXACT that holds ray for
 * ray on the decision boundaries too (aperture rim, tangent intercept,
 * critical angle, Newton exits), with the reference's signs of zero and
 * infinities.  The fast mode's NaN mask may differ within a few ulps of a
 * boundary, never at the aperture rim when the intercept is the reference's
 * own (tests/test_gpu_domain_edges.py).  Launch rays are expected to be
 * finite: a NaN or infinite component gives NaN from that surface on where
 * the reference has NaN or an infinity (the mask and counts agree).
 *
 * A context is bound to one GPU and one CUDA stream and is not thread-safe;
 * use one context per GPU (one process per GPU in multi-GPU runs).
 */
#ifndef RTX_H
#define RTX_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RTX_ABI_VERSION 3

/* maximum number of even-asphere coefficients per surface (Spheroid.aspherics,
 * elements.py:422-424).  Longer lists are rejected with RTX_E_UNSUPPORTED. */
#define RTX_MAX_ASPH 10
/* maximum number of surfaces in one trace call (bounded by the shared-memory
 * staging of the surface table) */
#define RTX_MAX_SURFACES 256

/* rtx_surface.flags */
#define RTX_F_ROTATED 1u /* apply rot (TransformMixin.rotated, elements.py:135) */
#define RTX_F_ALT     2u /* Spheroid.alternate_intersection, elements.py:497-498 */

/* dtype */
#define RTX_F64 0
#define RTX_F32 1

/* keep policy */
#define RTX_KEEP_ALL  0 /* store every surface: outputs have S rows   */
#define RTX_KEEP_LAST 1 /* store only the last surface: outputs have 1 row */

/* trace flags */
#define RTX_EXACT      1u /* FP64 only: unfused IEEE arithmetic in numpy's
                             evaluation order (bit-identical to the reference
                             on unrotated analytic surfaces) */
#define RTX_STORE_DIRECT 2u /* debug: force per-thread strided stores instead
                               of the shared-memory staged bulk (TMA) stores */
#define RTX_RPT1       4u /* tuning: one ray per thread  (default: library's choice) */
#define RTX_RPT2       8u /* tuning: two rays per thread.  An explicit RPT is
                             honoured at every N wherever the pitch and the
                             output alignment allow it (ld a multiple of 32*RPT,
                             16-byte aligned outputs, a table that leaves room
                             for the staging buffers); elsewhere the launch
                             steps down as it does for its own choice.  The
                             results never depend on the kernel chosen
                             (rtx_last_launch_config reports it). */
#define RTX_GATHER_XY 16u /* rtx_trace_gather: the intercept buffers dst[k] are
                             (Ntotal, 2) arrays receiving x,y only -- what a spot
                             diagram reads (rayopt/analysis.py:274): 16 instead of
                             24 bytes per ray over NVLink */

/* errors */
#define RTX_OK              0
#define RTX_E_BADARG       -1
#define RTX_E_UNSUPPORTED  -2
#define RTX_E_NOMEM        -3 /* also: a buffer the context keeps across calls could
                                 not grow; the old one is kept and nothing is freed */

/*
 * One traced surface for one wavelength: everything System.propagate
 * (system.py:459-464) and Interface.propagate (elements.py:306-315) read off
 * the Element.  "Derived" members are scalars the reference computes in
 * Python per call; a caller that wants bit-identical results must compute
 * them with the same expressions (rayopt_b200/surface_table.py does);
 * rtx_surface_finalize() fills them the C way.
 */
typedef struct rtx_surface {
    double offset[3]; /* e.offset, subtracted in the incoming frame (system.py:461) */
    double rot[9];    /* e.rot_normal, row-major; to_normal is y @ rot.T,
                         from_normal is y @ rot (elements.py:156-175); used
                         only if RTX_F_ROTATED */
    double c;         /* Spheroid.curvature */
    double k;         /* Spheroid.conic */
    double kc2;       /* derived: (1 + k)*c**2          (elements.py:448,467) */
    double radius2;   /* derived: radius**2, +inf = no aperture (elements.py:207) */
    double mu;        /* 1 (no material), -1 (mirror) or n0/n (elements.py:283-289) */
    double muf;       /* derived: abs(mu)               (elements.py:360) */
    double sgn;       /* derived: sign(mu)              (elements.py:367) */
    double mu2m1;     /* derived: mu**2 - 1             (elements.py:366) */
    double n0;        /* index before the surface: t = s*n0 (elements.py:315) */
    double n;         /* index after the surface (fills GeometricTrace.n) */
    double asph[RTX_MAX_ASPH];  /* Spheroid.aspherics[j] multiplies r^(2(j+1)) */
    double dasph[RTX_MAX_ASPH]; /* derived: 2*(j+1)*asph[j] (elements.py:472) */
    int32_t n_asph;   /* -1: aspherics is None (analytic intercept);
                         >=0: len(aspherics), Newton intercept even if 0
                         (elements.py:478-479) */
    uint32_t flags;   /* RTX_F_* */
} rtx_surface;

typedef struct rtx_ctx rtx_ctx;

/* ---- library ---------------------------------------------------------- */
int rtx_abi_version(void);
/* sizeof(rtx_surface) / sizeof(rtx_aim) / sizeof(rtx_opd) as compiled, for
 * binding-side layout checks */
size_t rtx_sizeof_surface(void);
size_t rtx_sizeof_aim(void);
size_t rtx_sizeof_opd(void);
/* number of CUDA devices visible, or 0 */
int rtx_device_count(void);
/* static string for an rtx (negative) or CUDA (positive) error code */
const char *rtx_strerror(int code);
/* fill the derived members of n records from c,k,mu,asph and `radius` */
int rtx_surface_finalize(rtx_surface *surf, int n, const double *radius);

/* ---- context ---------------------------------------------------------- */
int rtx_init(int device, rtx_ctx **out);
int rtx_free(rtx_ctx *ctx);
int rtx_sync(rtx_ctx *ctx);
/* device properties: SM count, and bytes of free / total HBM */
int rtx_device_info(rtx_ctx *ctx, int *sm_count, size_t *free_bytes,
                    size_t *total_bytes, char *name, int name_len);

/* ---- memory (so that host code needs no other CUDA binding) ----------- */
int rtx_malloc(rtx_ctx *ctx, size_t bytes, void **dptr);
int rtx_free_device(rtx_ctx *ctx, void *dptr);
int rtx_host_alloc(rtx_ctx *ctx, size_t bytes, void **hptr); /* pinned */
/* ctx may be NULL (page-locked memory may outlive the context that made it) */
int rtx_host_free(rtx_ctx *ctx, void *hptr);
/*
 * NUMA placement of the calling thread (one process per GPU): enable = 1 pins
 * the thread to the CPUs of the NUMA node this context's GPU hangs off
 * (/sys/bus/pci/devices/<bus id>/numa_node) and makes that node the preferred
 * one for its allocations, so that page-locked buffers allocated afterwards
 * (rtx_host_alloc, the library's own bounce buffers) are local to the GPU's
 * PCIe root; enable = 0 restores the affinity and policy saved by the last
 * bind.  *node (may be NULL) receives the node, -1 when the platform does not
 * report one (nothing is changed then).
 */
int rtx_numa_bind(rtx_ctx *ctx, int enable, int *node);
/* asynchronous on the context stream; rtx_sync() to complete */
int rtx_memcpy_h2d(rtx_ctx *ctx, void *dst, const void *src, size_t bytes);
int rtx_memcpy_d2h(rtx_ctx *ctx, void *dst, const void *src, size_t bytes);
int rtx_memcpy_d2d(rtx_ctx *ctx, void *dst, const void *src, size_t bytes);
/* strided D2H: `height` rows of `width` bytes */
int rtx_memcpy2d_d2h(rtx_ctx *ctx, void *dst, size_t dpitch, const void *src,
                     size_t spitch, size_t width, size_t height);
int rtx_memset(rtx_ctx *ctx, void *dptr, int value, size_t bytes);

/* ---- timing on the context stream (CUDA events) ----------------------- */
int rtx_timer_start(rtx_ctx *ctx);
int rtx_timer_stop(rtx_ctx *ctx, float *ms); /* synchronises */
/* device time of the most recent trace kernel launch(es) of the last
 * rtx_trace call, measured with events around the launch */
int rtx_last_kernel_ms(rtx_ctx *ctx, float *ms);
/* number of kernels this context has launched so far */
int64_t rtx_launch_count(rtx_ctx *ctx);
/* CTAs the most recent trace kernel launch ran with (a persistent grid: one
 * resident wave, fewer when clusters of CTAs leave SMs unused) */
int rtx_last_launch_ctas(rtx_ctx *ctx, int *ctas);
/* configuration of the most recent trace kernel launch: cfg = {rays per
 * thread, store path (0 per-thread, 1 per-warp bulk, 2 per-CTA bulk), warps
 * per CTA, staging buffers, CTAs per cluster as launched (1 where the
 * clustered kernel fell back to the per-CTA one)}.  All zero before the first
 * launch. */
int rtx_last_launch_config(rtx_ctx *ctx, int cfg[5]);

/* ---- the hot path ------------------------------------------------------ */
/*
 * March N rays through S surfaces in one launch.  Replaces the loop
 * GeometricTrace.propagate -> System.propagate (geometric_trace.py:72-80,
 * system.py:459-464).
 *
 *  surf[S]  host pointer, surface records for system[start:stop]
 *  rot0     host pointer to 9 doubles or NULL: rot_normal of system[start-1]
 *           when that element is rotated; the launch rays are mapped with
 *           from_normal (y @ rot0) first (geometric_trace.py:76)
 *  dtype    RTX_F64 / RTX_F32: element type of ALL ray arrays
 *  y0,u0    DEVICE pointers, (N,3) C-contiguous: launch rays in the normal
 *           frame of system[start-1]
 *  clip     0/1: the `clip` argument of propagate (elements.py:309-310)
 *  keep     RTX_KEEP_ALL / RTX_KEEP_LAST
 *  ld       row pitch of the outputs in RAYS (>= N).  Outputs are DEVICE
 *           arrays Y,U,I: (rows, ld, 3), T: (rows, ld); rows = S or 1.
 *           With ld a multiple of 128 rays (64 suffices in FP64) the kernel
 *           uses staged bulk (TMA) stores and writes whole groups of 32 x
 *           rays-per-thread rays: columns N .. up(N, 32 rpt)-1 are padding
 *           and receive unspecified values, and nothing at or after column
 *           up(N, 32 rpt) of a row is written (rpt as rtx_last_launch_config
 *           reports it); a multiple of 32 or 64 selects a kernel with
 *           fewer rays per thread; any other ld takes the per-thread store
 *           path and touches only columns < N.
 *           Y: intercepts, U: excidence, I: incidence directions (unclipped),
 *           T: optical path s*n0 -- all in the surface-normal frame, exactly
 *           the tuple System.propagate yields (system.py:463).
 *           Any of Y,U,I,T may be NULL to skip storing that array.
 */
int rtx_trace(rtx_ctx *ctx, const rtx_surface *surf, int S,
              const double *rot0, int dtype, int64_t N,
              const void *y0, const void *u0, int clip, int keep, int64_t ld,
              void *Y, void *U, void *I, void *T, unsigned flags);

/*
 * Batched bundles (SURVEY 8f-3): nb <= RTX_MAX_BATCH bundles of the SAME lens
 * (S surfaces each) -- typically one per wavelength or field: surf[b] its
 * table, N[b] its rays, y0[b], u0[b], Y[b].. its DEVICE arrays (rows x ld
 * pitch shared; Y, U, I, T may each be NULL as a whole) -- marched by ONE
 * launch: the persistent CTAs walk a launch-wide tile list and re-stage the
 * surface table (TMA) when they cross into the next bundle.  Removes the
 * kernel boundaries between the wavelength traces of one analysis step.
 */
#define RTX_MAX_BATCH 8
int rtx_trace_batch(rtx_ctx *ctx, int nb, const rtx_surface *const *surf, int S,
                    const double *rot0, int dtype, const int64_t *N,
                    const void *const *y0, const void *const *u0, int clip,
                    int keep, int64_t ld, void *const *Y, void *const *U,
                    void *const *I, void *const *T, unsigned flags);

/*
 * The same with HOST buffers in the reference layout, any number of bundles
 * (nb >= 1; per bundle y0,u0 (N[b],3) and Y,U,I (rows,N[b],3), T (rows,N[b])):
 * the front end for callers that issue many SMALL traces of one lens --
 * Analysis loops 3 fields x 3-5 wavelengths x 150-ray bundles
 * (rayopt/analysis.py:226-245, 266-280).  All launch rays go up in ONE H2D
 * from a page-locked bounce buffer, the bundles are marched 8 per launch
 * (rtx_trace_batch), all results come back in ONE D2H, one synchronisation.
 * Bundles too large for the bounce buffer are traced one by one through
 * rtx_trace_host.  Y, U, I, T may each be NULL as a whole.
 */
int rtx_trace_batch_host(rtx_ctx *ctx, int nb, const rtx_surface *const *surf,
                         int S, const double *rot0, int dtype, const int64_t *N,
                         const void *const *y0, const void *const *u0, int clip,
                         int keep, void *const *Y, void *const *U,
                         void *const *I, void *const *T, unsigned flags);

/*
 * Optional warp-ballot vignetting mask for the following rtx_trace /
 * rtx_trace_gather calls on device buffers: dmask (DEVICE, ceil(N/32) words,
 * or NULL to switch it off) receives bit (ray % 32) of word ray / 32 = 1 when
 * the ray leaves the last traced surface with a finite direction -- i.e. it
 * was not clipped (Element.clip, elements.py:206-209) and hit no NaN
 * condition on the way (elements.py:347-348, 367, 496).
 */
int rtx_set_mask_output(rtx_ctx *ctx, uint32_t *dmask);

/*
 * Optional per-ray optical path sum for the following rtx_trace calls on
 * device buffers: dsum (DEVICE, N values of the trace dtype, or NULL = off)
 * receives sum over traced surfaces 0..upto (inclusive; upto < 0: all) of
 * t -- the accumulation GeometricTrace.opd starts from
 * (rayopt/geometric_trace.py:102), without reading the (S,N) array again.
 * The sum is taken left to right over the t values as they are stored (each
 * rounded to the trace dtype), so it is bit-identical to adding the stored
 * T rows 0..upto in order, in every mode and kernel configuration.  Only
 * entries 0..N-1 are written.
 */
int rtx_set_path_sum_output(rtx_ctx *ctx, void *dsum, int upto);

/*
 * Same call with HOST buffers in the reference layout: y0,u0 (N,3);
 * Y,U,I (rows,N,3), T (rows,N) C-contiguous (GeometricTrace.y/u/i/t rows
 * start..stop-1).  Synchronous.  Three regimes by size (rays + results):
 *   <= 16 KB  (ray aiming: 1-3 rays, hundreds of calls, rayopt/system.py:
 *             507-555) ZERO-COPY: the kernel reads the rays from and writes
 *             the results to a page-locked bounce buffer over PCIe -- one
 *             launch, one synchronisation;
 *   <= 4 MB   one H2D, one launch, one D2H through the bounce buffer;
 *   larger    rays are processed in ~256 MB chunks; H2D, kernel and D2H of
 *             consecutive chunks overlap on two streams.  Host buffers from
 *             rtx_host_alloc (pinned) copy at full PCIe rate; pageable ones
 *             work too.
 * The mask / path-sum side outputs do not apply to host-buffer calls.
 */
int rtx_trace_host(rtx_ctx *ctx, const rtx_surface *surf, int S,
                   const double *rot0, int dtype, int64_t N,
                   const void *y0, const void *u0, int clip, int keep,
                   void *Y, void *U, void *I, void *T, unsigned flags);

/* ---- fused trace + gather over peer memory (multi-GPU, SURVEY 8e) ------- */
/*
 * Cross-process device memory: export a buffer of this context's GPU as an
 * opaque 64-byte handle (cudaIpcGetMemHandle), open a handle exported by
 * another process of the same node (peer access over NVLink is enabled
 * lazily), close it again.
 */
#define RTX_IPC_HANDLE_BYTES 64
int rtx_ipc_export(rtx_ctx *ctx, void *dptr, unsigned char *handle);
int rtx_ipc_open(rtx_ctx *ctx, const unsigned char *handle, void **dptr);
int rtx_ipc_close(rtx_ctx *ctx, void *dptr);
/*
 * Trace this rank's shard (N rays, DEVICE y0,u0) and store the LAST surface's
 * intercepts straight into `npeers` (<= 8) gather buffers dst[k] -- (Ntotal_pad, 3)
 * arrays of `dtype` that are local or peer-GPU memory (rtx_ipc_open) -- at ray
 * offset dst_offset: the all-gather of GeometricTrace.y[-1] is done by the
 * trace kernel's own TMA bulk stores over NVLink instead of a separate
 * collective.  dst_i (may be NULL) is a second set of npeers buffers that
 * receive the last surface's INCIDENCE directions i[-1] the same way (the
 * through-focus spots of rayopt/analysis.py:274-280 read y[-1] and i[-1]).
 * Bulk stores need 16-byte aligned runs and write whole groups of 32 x
 * rays-per-thread rays: with dst_offset and N multiples of 64 rays (FP64;
 * 128 for the fastest FP32 kernel) exactly rays dst_offset .. dst_offset +
 * N - 1 are written by bulk stores; for any other N or offset the library
 * steps down to a kernel with smaller groups and finally to per-ray stores
 * that touch exactly N rays, so a shard can never spill into its
 * neighbour's range.  Asynchronous on
 * the context stream; after rtx_sync on every rank and a cross-rank barrier
 * all buffers hold the full spot.
 */
int rtx_trace_gather(rtx_ctx *ctx, const rtx_surface *surf, int S,
                     const double *rot0, int dtype, int64_t N, const void *y0,
                     const void *u0, int clip, int npeers, void *const *dst,
                     void *const *dst_i, int64_t dst_offset, unsigned flags);

/* ---- self-test --------------------------------------------------------- */
/*
 * The kernels use their own branch-free FP64 division / sqrt / rsqrt (the
 * library sequences minus the slow-path subroutine).  For n host operand
 * pairs (a, b) writes 6*n doubles to `out` (host): a/b (engine), a/b (IEEE
 * __ddiv_rn), sqrt(a) (engine), sqrt(a) (IEEE), 1/sqrt(a) (engine),
 * 1/sqrt(a) (IEEE).
 */
int rtx_selftest_math(rtx_ctx *ctx, int64_t n, const double *a, const double *b,
                      double *out);
/*
 * The other primitives: for n host operand triples (a, b, c) writes 7*n
 * doubles to `out` (host): a/b and c/b from the shared-reciprocal division of
 * exact-mode refraction, a/b and c/b (IEEE __ddiv_rn), 1/b (the fast Newton
 * step's reciprocal), sqrt(a) and 1/sqrt(a) (the fast Newton sag's pair).
 */
int rtx_selftest_math2(rtx_ctx *ctx, int64_t n, const double *a, const double *b,
                       const double *c, double *out);
/*
 * The exact predicates of rtx_delaunay: for n host point quadruples pts[8i..8i+7]
 * = (a, b, c, d) writes 2*n ints to `out` (host): the sign of orient2d(a, b, c)
 * (> 0: counter-clockwise) and of incircle(a, b, c, d) (> 0: d strictly inside
 * the circle through a, b, c when they are counter-clockwise).  Exact for
 * coordinates in rtx_delaunay's domain.
 */
int rtx_selftest_predicates(rtx_ctx *ctx, int64_t n, const double *pts, int *out);

/* ---- fused last-surface reductions (geometric_trace.py:171-183) ------- */
/*
 * Weighted moments of DEVICE intercepts y (N,3), dtype as given, about
 * `center` (host, 2 doubles, or NULL for the origin); dx = x - center[0]:
 * m[0]=sum w, m[1]=sum w*dx, m[2]=sum w*dy, m[3]=sum w*(dx^2+dy^2),
 * m[4]=count finite, m[5]=count total, m[6]=sum dx, m[7]=sum dy.
 * Rays with non-finite x or y are skipped (counted in m[5] only).
 * w (device, N values of dtype) may be NULL (w = 1).  m: host, 8 doubles.
 * Two calls (moments about 0, then about the mean) give the reference's
 * rms() without moving y to the host; per-rank moments add up
 * (all-reduce of 8 doubles) for ray-sharded multi-GPU runs.
 */
int rtx_moments(rtx_ctx *ctx, int dtype, int64_t N, const void *y,
                const void *w, const double *center, double *m);

/* ---- fused epilogues: the march with no per-surface stores (SURVEY 8f-1, 8f-4) */
/*
 * rms / centroid / refocus moments of surface S-1 in ONE launch from the
 * launch rays (DEVICE y0,u0; surf[S] = system[start:at+1]): the trace kernel
 * keeps the rays in registers, accumulates the moments there and writes 20
 * doubles -- GeometricTrace.rms (rayopt/geometric_trace.py:171-183) and the
 * focus shift of GeometricTrace.refocus (:82-99) of 1e9 rays without storing
 * a single intercept.  About the guess centres center[0..1] (intercept x,y)
 * and center[2..3] (slope i_x/i_z, i_y/i_z) -- e.g. the chief ray's, so that
 * the shift to the true means is cancellation-free (host, 4 doubles or NULL);
 * w: DEVICE weights (N values of dtype) or NULL (= 1).  m (host, 20 doubles):
 *   m[0..7]   as rtx_moments (sum w, sum w dx, sum w dy, sum w (dx^2+dy^2),
 *             #finite, #total, sum dx, sum dy)
 *   m[8..19]  over the rays with a finite slope: #good, sum dy (2), sum du (2),
 *             sum w, sum w dy (2), sum w du (2), sum w dy.du, sum w du.du
 * Per-rank moments add up (one all-reduce of 20 doubles) for ray-sharded runs.
 */
#define RTX_NMOMENTS 20
int rtx_trace_reduce(rtx_ctx *ctx, const rtx_surface *surf, int S,
                     const double *rot0, int dtype, int64_t N, const void *y0,
                     const void *u0, int clip, const void *w,
                     const double *center, double *m, unsigned flags);

/*
 * rtx_trace_reduce for many (surface table, launch bundle) items in ONE
 * launch -- the tolerance analysis of thousands of perturbed lenses.
 *   tables   host, nt*S records: table t is tables[t*S .. t*S+S-1]
 *   rot0     shared by every table (NULL: none)
 *   bundles  b < nb: DEVICE y0[b], u0[b] (N[b],3) of dtype; any number of
 *            items may share one (the rays are read, never copied)
 *   item i   marches bundle item_bundle[i] through table item_table[i] about
 *            the guess centres centers[4i .. 4i+3] (host (nitems,4), or NULL
 *            for 0), as rtx_trace_reduce's `center`
 *   m        host (nitems, RTX_NMOMENTS): row i is item i's 20 moments, as
 *            rtx_trace_reduce defines them with w = NULL (zeros for N = 0);
 *            exactly nitems*20 doubles are written
 * Each ray's state at surface S-1 is the last row rtx_trace stores for the
 * same table, in every mode.  The sums are deterministic: item i's moments
 * are the sum of its own 512-ray tiles in tile order, each tile summed by a
 * warp shuffle tree and then its 8 warps in order (per-tile partials in the
 * context and a second pass, no atomics).  So an item gives the same bits in
 * every call and context, whatever the grid and whatever other items share
 * the launch, in any order.  Error bound against the exact sum:
 * (ceil(N/512) + 64) eps sum|term|.
 * RTX_E_BADARG, before any device work or allocation: NULL ctx, tables, N,
 * y0, u0, item_table, item_bundle or m; nt, nb or nitems < 1; S outside
 * 1..RTX_MAX_SURFACES; a table or bundle index out of range; N[b] < 0; NULL
 * y0[b] or u0[b] with N[b] > 0; a bad dtype.  A record with n_asph >
 * RTX_MAX_ASPH gives RTX_E_UNSUPPORTED, as in every march, and so does
 * RTX_EXACT with RTX_F32.  The device tables, the items and the tile partials
 * are kept in the context: RTX_E_NOMEM before allocating when they do not fit.
 * Synchronous; rtx_last_kernel_ms covers the two kernels.
 */
int rtx_trace_reduce_many(rtx_ctx *ctx, int nt, const rtx_surface *tables, int S,
                          const double *rot0, int dtype, int nb, const int64_t *N,
                          const void *const *y0, const void *const *u0,
                          int64_t nitems, const int32_t *item_table,
                          const int32_t *item_bundle, const double *centers,
                          int clip, double *m, unsigned flags);

/*
 * The per-ray part of GeometricTrace.opd (rayopt/geometric_trace.py:101-131)
 * as the epilogue of the march to surface `after` (surf[S] = system[1:after+1]):
 *   A = sum_s t[s] - tj*n0 + ti*n_after,   P = y' + ti*u' - (0, 0, radius)
 * with tj = u0_ref.(y0_ref - y0) for an object at infinity (`infinite`, :104-109),
 * y' = y[after] @ M + d, u' = u[after] @ M the change to the image frame
 * (:116-120; M = ea.rot_normal @ ei.rot_normal.T, d = (origins[after] -
 * origins[image]) @ ei.rot_normal.T - y[image, ref]) and ti the intercept with
 * the reference sphere Spheroid(curvature=1/radius) after y'_z += radius
 * (:123-124).  The caller finishes with the reference ray:
 *   t = -(A - A[ref])/(l/scale),  py = P - P[ref].
 * A: DEVICE (N,), P: DEVICE (N,3) of dtype.  Asynchronous.
 */
typedef struct rtx_opd {
    double y0_ref[3], u0_ref[3]; /* launch ray `ref` (row 0 of the trace) */
    double n0, n_after;
    double M[9], d[3];
    double radius;
    int32_t infinite;
    int32_t reserved;
} rtx_opd;
int rtx_trace_opd(rtx_ctx *ctx, const rtx_surface *surf, int S,
                  const double *rot0, int dtype, int64_t N, const void *y0,
                  const void *u0, int clip, const rtx_opd *opd, void *A,
                  void *P, unsigned flags);

/*
 * Through-focus spot images (Analysis.spots, rayopt/analysis.py:250-283) as
 * integer histograms.  For each ray and plane k < planes, in FP64 with every
 * operation separately rounded (FP32 rays are widened first):
 *   d = y_xy - c,  u = i_xy / i_z,  q = (d + z[k] u) - o[k]
 *   radial = 0: (q_x, q_y) binned as np.histogram2d(qx, qy, (nx, ny), range)
 *   radial = 1: r = sqrt(q_x^2 + q_y^2) binned as np.histogram(r, nx, range[0])
 * Binning: edges e_j = j*step + lo, step = (hi - lo)/n, e_n = hi
 * (np.linspace); bin = searchsorted(e, x, "right") - 1 with x == hi in the
 * last bin; points outside [lo, hi], NaN and +-inf are not counted.
 *
 * counts: DEVICE uint64 (planes, nx, ny) (radial: (planes, nx)), ADDED to (the
 * caller zeroes it), or NULL.  tally: host (planes, 2) uint64 = rays binned,
 * rays with a non-finite q.  extent: host (planes, 3) doubles = max |q_x|,
 * max |q_y|, max r over the rays with a finite q (0 when there is none).
 * Counts, tallies and extents are exact, so they are the same in every call,
 * context and chunking of a bundle, and chunks add up.
 *
 * RTX_E_BADARG, before any device work, for planes outside 1..16, nx or ny
 * < 1, ny != 1 in radial mode, planes*nx*ny >= 2^31, a non-finite range end,
 * lo >= hi, a step (hi - lo)/n that is not a normal number, a non-finite z
 * or o, or counts and extent both NULL.  N = 0 adds nothing.
 */
#define RTX_SPOT_MAX_PLANES 16
typedef struct rtx_spot {
    int32_t planes, radial;           /* K in 1..16; 0: 2-D image, 1: radial */
    int64_t nx, ny;                   /* bins (radial: nx; ny must be 1) */
    double range[2][2];               /* [[x_lo, x_hi], [y_lo, y_hi]]; radial: range[0] */
    double c[2];                      /* subtracted from y_xy first (the chief ray's) */
    double z[RTX_SPOT_MAX_PLANES];    /* defocus distances */
    double o[RTX_SPOT_MAX_PLANES][2]; /* per-plane offsets subtracted last */
} rtx_spot;
size_t rtx_sizeof_spot(void);
/* the march to surface S-1 (as rtx_trace_reduce) with the binning as its
 * epilogue: nothing per ray is stored.  Synchronous. */
int rtx_trace_spot(rtx_ctx *ctx, const rtx_surface *surf, int S,
                   const double *rot0, int dtype, int64_t N, const void *y0,
                   const void *u0, int clip, const rtx_spot *spot,
                   uint64_t *counts, uint64_t *tally, double *extent,
                   unsigned flags);
/* the same binning of stored rows: y, inc DEVICE (N,3) of dtype (a trace's
 * y[at] and i[at]).  Synchronous. */
int rtx_spot_rows(rtx_ctx *ctx, int dtype, int64_t N, const void *y,
                  const void *inc, const rtx_spot *spot, uint64_t *counts,
                  uint64_t *tally, double *extent);

/*
 * Geometric OTF through focus: the Fourier transform of the spot diagram of
 * stored rows y, inc (DEVICE (N,3) of dtype; a trace's y[at] and i[at]).
 * Each ray's point at plane k is rtx_spot_rows' (FP64, every operation
 * separately rounded, FP32 rows widened first):
 *   d = y_xy - c,  u = i_xy / i_z,  q_k = (d + z[k] u) - o[k]
 * A ray counts at plane k when both components of q_k are finite.  With
 * nu_j = j*dnu (one rounded product), j < F, and a in {x, y}:
 *   S[k,a,j] = sum over the counted rays of exp(-2 pi i nu_j q_k[a])
 *   count[k] = number of counted rays;  OTF = S / count,  MTF = |OTF|
 * S[k,a,0] is exactly count[k].  sums: host (K, 2, F, 2) doubles (re, im),
 * count: host (K) int64; exactly K*2*F*2 doubles and K counts are written,
 * zeros for N = 0.  Synchronous; rtx_last_kernel_ms covers both kernels.
 *
 * Deterministic: the rays are cut into slots of RTX_OTF_SLOT; each of the
 * slot's 8 runs of RTX_OTF_SLOT/8 rays is summed in ray order, the runs in
 * order, then the slot sums in slot order (a second kernel; no atomics).  The
 * bits depend only on the rows and the spec, not on the grid, context or call.
 * Each term starts from one sincospi for the first of a block of
 * RTX_OTF_BLOCK frequencies and steps by the phasor exp(-2 pi i dnu q).
 *
 * Error bound, eps = 2^-52, Phi = max |nu_j q_k[a]| over the counted rays:
 *   |S - S_exact| <= (D + 13 Phi + 5 RTX_OTF_BLOCK) eps count[k]
 *   D = RTX_OTF_SLOT/8 + 8 + ceil(N / RTX_OTF_SLOT)   (the summation depth)
 * per component.  13 Phi bounds the rounding of nu_j q and of the step
 * phase, the recurrence's drift from fl(j dnu) and the step's error carried
 * through RTX_OTF_BLOCK - 1 products (4 pi Phi); 5 RTX_OTF_BLOCK the 2 ulp of
 * each sincospi component and the rounding of each complex product.
 *
 * RTX_E_BADARG, before any device work or allocation: NULL ctx, spec, sums or
 * count; NULL y or inc with N > 0; N < 0; a bad dtype; planes outside
 * 1..RTX_OTF_MAX_PLANES, nfreq outside 1..RTX_OTF_MAX_FREQS; a non-finite
 * dnu, c, z or o.  The slot sums are kept in the context
 * (ceil(N/RTX_OTF_SLOT) (K*2*F*2 + K) doubles): RTX_E_NOMEM before
 * allocating when they do not fit.
 */
#define RTX_OTF_MAX_PLANES 16
#define RTX_OTF_MAX_FREQS  256
#define RTX_OTF_SLOT       16384 /* rays per slot of the deterministic sum */
#define RTX_OTF_BLOCK      16    /* frequencies per sincospi */
typedef struct rtx_otf {
    int32_t planes, nfreq;            /* K in 1..16, F in 1..256 */
    double dnu;                       /* nu_j = j*dnu */
    double c[2];                      /* subtracted from y_xy first */
    double z[RTX_OTF_MAX_PLANES];     /* defocus distances */
    double o[RTX_OTF_MAX_PLANES][2];  /* per-plane offsets subtracted last */
} rtx_otf;
size_t rtx_sizeof_otf(void);
int rtx_otf_rows(rtx_ctx *ctx, int dtype, int64_t N, const void *y, const void *inc,
                 const rtx_otf *spec, double *sums, int64_t *count);

/* ---- lens-parameter derivatives of the image point ---------------------- */
/*
 * The image point q = (y_x, y_y) of every ray at surface S-1 and its exact
 * derivatives J = dq/dp with respect to P lens parameters, from one march
 * (forward-mode tangents; FP64 only).
 *
 * A parameter p is a list of moves: moves[m] for m in param_first[p] ..
 * param_first[p+1]-1 is the derivative of the record surf[move_row[m]] with
 * respect to p (every member the kernel reads: offset, rot, c, k, kc2, mu,
 * muf, mu2m1, n0, asph, dasph; flags, n_asph, sgn and radius2 are ignored),
 * so a parameter may move several rows (a pickup, a refractive index).
 *
 *  surf, S, rot0, y0, u0, N, clip  as rtx_trace (dtype must be RTX_F64)
 *  P           1 .. RTX_MAX_PARAMS
 *  param_first host, P+1 int32 offsets: param_first[0] = 0, strictly rising
 *  move_row    host, param_first[P] rows in 0 .. S-1
 *  moves       host, param_first[P] records
 *  q           DEVICE (N, 2) doubles
 *  J           DEVICE (P, 2, ld) doubles: J[(2p + a) ld + k] = dq_a/dp of ray
 *              k; ld >= N; columns N .. ld-1 are not written
 *
 * q equals the last row rtx_trace stores for the same arguments (its x, y),
 * bit for bit, in each mode (RTX_EXACT or not).  J is the derivative of that
 * march with the intercept taken as the EXACT root of the surface (implicit
 * differentiation at the primal hit point, not of Newton's iterate): there is
 * no derivative through ray aiming, clipping decisions, the choice of an
 * intercept branch or the Newton stopping rule.  The tangents are FP64 with
 * fused multiply-adds in both modes.  A ray whose q is NaN has NaN
 * derivatives; a finite q may have a non-finite derivative where the ray
 * grazes a surface (rtx_jacobian_sums counts those).
 *
 * RTX_E_BADARG, before any device work or allocation: NULL ctx, surf, y0,
 * u0, param_first, move_row, moves, q or J; S outside 1..RTX_MAX_SURFACES;
 * N < 0; P outside 1..RTX_MAX_PARAMS; param_first[0] != 0 or a parameter
 * without moves (param_first not strictly rising); a move_row outside
 * 0..S-1; a move with a non-zero mu, muf or mu2m1 on a row whose mu is 1
 * (that row does not refract, so the march has no derivative with respect
 * to them); ld < N; a dtype other than RTX_F64.  A record of surf with n_asph >
 * RTX_MAX_ASPH gives RTX_E_UNSUPPORTED, as in every march.  The tangent
 * records are kept in the context.  Asynchronous; rtx_last_kernel_ms covers
 * the kernel.
 */
#define RTX_MAX_PARAMS 64
int rtx_trace_jacobian(rtx_ctx *ctx, const rtx_surface *surf, int S,
                       const double *rot0, int dtype, int64_t N, const void *y0,
                       const void *u0, int clip, int P, const int32_t *param_first,
                       const int32_t *move_row, const rtx_surface *moves, void *q,
                       void *J, int64_t ld, unsigned flags);

/*
 * Gauss-Newton sums of rtx_trace_jacobian's q (DEVICE (N, 2)) and J (DEVICE
 * (P, 2, ld)) about the centre c (host, 2 doubles, or NULL for 0), with
 * d = fl(q - c).  A ray enters iff q and all of its 2P derivatives are
 * finite.  out (host, W = 5 + 3P + P(P+1)/2 doubles), over the rays that
 * enter:
 *   out[0]              n
 *   out[1..2]           sum d_x, sum d_y
 *   out[3]              sum |d|^2
 *   out[4 + 2a + x]     G_a = sum dq/dp_a           (a < P, x the axis)
 *   out[4 + 2P + a]     H_a = sum d . dq/dp_a
 *   out[4 + 3P + ...]   K_ab = sum dq/dp_a . dq/dp_b, a <= b, row-major
 *                       packed upper triangle (P(P+1)/2 values)
 *   out[W - 1]          rays with a finite q and a non-finite derivative
 *                       (they do not enter)
 * Deterministic: each RTX_JAC_SLOT-ray slot is summed in ray order by one
 * thread per output, the slot sums then in slot order (a second kernel; no
 * atomics), so the bits depend only on q, J and c.  Error bound against the
 * exact sum of the same terms, eps = 2^-52:
 *   |out - exact| <= (2 RTX_JAC_SLOT + ceil(N / RTX_JAC_SLOT)) eps sum|term|
 * where the terms are the single products of d and J entries each output
 * adds (two per ray for sum |d|^2, H and K).  Counts are exact.
 * RTX_E_BADARG, before any device work or allocation: NULL ctx or out; NULL
 * q or J with N > 0; N < 0; P outside 1..RTX_MAX_PARAMS; ld < N.  The slot
 * sums are kept in the context: RTX_E_NOMEM before allocating when they do
 * not fit.  Synchronous; rtx_last_kernel_ms covers both kernels.
 */
#define RTX_JAC_SLOT 16384
int rtx_jacobian_sums(rtx_ctx *ctx, int64_t N, int P, const void *q, const void *J,
                      int64_t ld, const double *center, double *out);

/* ---- lens-parameter derivatives of the wavefront ------------------------ */
/*
 * rtx_trace_opd's optical path A of every ray and its exact derivatives
 * dA = dA/dp with respect to P lens parameters, from one march (forward-mode
 * tangents; FP64 only).  surf, S, rot0, y0, u0, N, clip and opd are
 * rtx_trace_opd's (surf = system[1:after+1]); P, param_first, move_row and
 * moves are rtx_trace_jacobian's, on those rows.  The epilogue's reference
 * sphere moves with the lens through
 *  dopd   host, (P, 4) doubles: per parameter d(opd->d)[0..2], d(opd->n_after)
 * (moves of the image surface reach A only through them); its radius and the
 * frame change M are held fixed.
 *  A      DEVICE (N,) doubles
 *  dA     DEVICE (P, ld) doubles: dA[p ld + k] = dA_k/dp; ld >= N; columns
 *         N .. ld-1 are not written
 *
 * A equals rtx_trace_opd's A for the same arguments, bit for bit, in each
 * mode (RTX_EXACT or not).  dA is the derivative of that march and
 * epilogue: the path's tangent adds n0 ds + s dn0 at every surface (s the
 * surface's intercept distance, n0 its index), the sphere intercept ti is
 * differentiated implicitly at its root as the surfaces' intercepts are
 * (rtx_trace_jacobian), and dA = dT + n_after dti + ti d(n_after).  The
 * input-plane term of an object at infinity has no derivative (the launch
 * rays are fixed).  The tangents are FP64 with fused multiply-adds in both
 * modes.  A ray whose A is NaN has NaN derivatives; a finite A may have a
 * non-finite derivative where the ray grazes a surface (rtx_wavefront_sums
 * counts those).
 *
 * RTX_E_BADARG, before any device work or allocation: every refusal of
 * rtx_trace_jacobian (with A, dA in place of q, J); a NULL opd, or a NULL
 * dopd with P > 0; an opd radius that is 0 or not finite; a non-finite dopd
 * entry; a move with a non-zero rot on row S-1 (M is held fixed).  A record
 * of surf with n_asph > RTX_MAX_ASPH gives RTX_E_UNSUPPORTED.  The tangent
 * records and dopd are kept in the context.  Asynchronous;
 * rtx_last_kernel_ms covers the kernel.
 */
int rtx_trace_opd_jacobian(rtx_ctx *ctx, const rtx_surface *surf, int S,
                           const double *rot0, int dtype, int64_t N, const void *y0,
                           const void *u0, int clip, const rtx_opd *opd, int P,
                           const int32_t *param_first, const int32_t *move_row,
                           const rtx_surface *moves, const double *dopd, void *A,
                           void *dA, int64_t ld, unsigned flags);

/*
 * Gauss-Newton sums of rtx_trace_opd_jacobian's A (DEVICE (N,)) and dA
 * (DEVICE (P, ld)) about the guess piston a0, with d = fl(A - a0).  A ray
 * enters iff A and all of its P derivatives are finite.  P = 0 is allowed
 * (dA is then not read and may be NULL): n, sum d and sum d^2 of any A.
 * out (host, W = 4 + 2P + P(P+1)/2 doubles), over the rays that enter:
 *   out[0]              n
 *   out[1]              sum d
 *   out[2]              sum d^2
 *   out[3 + a]          G_a = sum dA/dp_a           (a < P)
 *   out[3 + P + a]      H_a = sum d dA/dp_a
 *   out[3 + 2P + ...]   K_ab = sum dA/dp_a dA/dp_b, a <= b, row-major
 *                       packed upper triangle (P(P+1)/2 values)
 *   out[W - 1]          rays with a finite A and a non-finite derivative
 *                       (they do not enter)
 * Deterministic, in the same slots and order as rtx_jacobian_sums, and
 * within the same bound:
 *   |out - exact| <= (2 RTX_JAC_SLOT + ceil(N / RTX_JAC_SLOT)) eps sum|term|
 * where the terms are the single products of d and dA entries each output
 * adds.  Counts are exact.  RTX_E_BADARG, before any device work or
 * allocation: NULL ctx or out; NULL A with N > 0, or NULL dA with N > 0 and
 * P > 0; N < 0; P outside 0..RTX_MAX_PARAMS; ld < N.  The slot sums are kept
 * in the context: RTX_E_NOMEM before allocating when they do not fit.
 * Synchronous; rtx_last_kernel_ms covers both kernels.
 */
int rtx_wavefront_sums(rtx_ctx *ctx, int64_t N, int P, const void *A, const void *dA,
                       int64_t ld, double a0, double *out);

/* ---- lens-parameter derivatives of the geometric OTF -------------------- */
/*
 * The geometric OTF sums of image points q and their derivatives with
 * respect to P lens parameters, at F arbitrary frequencies:
 *  q       DEVICE, qstride doubles per ray: 2 for rtx_trace_jacobian's q,
 *          3 for a keep-LAST row of rtx_trace (its y; only x, y are read)
 *  J       DEVICE (P, 2, ld), rtx_trace_jacobian's; not read when P = 0
 *  center  host, 2 doubles, or NULL for 0
 *  freqs   host, nfreq doubles nu_j (cycles per length unit), any order
 * With d = fl(q - c), a ray enters iff q and all 2P of its derivatives are
 * finite.  Over the rays that enter, for axis a in {x, y}:
 *   S[a, j]     = sum exp(-2 pi i nu_j d_a)
 *   dS[p, a, j] = sum -2 pi i nu_j J[p, a] exp(-2 pi i nu_j d_a)
 * dS is the derivative of S with c held fixed.  Moving c multiplies S by a
 * phase, so |S|, the MTF |S|/n and a polychromatic MTF of wavelengths that
 * share one centre do not depend on it: d|S|/dp = Re(conj(S) dS/dp)/|S|.
 * out (host, W = RTX_OTF_JAC_WIDTH(P, F) doubles; complex values as (re, im)):
 *   out[0]                                 n, the rays that enter
 *   out[1 + 2 (a F + j) + {0, 1}]          S[a, j]
 *   out[1 + 4F + 2 ((2p + a) F + j) + {0, 1}]   dS[p, a, j]
 *   out[W - 1]                             bad: rays with a finite q and a
 *                                          non-finite derivative (they do
 *                                          not enter)
 * zeros for N = 0.  Per ray and (a, j) one sincospi(2 fl(nu_j d_a)); the
 * kernel sums S and T = sum J e (e = exp(-2 pi i nu d)) and the host forms
 * dS = -2 pi i nu T from fl(fl(2 pi) nu) T.
 *
 * Deterministic: the rays are cut into slots of RTX_OTF_JAC_SLOT; each of
 * the slot's 8 runs of RTX_OTF_JAC_SLOT/8 rays is summed in ray order, the
 * runs in order, then the slot sums in slot order (a second kernel; no
 * atomics).  The bits depend only on q, J, c and the frequencies.  S depends
 * on P only through which rays enter: with bad = 0 it is the same, bit for
 * bit, as the P = 0 call's on the same points (either qstride).
 *
 * Error bound against the exact sums of the same d, eps = 2^-52,
 * Phi = max |nu_j d_a| over the rays that enter:
 *   S:   |S - S_exact|   <= (D + 4 Phi + 3) eps n          per component
 *   dS:  |dS - dS_exact| <= (D + 4 Phi + 5) eps sum_k 2 pi |nu_j J_k[p, a]|
 *   D = RTX_OTF_JAC_SLOT/8 + 8 + ceil(N / RTX_OTF_JAC_SLOT)   (summation depth)
 * D bounds the additions (each component of each partial sum is at most
 * the sum of the terms' magnitudes); 4 Phi the rounding of nu d, which moves
 * the phase by at most pi Phi eps; 3 the 2 ulp of each sincospi component
 * and one more; for dS 2 more for the FMA's product and the host's scaling
 * by fl(fl(2 pi) nu).  Counts are exact.
 *
 * RTX_E_BADARG, before any device work or allocation: NULL ctx or out; NULL
 * q with N > 0, or NULL J with N > 0 and P > 0; N < 0; P outside
 * 0..RTX_MAX_PARAMS; qstride not 2 or 3; ld < N with P > 0; nfreq outside
 * 1..RTX_OTF_MAX_FREQS; a NULL freqs; a non-finite frequency or centre.
 * The slot sums and a ray mask are kept in the context: RTX_E_NOMEM before
 * allocating when they do not fit.  Synchronous; rtx_last_kernel_ms covers
 * the three kernels.
 */
#define RTX_OTF_JAC_SLOT 4096 /* rays per slot of the deterministic sum */
#define RTX_OTF_JAC_WIDTH(P, F) (2 + 4 * (F) + 4 * (P) * (F))
int rtx_otf_jacobian_sums(rtx_ctx *ctx, int64_t N, int P, const void *q, int qstride,
                          const void *J, int64_t ld, const double *center, int nfreq,
                          const double *freqs, double *out);

/* ---- tolerance analysis on the geometric OTF ----------------------------- */
/*
 * The geometric OTF sums of many (surface table, launch bundle) items in ONE
 * launch -- the MTF of thousands of perturbed lenses.  tables, S, rot0,
 * dtype, nb, N, y0, u0, nitems, item_table, item_bundle and clip are
 * rtx_trace_reduce_many's; item i is centred on centers[2i .. 2i+1] (host
 * (nitems, 2), or NULL for 0).  Every item shares the planes z (host, K =
 * planes values) and the frequencies freqs (host, F = nfreq values nu_j in
 * cycles per length unit, any order: rtx_otf_jacobian_sums' convention).
 * Each ray's state at surface S-1 is the last row rtx_trace stores for the
 * same table, in every mode, and its point at plane k is rtx_otf_rows' with
 * no offset (FP64, every operation separately rounded, FP32 rays widened
 * first):
 *   d = y_xy - c,  u = i_xy / i_z,  q_k = d + z[k] u
 * A ray counts at plane k iff both components of q_k are finite (so a ray
 * with i_z = 0 counts at no plane, not even at z = 0).  For a in {x, y}:
 *   S[k,a,j] = sum over the counted rays of exp(-2 pi i nu_j q_k[a])
 *   count[k] = number of counted rays;  OTF = S / count,  MTF = |OTF|
 * with one sincospi(2 fl(nu_j q_k[a])) per term.  sums: host (nitems, K, 2,
 * F, 2) doubles (re, im), count: host (nitems, K) int64; exactly
 * nitems*K*2*F*2 doubles and nitems*K counts are written, zeros for N = 0.
 *
 * Deterministic: in each 512-ray tile of an item the rays are staged in
 * shared memory; for each (plane, axis, frequency) unit lane l adds the
 * terms of rays l, l + 32, .., l + 480 in that order, the 32 lanes are added
 * by a shuffle tree, and the tile's sums go to its own row in the context.
 * A second kernel adds each item's rows in tile order (no atomics).  So an
 * item gives the same bits in every call and context, whatever the grid and
 * whatever other items share the launch, in any order.
 *
 * Error bound against the exact sums of the same q_k, eps = 2^-52,
 * Phi = max |nu_j q_k[a]| over the counted rays:
 *   |S - S_exact| <= (D + 4 Phi + 3) eps count[k]   per component
 *   D = 20 + ceil(N / 512)   (the summation depth)
 * D bounds the additions: 15 in a lane, 5 in the shuffle tree and
 * ceil(N/512) - 1 over the tiles, each partial sum's components at most the
 * sum of the terms' magnitudes; 4 Phi the rounding of nu q, which moves the
 * phase by at most pi Phi eps; 3 the 2 ulp of each sincospi component and
 * one more.  Counts are exact.
 *
 * RTX_E_BADARG, before any device work or allocation: every refusal of
 * rtx_trace_reduce_many (with sums and count in place of m); planes outside
 * 1..RTX_OTF_MAX_PLANES or nfreq outside 1..RTX_OTF_MAX_FREQS; a NULL z,
 * freqs, sums or count; a non-finite z, frequency or centre.  RTX_E_UNSUPPORTED
 * as rtx_trace_reduce_many.  The device tables, the items and the tile rows
 * ((K*2*F*2 + K) doubles per tile) are kept in the context: RTX_E_NOMEM
 * before allocating when they do not fit.  Synchronous; rtx_last_kernel_ms
 * covers the two kernels.
 */
int rtx_trace_otf_many(rtx_ctx *ctx, int nt, const rtx_surface *tables, int S,
                       const double *rot0, int dtype, int nb, const int64_t *N,
                       const void *const *y0, const void *const *u0,
                       int64_t nitems, const int32_t *item_table,
                       const int32_t *item_bundle, const double *centers,
                       int clip, int planes, const double *z, int nfreq,
                       const double *freqs, double *sums, int64_t *count,
                       unsigned flags);

/* ---- tolerance analysis on the rms wavefront ----------------------------- */
/*
 * rtx_trace_opd's per-ray path A and sphere point P of many (surface table,
 * launch bundle) items in ONE launch, reduced to the sums of a least-squares
 * fit of piston and tilt -- the rms wavefront of thousands of perturbed
 * lenses.  tables, S, rot0, nb, N, y0, u0, nitems, item_table, item_bundle
 * and clip are rtx_trace_reduce_many's; the tables are the march to `after`,
 * as rtx_trace_opd's (surf[S] = system[1:after+1]: the image record is not
 * marched).  Item i has its own sphere specs[i] (host, nitems records), its
 * piston guess a0[i] (host, nitems doubles, or NULL for 0) and its pupil
 * centre centers[2i .. 2i+1] (host (nitems, 2), or NULL for 0).
 *
 * Per ray, in FP64 with every operation separately rounded: A and P are the
 * values rtx_trace_opd writes for the item's table and spec, bit for bit,
 *   a = A - a0,  x = P_x - c_x,  y = P_y - c_y
 * and the ray enters iff a, x and y are all finite.  sums: host (nitems,
 * RTX_WFE_NSUMS), each row over the rays that enter, in this order:
 *   n, sum a, sum a^2, sum x, sum y, sum x^2, sum xy, sum y^2, sum ax, sum ay
 * zeros for N = 0; exactly nitems*RTX_WFE_NSUMS doubles are written.  With
 * a0 = A[ref], c = P_xy[ref] the residuals are opd()'s chief-referenced t
 * (times -l/scale) and py.
 *
 * Deterministic as rtx_trace_reduce_many: each 512-ray tile's sums (every
 * product rounded once, then a lane's 2 rays, a shuffle tree, the 8 warps
 * in order) go to the tile's own row, and a second kernel adds each item's
 * rows in tile order (no atomics).  An item gives the same bits in every
 * call and context, whatever other items share the launch, in any order.
 * Error bound against the exact sums of the same a, x, y (the terms are
 * the exact products), eps = 2^-52:
 *   |sum - exact| <= (ceil(N/512) + 64) eps sum|term|   per sum
 * (the summation depth is 12 + ceil(N/512) additions and one product
 * rounding, each eps/2).  Counts are exact.
 *
 * FP64 only, fast or RTX_EXACT: RTX_F32 returns RTX_E_UNSUPPORTED (an FP32
 * path sum of a ~100 mm track is worth about 0.02 waves).  RTX_E_BADARG,
 * before any device work or allocation: every refusal of
 * rtx_trace_reduce_many (with sums in place of m); a NULL specs; a
 * non-finite a0, centre or spec member; a zero radius.  The device tables,
 * the items, their specs and the tile rows (RTX_NMOMENTS doubles per tile)
 * are kept in the context: RTX_E_NOMEM before allocating when they do not
 * fit.  Synchronous; rtx_last_kernel_ms covers the two kernels.
 */
#define RTX_WFE_NSUMS 10
int rtx_trace_opd_many(rtx_ctx *ctx, int nt, const rtx_surface *tables, int S,
                       const double *rot0, int dtype, int nb, const int64_t *N,
                       const void *const *y0, const void *const *u0,
                       int64_t nitems, const int32_t *item_table,
                       const int32_t *item_bundle, const rtx_opd *specs,
                       const double *a0, const double *centers, int clip,
                       double *sums, unsigned flags);

/* ---- Zernike decomposition of the wavefront ------------------------------ */
/*
 * rtx_trace_opd_many's items and per-ray residuals, reduced to the sums of
 * a least-squares fit of the Zernike polynomials Z_1 .. Z_J to a.
 * Arguments as rtx_trace_opd_many, plus the radial order `order` (0 ..
 * RTX_ZRN_MAX_ORDER; J = (order+1)(order+2)/2 <= 45) and rho (host, nitems
 * doubles), item i's normalisation radius: the pupil point of a ray is
 * (u, v) = (x, y)/rho.  Per ray a, x, y and the entry rule (a, x and y all
 * finite) are rtx_trace_opd_many's, bit for bit.
 *
 * Basis: Noll's order, orthonormal on the unit disc (mean of Z_j Z_k over
 * the disc = delta_jk).  Z_j has radial order n and azimuthal order m,
 *   Z = sqrt(n+1) R_n^0(r)                  m = 0
 *   Z = sqrt(2(n+1)) R_n^m(r) cos(m theta)  j even
 *   Z = sqrt(2(n+1)) R_n^m(r) sin(m theta)  j odd
 * with theta from the image-frame x axis (so Z2 = 2u, Z3 = 2v, Z4 =
 * sqrt3 (2r^2 - 1), Z5 = sqrt6 r^2 sin 2theta, Z6 = sqrt6 r^2 cos 2theta,
 * Z7 = sqrt8 (3r^3 - 2r) sin theta, Z11 = sqrt5 (6r^4 - 6r^2 + 1)).  The
 * device evaluates it without atan2, every operation separately rounded:
 * u = x/rho, v = y/rho, s = u^2 + v^2, R_n^m/r^m by Horner in s with its
 * integer coefficients c_k, (u + iv)^m by repeated complex multiplication,
 * Z = (N Q) Re or Im of it with N the rounded sqrt.
 *
 * sums: host (nitems, E), E = (J+1)(J+2)/2: the upper triangle, row-major,
 * of the Gram sums of v = (a, Z_1, .., Z_J) over the rays that enter:
 *   sum a^2, sum a Z_1 .. sum a Z_J, sum Z_1 Z_1, sum Z_1 Z_2, .. sum Z_J Z_J
 * so sum a Z_1 = sum a and sum Z_1 Z_1 = n exactly (Z_1 = 1).  r2max: host
 * (nitems,), the largest x^2 + y^2 (each rounded) over the rays that enter,
 * 0 for none; exact.  Zeros for N = 0.
 *
 * Deterministic: each 512-ray tile's row (each entry added over the tile's
 * rays in ray order by one thread, every product and sum rounded once; the
 * max is exact) goes to the tile's own row, and a second kernel adds each
 * item's rows in tile order (no atomics).  An item's bits depend only on
 * its rays, table, spec, a0, centre and rho.
 *
 * Error bound, eps = 2^-52, in two parts:
 *  (a) one basis value against the exact Z_j at the same (x, y)/rho, at
 *      the normalised radius r = |(x, y)|/rho and R = max(1, r):
 *        |Z~_j - Z_j| <= (n+2)^2 eps N_j A_j R^n
 *      N_j = sqrt(n+1) or sqrt(2(n+1)), A_j = sum_k |c_k| the sum of R_n^m's
 *      coefficient magnitudes (R_8^0: 321).  Derivation, u = eps/2:
 *      rounding u, v perturbs the point by <= u r, worth n^2 u sup|Z| over
 *      the disc of radius R by Kellogg's bound |grad p| <= n^2 sup|p| / R,
 *      and sup|Z| <= N A R^n; s carries 2u, worth 2K u N A R^n through
 *      |dQ/ds| <= K A R^(2K-2); Horner of degree K adds 2K u N A R^n; each
 *      complex product adds sqrt2 * 2u |C||w|, so C_m is within 2 sqrt2 m
 *      u R^m; N and the two products add 3u.  The sum, n^2 + 4K + 2.9m + 3
 *      <= (n+2)^2 - 1 with n = 2K + m, times u, is within the bound.
 *  (b) the summation of the rounded products of the device values:
 *        |sum - sum of the products| <= (512 + ceil(N/512)) eps sum|term|
 *      (a tile's depth is 511 additions and the product's rounding, each
 *      u, and ceil(N/512) - 1 additions join the tiles).
 * A sum's error against the exact sums of the exact basis is therefore
 * within (b) plus sum over the rays of E_p |v_q| + |v_p| E_q + E_p E_q with
 * E the bound (a) of each factor (0 for a).  Counts and r2max are exact.
 *
 * FP64 only, fast or RTX_EXACT: RTX_F32 returns RTX_E_UNSUPPORTED.
 * RTX_E_BADARG, before any device work or allocation: every refusal of
 * rtx_trace_opd_many; a NULL rho or r2max; an order outside 0 ..
 * RTX_ZRN_MAX_ORDER; a non-finite or non-positive rho.  The tile rows
 * (E + 1 doubles per tile) are kept in the context with the tables, items
 * and specs: RTX_E_NOMEM before allocating when they do not fit.
 * Synchronous; rtx_last_kernel_ms covers the two kernels.
 */
#define RTX_ZRN_MAX_ORDER 8
int rtx_trace_zernike_many(rtx_ctx *ctx, int nt, const rtx_surface *tables,
                           int S, const double *rot0, int dtype, int nb,
                           const int64_t *N, const void *const *y0,
                           const void *const *u0, int64_t nitems,
                           const int32_t *item_table,
                           const int32_t *item_bundle, const rtx_opd *specs,
                           const double *a0, const double *centers, int clip,
                           int order, const double *rho, double *sums,
                           double *r2max, unsigned flags);

/* ---- launch rays generated in HBM (SURVEY 8f-2) -------------------------- */
/*
 * The pupil grids of pupil_distribution (rayopt/utils.py:118-199), Pupil.map
 * with its elliptical filter (rayopt/pupils.py:97-107) and
 * Conjugate.aim (rayopt/conjugates.py:137-166, 236-255) evaluated per ray on
 * the device.  Candidates rejected by a predicate (mesh points outside the
 * unit circle, rays outside the filter ellipse) are squeezed out in order
 * (two passes: block counts, host prefix sum, generation).
 *
 *  conjugate  0 infinite: frame = {u[3], ybase[3] = yz - z*u, s[3], m[3]}
 *             1 finite:   frame = {y[3] object point, u0[3], s[3], m[3]}
 *             (the projection, a telecentric pupil and a curved FINITE object
 *             surface only change these per-field constants: the host computes
 *             them with the reference's expressions, rayopt_b200/rays.py)
 *  grid       RTX_GRID_*; n = rings (hexapolar), mesh side (square,
 *             triangular: n x n points clipped to the unit circle + centre
 *             ray), number of random rays (+ centre ray); RTX_GRID_LINES: up to
 *             two np.linspace segments seg[k] = (x0, y0, x1, y1) of seg_m[k]
 *             points (meridional, sagittal, cross, tee, half-meridional);
 *             RTX_GRID_GIVEN: pupil coordinates yp, DEVICE (n_given, 2) FP64
 *  pmax       Pupil.map's scale fabs(a).max() (finite: of arctan2(a, z))
 *  filter     keep ((q - fc)^2 / fd2).sum() <= 1, q the scaled coordinates
 *  curved     infinite object only: intercept the rays with `surface`
 *             (system[0], in its own frame) instead of the plane z = 0
 */
#define RTX_GRID_GIVEN      0
#define RTX_GRID_HEXAPOLAR  1
#define RTX_GRID_SQUARE     2
#define RTX_GRID_TRIANGULAR 3
#define RTX_GRID_RANDOM     4
#define RTX_GRID_LINES      5
typedef struct rtx_aim {
    int32_t conjugate, grid, filter, curved;
    int64_t n;
    uint64_t seed;      /* RTX_GRID_RANDOM: counter-based generator */
    double seg[2][4];
    int64_t seg_m[2];
    double frame[12];
    double pmax, z;
    double fc[2], fd2[2];
    rtx_surface surface;
} rtx_aim;
/* number of rays the spec generates (runs the counting pass when a predicate
 * can reject candidates; the plan is cached in the context) */
int rtx_aim_plan(rtx_ctx *ctx, const rtx_aim *spec, int64_t n_given,
                 const void *yp, int64_t *n_rays);
/* rays first .. first+count-1 of the bundle into DEVICE y0,u0 (count,3) of
 * dtype; yp_out: optional DEVICE (count,2) FP64 receiving the fractional pupil
 * coordinates of those rays.  Asynchronous on the context stream. */
int rtx_aim_rays(rtx_ctx *ctx, const rtx_aim *spec, int64_t n_given,
                 const void *yp, int dtype, int64_t first, int64_t count,
                 void *y0, void *u0, void *yp_out);

/*
 * Moments for GeometricTrace.refocus (rayopt/geometric_trace.py:82-99) on
 * DEVICE arrays of one surface: y = intercepts (N,3), inc = incidence
 * directions (N,3); u = inc_xy/inc_z (tanarcsin); rays with non-finite u are
 * skipped.  About `center` = (y_x, y_y, u_x, u_y) (host, or NULL = 0):
 * m[0]=#good, m[1]=#total, m[2..3]=sum dy, m[4..5]=sum du,
 * m[6]=sum w (dy.du), m[7]=sum w (du.du).  The focus shift is
 * -m[6]/m[7] taken about the means of the good rays (two calls).
 */
int rtx_focus_moments(rtx_ctx *ctx, int dtype, int64_t N, const void *y,
                      const void *inc, const void *w, const double *center,
                      double *m);

/* ---- diffraction PSF (GeometricTrace.psf, rayopt/geometric_trace.py:133-169) */
/*
 * Linear interpolation of scattered values on a GIVEN triangulation -- the
 * evaluation of griddata(method="linear", fill_value=nan)
 * (geometric_trace.py:141) with the triangulation scipy.spatial.Delaunay made
 * on the host.  All arrays are DEVICE arrays of `dtype` (RTX_F64 only; RTX_F32
 * returns RTX_E_UNSUPPORTED):
 *   pts (M,2) points, vals (M,) their values,
 *   simplices (T,3) int32 and transform (T,3,2): Delaunay.simplices and
 *     Delaunay.transform as they are (degenerate simplices keep their NaNs and
 *     never cover a node),
 *   gh (n,) the grid axis, 2 <= n <= 46340: node (i, j) is (gh[i], gh[j]);
 *     any strictly monotone finite axis, ascending or descending, evenly
 *     spaced or not (each simplex finds its nodes by binary search on gh;
 *     the axis is not checked, another one gives unspecified outputs),
 *   out (n,n) receives the values, NaN where no simplex covers the node,
 *   winner (n,n) int32 or NULL receives the covering simplex, the lowest
 *     index among the simplices that cover the node within scipy's tolerance
 *     (100 DBL_EPSILON in barycentric coordinates), INT32_MAX for none.
 * The barycentric coordinates and the value follow scipy's evaluation order
 * with unfused IEEE operations: a node whose covering simplex is the one
 * Delaunay.find_simplex returns gets griddata's value bit for bit.
 * Asynchronous; rtx_last_kernel_ms gives the device time of the call.
 */
int rtx_grid_linear(rtx_ctx *ctx, int dtype, int64_t M, const void *pts,
                    const void *vals, int64_t T, const int32_t *simplices,
                    const void *transform, int n, const void *gh, void *out,
                    int32_t *winner);

/*
 * Device bytes an rtx_psf call on an (n,n) grid with zero padding `pad`
 * allocates: the (pad n)^2 complex grid, plus cuFFT's work area unless the
 * context's cached plan already has that shape.  RTX_E_UNSUPPORTED without
 * cuFFT.
 */
int rtx_psf_bytes(rtx_ctx *ctx, int n, int pad, size_t *bytes);

/*
 * The diffraction PSF of a regridded OPD o (DEVICE (n,n), waves, NaN outside
 * the pupil; RTX_F64 only):
 *   z = where(isfinite(o), exp(-2 pi i o), 0)/sqrt(#finite), zero-padded at
 *       the end to (nx, ny) = (pad n, pad n),
 *   psf = |fft2(z)|^2/(nx ny)   DEVICE (nx, ny), unnormalised forward FFT.
 * stats (host, 5 doubles, or NULL) receives #finite nodes, sum psf, max psf,
 * and sum psf*k_p, sum psf*k_q with k the signed frequency index of
 * np.fft.fftfreq along each axis (0, 1, .., -1): times 1/(nx d) these are the
 * first moments about the frequency axes fftfreq(nx, d).  Sums are taken in a
 * fixed order (the same inputs give the same bits).
 * cuFFT (libcufft.so.11) is opened on the first call; without it the call
 * returns RTX_E_UNSUPPORTED.  The plan of the last (nx, ny) and its work area
 * are cached in the context.  When the complex grid and the work area do not
 * fit in free device memory the call returns RTX_E_NOMEM before it allocates
 * anything.  Synchronous.
 */
int rtx_psf(rtx_ctx *ctx, int dtype, int n, const void *o, int pad, void *psf,
            double *stats);

/*
 * Encircled-energy bins and line sums of a PSF -- what Analysis.opds
 * (rayopt/analysis.py:330-346) reduces it to -- in one read of the PSF.
 * psf is a DEVICE (nx, ny) array in the FFT order rtx_psf writes (RTX_F64
 * only; RTX_F32 returns RTX_E_UNSUPPORTED).  The shifted index I (of
 * np.fft.fftshift(psf)) is stored row (I - nx/2) mod nx, J likewise.  Host
 * outputs, each may be NULL (then skipped):
 *   ee (nbins,)  sum of the pixels whose bin about the centre (c0, c1), given
 *                in the shifted frame, is b = trunc(sqrt((J-c1)^2 + (I-c0)^2))
 *                with each operation rounded separately as numpy does:
 *                polar_sum(fftshift(psf), (c0, c1), "azimuthal")
 *                (special_sums.py:240-263, aspect 1, binsize 1),
 *   lsf0 (ny,)   column sums sum_I psf[I, J],
 *   lsf1 (nx,)   row sums sum_J psf[I, J], both in the stored order
 *                (ifftshift(fftshift(psf).sum(i))).
 * nbins must be np.bincount's length, 1 + the largest bin, which lies at a
 * corner of the array.  Every sum is taken in a fixed order (the same PSF and
 * centre give the same bits); the pixels are >= 0, so each sum's relative
 * error is at most (L + 200) DBL_EPSILON/2, L = ceil(tiles/132) with
 * tiles = ceil(nx/64) ceil(ny/64).  RTX_E_BADARG for NULL ctx or psf, nx or ny < 1, a non-finite
 * centre, another nbins, or a negative or non-finite pixel (found by the
 * kernel; outputs then unspecified).  Scratch of 133 (nbins + nx + ny) doubles
 * is kept in the context; RTX_E_NOMEM before allocating when it does not fit.
 * Synchronous; rtx_last_kernel_ms gives the device time of the call.
 */
int rtx_psf_profiles(rtx_ctx *ctx, int dtype, int64_t nx, int64_t ny,
                     const void *psf, double c0, double c1, int64_t nbins,
                     double *ee, double *lsf0, double *lsf1);

/*
 * Delaunay triangulation of M DEVICE points pts (M,2) on the device, in the
 * layout scipy.spatial.Delaunay gives and rtx_grid_linear takes (RTX_F64 only;
 * RTX_F32 returns RTX_E_UNSUPPORTED).  DEVICE outputs with room for 2*M
 * triangles; *T (host) receives their number:
 *   simplices (T,3) int32, counter-clockwise,
 *   neighbors (T,3) int32 or NULL: the triangle opposite vertex k, -1 on the hull,
 *   transform (T,3,2) FP64 or NULL: {Tinv, r}, r the last vertex and Tinv the
 *     inverse (explicit 2x2 formula) of T = [v0 - r, v1 - r] as columns;
 *     each entry within (3 rho + 3) DBL_EPSILON/2 of the exact inverse, rho =
 *     (|t00 t11| + |t01 t10|)/|det|; a NaN row where the rounded determinant
 *     is 0 (vertices collinear to rounding, never exactly), which covers no
 *     node, as scipy's transform is NaN for a nearly singular simplex.
 * The triangulation is exactly Delaunay: orient2d and incircle are exact
 * (rtx_selftest_predicates), an edge is flipped only when its opposite vertex
 * is strictly inside the circumcircle, and the triangles cover exactly the
 * convex hull, collinear hull points included, with no zero-area triangle.
 * Where the Delaunay triangulation is unique it is scipy's; among cocircular
 * points the choice is deterministic but may differ from qhull's.  An exact
 * duplicate of a point is not a vertex (the lowest index is kept).  The same
 * points give the same bits in every call and context.
 * Domain: every coordinate is 0 or 2^-200 <= |x| <= 2^200, so that no
 * product of the exact predicates underflows or overflows.
 * RTX_E_BADARG for M < 3 or M >= 2^30, a non-finite point or a coordinate
 * outside the domain, and when all points are collinear (scipy raises
 * QhullError).  The workspace (rtx_delaunay_bytes) is kept in the context;
 * RTX_E_NOMEM before allocating anything when it does not fit in free device
 * memory.  Not included there: the exact incircle's 3.3 KB stack frame, for
 * which the driver reserves local memory on every resident thread at the
 * first call in a context and keeps it (592 MB on an H100 80GB).  Synchronous; rtx_last_kernel_ms gives the device time of the call.
 */
int rtx_delaunay(rtx_ctx *ctx, int dtype, int64_t M, const void *pts, int64_t *T,
                 int32_t *simplices, int32_t *neighbors, void *transform);
/* device bytes of the workspace rtx_delaunay needs for M points (allocated by
 * a call only when the context keeps a smaller one) */
int rtx_delaunay_bytes(rtx_ctx *ctx, int64_t M, size_t *bytes);

/*
 * The finite exit-pupil points of a per-ray OPD, compacted in HBM: what
 * ResidentMixin.opd_rays and the filter of GeometricTrace.opd
 * (rayopt/geometric_trace.py:125-135) compute on the host, bit for bit.
 * A (N,) and P (N,3) are the DEVICE outputs of rtx_trace_opd (RTX_F64 only;
 * RTX_F32 returns RTX_E_UNSUPPORTED).  With aref = A[ref], pref = P[ref], for
 * each ray j, every operation separately rounded:
 *   t = -(A[j] - aref)/k   (k = l/scale, the wavelength in lens units),
 *   x = P[j].x - pref.x,  y = P[j].y - pref.y   (P[j].z plays no part).
 * The rays with x, y and t all finite are written in increasing j to the
 * DEVICE arrays pts (M,2) = (x, y) and vals (M,) = t; nothing is written at or
 * after index M.  *M (host) receives the count, *h (host) max(|x|, |y|) over
 * the kept rays (0 when M = 0).  A non-finite reference ray gives M = 0.
 * The compaction is a prefix sum of the keep flags; the maximum an integer
 * atomicMax on the bits of non-negative doubles: the same inputs give the
 * same bits.  Workspace of 4 N bytes kept in the context; RTX_E_NOMEM before
 * allocating it when it does not fit.  RTX_E_BADARG before any device work
 * for a NULL ctx or pointer, N < 1 or N >= 2^31, ref outside [0, N), and k
 * zero or not finite.  Synchronous (reads the 16 bytes of M and h);
 * rtx_last_kernel_ms gives the device time of the call.
 */
int rtx_opd_points(rtx_ctx *ctx, int dtype, int64_t N, const void *A, const void *P,
                   int64_t ref, double k, double *pts, double *vals, int64_t *M,
                   double *h);

/*
 * Finite count, minimum and maximum of a DEVICE grid o (n,) (RTX_F64 only;
 * RTX_F32 returns RTX_E_UNSUPPORTED): the PTP and the largest |o| Analysis.opds
 * takes of the regridded OPD (rayopt/analysis.py:309-315).  NaN and +-inf
 * are skipped; -0 counts below +0.  *count, *lo, *hi (host) receive the
 * results; lo and hi are NaN when no value is finite.  Exact (integer
 * atomics on order keys).  RTX_E_BADARG for a NULL ctx or pointer or n < 1.
 * Synchronous; rtx_last_kernel_ms gives the device time of the call.
 */
int rtx_grid_range(rtx_ctx *ctx, int dtype, int64_t n, const void *o, int64_t *count,
                   double *lo, double *hi);

/* ---- diffraction PSF by direct summation over the exit-pupil rays -------- */
/*
 * The Debye (Fourier) sum of the pupil function over the traced rays
 * themselves, on an image grid the caller chooses, through focus.  Inputs are
 * rtx_trace_opd's A (N,) and P (N,3) (DEVICE, FP64): P in the image frame
 * relative to the sphere centre, the chief ray's image point, so that
 * s_j = -P_j/R is the unit direction from the ray's sphere point to the
 * centre.  With the optional DEVICE weights w (N,) (NULL: all 1),
 *   U_k(a, b) = sum_j w_j exp(2 pi i [ (A_j - a0)/lambda
 *                                     + kappa (sx_j p_a + sy_j q_b + sz_j z_k) ])
 *   p_a = p0 + a dp (a < nx),  q_b = q0 + b dq (b < ny),  k < planes
 * over the rays whose A_j, P_j and w_j are finite; the others are left out
 * and counted.  a0 is the chief ray's A (it keeps the phases small), lambda
 * the wavelength in lens units, kappa = n_image/lambda, R the sphere radius
 * (rtx_opd.radius).  This is the first order in the image point X of
 * n |X - P_j|; +z is along the image frame's z, as in rtx_spot_rows.
 * At z = 0 on the grid p_a = fftfreq(nx, dx kappa/R) of a regridded OPD o
 * (nodes x_m = x_0 + m dx used as rays, w = 1, A = a0 - lambda o), rtx_psf's
 * PSF is |U|^2/(n nx ny) exactly (n the finite nodes): the FFT's own phase
 * convention, up to a unit phase per pixel.  The intensity in Strehl units is
 * I = |U|^2/(sum w)^2: 1 at the chief point for an aberration-free pupil.
 */
#define RTX_PUPIL_MAX_PLANES 16
#define RTX_PUPIL_MAX_PIXELS 4096  /* nx, ny */
#define RTX_PUPIL_CHUNK      32    /* rays summed into a fresh accumulator */
#define RTX_PUPIL_SLOT       2048  /* least rays per slot */
#define RTX_PUPIL_MAX_SLOTS  16
typedef struct rtx_pupil {
    int32_t planes;                  /* K in 1..16 */
    int32_t reserved;                /* 0 */
    int64_t nx, ny;                  /* 1..RTX_PUPIL_MAX_PIXELS */
    double a0;                       /* reference path (the chief ray's A) */
    double wavelength;               /* lambda in lens units */
    double kappa;                    /* n_image/lambda */
    double radius;                   /* R */
    double p0, dp, q0, dq;           /* p_a = p0 + a dp, q_b = q0 + b dq */
    double z[RTX_PUPIL_MAX_PLANES];  /* defocus distances */
} rtx_pupil;
size_t rtx_sizeof_pupil(void);

/*
 * rtx_pupil_sum ADDS U to the DEVICE complex (K, nx, ny) array U (re, im
 * interleaved, 2 K nx ny doubles) and writes *count (rays summed) and *sumw
 * (their sum of w; the count when w is NULL) on the host.  Calls add up, so
 * a bundle can be summed in chunks of rays (memory is bounded by the chunk).
 * Synchronous; rtx_last_kernel_ms covers both kernels.
 *
 * Kernel: per plane U_k = X^T diag(c_k) Y, X_j(a) = exp(2 pi i kappa sx_j
 * p_a), Y_j(b) = exp(2 pi i kappa sy_j q_b), c_kj = w_j exp(2 pi i [(A_j -
 * a0)/lambda + kappa sz_j z_k]): an (nx x N)(N x ny) complex product on the
 * FP64 tensor cores (mma m16n8k16).  X and Y of RTX_PUPIL_CHUNK rays are made
 * in shared memory once per chunk, with one sincospi per block of 8 pixels
 * stepped by the phasor of dp (dq), and serve up to 8 planes (K > 8 runs
 * ceil(K/8) plane groups).
 *
 * Deterministic: the rays are cut into slots of L = max(RTX_PUPIL_SLOT,
 * ceil(N/RTX_PUPIL_MAX_SLOTS)) rays rounded up to RTX_PUPIL_CHUNK; within a
 * slot each chunk is summed into a fresh accumulator and added to the slot's
 * sum in chunk order; a second kernel adds the slots in slot order and then
 * the result to U (no atomics).  The bits depend only on A, P, w, N and the
 * record, not on the launch grid, the context or the call.
 *
 * Error bound, eps = 2^-52, per component of the sum one call adds:
 *   |U - U_exact| <= (D + 24 Phi + 40) eps sum |w|
 *   D = 2 RTX_PUPIL_CHUNK + ceil(L/RTX_PUPIL_CHUNK) + slots + 1  (summation depth)
 *   Phi = max over the summed rays of |A_j - a0|/|lambda| + |kappa| (|sx_j|
 *         (|p0| + (nx-1)|dp|) + |sy_j| (|q0| + (ny-1)|dq|) + |sz_j| max|z_k|)
 * 24 Phi bounds the rounding of the phases (4 pi Phi for c, 7 pi Phi for each
 * of X and Y, whose steps carry the step phase's error through 7 products);
 * 40 the sincospi, product and step roundings of one term.
 *
 * RTX_E_BADARG, before any device work or allocation: NULL ctx, spec, U,
 * count or sumw; N < 0; NULL A or P with N > 0; planes outside 1..16; nx or
 * ny outside 1..RTX_PUPIL_MAX_PIXELS; reserved != 0; a zero or non-finite
 * wavelength or radius; a non-finite a0, kappa, p0, dp, q0, dq or z.  N = 0
 * adds nothing and launches nothing.  The slot sums (slots (2 K nx ny + 2)
 * doubles) are kept in the context: RTX_E_NOMEM before allocating them when
 * they do not fit in free device memory.
 */
int rtx_pupil_sum(rtx_ctx *ctx, int64_t N, const double *A, const double *P,
                  const double *w, const rtx_pupil *spec, double *U, int64_t *count,
                  double *sumw);

/*
 * I = scale |U_k(a, b)|^2 ADDED to the DEVICE (K, nx, ny) PSF psf, for the
 * complex U of rtx_pupil_sum on the grid of `spec` (scale = 1/(sum w)^2 gives
 * Strehl units; calls for several wavelengths with their spectral weights
 * accumulate a polychromatic PSF).  stats (host, (K, 5) doubles, or NULL)
 * receives per plane, over the PSF after the addition: sum psf, max psf, the
 * flat index a ny + b of its first maximum, sum psf p_a and sum psf q_b.  The
 * sums are taken in a fixed order (fixed blocks of pixels, fixed tree order,
 * the blocks in order on the host): the same inputs give the same bits.
 * RTX_E_BADARG before any device work for a NULL ctx, spec, U or psf, a
 * record rtx_pupil_sum refuses, or a non-finite scale.  Scratch of
 * K ceil(nx ny/2048) 5 doubles is kept in the context; RTX_E_NOMEM before
 * allocating it when it does not fit.  Synchronous; rtx_last_kernel_ms gives
 * the device time of the call.
 */
int rtx_pupil_intensity(rtx_ctx *ctx, const rtx_pupil *spec, const double *U, double scale,
                        double *psf, double *stats);

#ifdef __cplusplus
}
#endif
#endif /* RTX_H */
