// Kernel body of the image-source room impulse response (kapre_rir_ism; DESIGN.md §RIR).
//
// Room [0, Lx] x [0, Ly] x [0, Lz], source s, microphone m, walls (x=0, x=Lx, y=0, y=Ly, z=0, z=Lz) with pressure
// reflection coefficients beta_w.  An image is (n, p), n in Z^3, p in {0, 1}^3:
//   i_d = 2 n_d L_d + (1 - 2 p_d) s_d,   r = |i - m|,   tau = r fs / c samples,
//   g = prod_d beta_(d,lo)^|n_d - p_d| beta_(d,hi)^|n_d| / (4 pi r),
//   h[floor(tau) + k] += g w[k] sinc(k - half - frac(tau)),   k = 0 .. W-1,   w = np.hanning(W),
// with only the images of order sum_d (|n_d - p_d| + |n_d|) <= max_order when it is set.
//
// One CTA per tile of 32 nw output samples of one (item, mic); thread `tid` owns sample t0 + tid and sums its taps in
// float32, in one fixed global order of the images: (n_x, p_x, n_y, p_y, n_z, p_z) ascending.  The CTA enumerates the
// images whose taps reach the tile (a spherical shell around the mic): rows (n_x, p_x) that meet the ball, the columns
// (n_y, p_y) of each row that meet it, and per column the n_z ranges of the shell's two caps.  Each column batch is
// counted, prefix-summed and written into a shared-memory chunk in enumeration order, which every warp then walks in
// order.  So h[t] is the same sum in the same order whatever the tile size, the first sample requested, the batch or
// the grid, and the kernel needs no atomics.
//
// tau is formed in float64 with the restatement's exact operation order ((2 n) L +- s - m, then
// sqrt((dx dx + dy dy) + dz dz), then (r fs) / c, each rounded once), so floor(tau) and frac(tau) are bit for bit
// those of tests/rir_ref.py.  With nc = round(tau) and e = tau - nc in [-1/2, 1/2] (exact),
//   sinc(k - half - f) = (-1)^(jj + 1) sin(pi e) / (pi (jj - e)),   jj = floor(tau) + k - half - nc,
// so an image needs one float64 sin (A = g sin(pi e) / pi, rounded once) and a tap is A ws[k] / (jj - e) in float32,
// with the window's sign pattern folded into ws.  Referring jj to the nearest integer keeps the denominator's
// relative error at 2 ulp when e is tiny.  e = 0 gives the single tap g w[half].
//
// The body is written as barrier-free phases (KB_RIR_THREADS ... KB_RIR_SYNC); the CPU emulation under KB_HOST_EMU
// runs each phase as a loop over the CTA's threads.
#pragma once
#include "kb_common.h"

#define KB_RIR_REC 14                 // float64 per item: room[3], source[3], beta[6], max_order (-1: none), start
#define KB_RIR_MAX_W 255              // longest fractional-delay filter
#define KB_RIR_MAX_NW 8               // warps per CTA (32 output samples each)
#define KB_RIR_CAP 1024               // images staged per chunk
#define KB_RIR_MAX_IMAGES (1LL << 24) // cap on a response's analytic image bound (DESIGN.md §RIR)

#if defined(KB_HOST_EMU)
#define KB_RIR_FN inline
#define KB_RIR_THREADS for (int tid = 0; tid < nt; ++tid)
#define KB_RIR_SYNC
#else
#define KB_RIR_FN __device__ __forceinline__
#define KB_RIR_THREADS for (int tid = (int)threadIdx.x, once_ = 1; once_; once_ = 0)
#define KB_RIR_SYNC __syncthreads()
#endif

struct KbRirParams {
    const double* rec;                     // (B, KB_RIR_REC)
    const double* mic;                     // (B, M, 3)
    float* out;                            // (B, M, L) at element strides (o_sb, o_sm, o_st)
    long long o_sb, o_sm, o_st;
    int B, M, L, W, nw, n_tt;              // n_tt = ceil(L / (32 nw)) tiles per (item, mic)
    double fs, c;
    float ws[KB_RIR_MAX_W];                // w[k] (-1)^(k + 1 - half)
};

struct KbRirImg { int n0, nch; float e, A; };   // floor(tau), round(tau) + half, tau - round(tau), +-g sin(pi e)/pi

// Shared memory of one CTA (bytes), for nt = 32 nw threads.
struct KbRirSmem { int img, ws, acc, cnt, tmp, ny0, total; };
KB_HD KbRirSmem kb_rir_smem(int nt) {
    KbRirSmem s;
    int off = 0;
    s.img = off; off += KB_RIR_CAP * (int)sizeof(KbRirImg);
    s.ws = off; off += kb_align16(KB_RIR_MAX_W * 4);
    s.acc = off; off += nt * 4;
    s.cnt = off; off += nt * 4;            // row or column counts, scanned in place
    s.tmp = off; off += nt * 4;
    s.ny0 = off; off += nt * 4;            // first n_y of each row of the row group
    s.total = kb_align16(off);
    return s;
}

// Rounded float64 steps, never contracted into FMAs: tau must be the restatement's bit for bit.
KB_HD double kb_rir_add(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __dadd_rn(a, b);
#else
    return a + b;
#endif
}
KB_HD double kb_rir_mul(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __dmul_rn(a, b);
#else
    return a * b;
#endif
}
KB_HD double kb_rir_sqrt(double a) {
#if defined(__CUDA_ARCH__)
    return __dsqrt_rn(a);
#else
    return std::sqrt(a);
#endif
}
KB_HD double kb_rir_div(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __ddiv_rn(a, b);
#else
    return a / b;
#endif
}

// Image coordinate minus the mic's: (2 n) L + (1 - 2 p) s - m.
KB_HD double kb_rir_d(int n, int p, double L, double s, double m) {
    return kb_rir_add(kb_rir_add(kb_rir_mul(2.0 * n, L), p ? -s : s), -m);
}

// The n with |(2 n) L + (1 - 2 p) s - m| <= R for p = 0 or 1, widened by one step each way so that no rounding in
// the bound can drop an image (the exact test is on tau).  lo > hi when there is none.
KB_HD void kb_rir_nrange(double L, double s, double m, double lo_d, double hi_d, int* lo, int* hi) {
    *lo = (int)floor((lo_d + m - s) / (2.0 * L)) - 1;
    *hi = (int)ceil((hi_d + m + s) / (2.0 * L)) + 1;
}

KB_HD double kb_rir_powi(double b, int n) {
    double r = 1.0;
    while (n > 0) {
        if (n & 1) r *= b;
        b *= b;
        n >>= 1;
    }
    return r;
}

KB_HD int kb_rir_iabs(int v) { return v < 0 ? -v : v; }

// Exact integer jj as a float (|jj| < 2^22): on the device without an I2F conversion.
KB_HD float kb_rir_i2f(int v) {
#if defined(__CUDA_ARCH__)
    return __fsub_rn(__int_as_float(0x4B400000 + v), 12582912.0f);
#else
    return (float)v;
#endif
}

KB_HD float kb_rir_rcp(float d) {
#if defined(__CUDA_ARCH__)
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(d));
    return r;
#else
    return 1.0f / d;
#endif
}

// Geometry of one tile, the same in every thread.
struct KbRirTile {
    const double* rec;
    double mx, my, mz, rlo2, rhi2, rhi;
    int nlo, nhi;                          // floor(tau) range whose taps reach the tile
    int max_order, nx0, nrows;
};

// The images of column (nx, px, ny, py) in enumeration order: calls f(nx, px, ny, py, nz, pz, floor(tau), tau, r) for
// each image that reaches the tile and passes the order filter.  Returns their count.
template <typename F>
KB_HD int kb_rir_column(const KbRirParams& p, const KbRirTile& T, int nx, int px, int ny, int py, F f) {
    const double* R = T.rec;
    const double dx = kb_rir_d(nx, px, R[0], R[3], T.mx), dy = kb_rir_d(ny, py, R[1], R[4], T.my);
    const double q = kb_rir_add(kb_rir_mul(dx, dx), kb_rir_mul(dy, dy));
    if (q > T.rhi2) return 0;
    const double zhi = sqrt(T.rhi2 - q), zlo = q < T.rlo2 ? sqrt(T.rlo2 - q) : 0.0;
    int a0, a1, b0, b1;
    kb_rir_nrange(R[2], R[5], T.mz, -zhi, -zlo, &a0, &a1);
    kb_rir_nrange(R[2], R[5], T.mz, zlo, zhi, &b0, &b1);
    if (a1 >= b0 - 1) { a1 = b1; b0 = b1 + 1; }         // the caps' ranges meet: one range
    const int ox = kb_rir_iabs(nx - px) + kb_rir_iabs(nx), oy = kb_rir_iabs(ny - py) + kb_rir_iabs(ny);
    int count = 0;
    for (int part = 0; part < 2; ++part) {
        const int n_lo = part ? b0 : a0, n_hi = part ? b1 : a1;
        for (int nz = n_lo; nz <= n_hi; ++nz)
            for (int pz = 0; pz < 2; ++pz) {
                const int order = ox + oy + kb_rir_iabs(nz - pz) + kb_rir_iabs(nz);
                if (T.max_order >= 0 && order > T.max_order) continue;
                const double dz = kb_rir_d(nz, pz, R[2], R[5], T.mz);
                const double r = kb_rir_sqrt(kb_rir_add(q, kb_rir_mul(dz, dz)));
                const double tau = kb_rir_div(kb_rir_mul(r, p.fs), p.c);
                const double fl = floor(tau);
                if (fl < (double)T.nlo || fl > (double)T.nhi) continue;
                ++count;
                f(nx, px, ny, py, nz, pz, (int)fl, tau, r);
            }
    }
    return count;
}

// Column ci of the row group: the row by bisection over the rows' inclusive column offsets, then (ny, py).
KB_HD void kb_rir_column_of(const KbRirTile& T, const int* cnt, const int* ny0, int nt, int rbase, int ci, int* nx,
                            int* px, int* ny, int* py) {
    int lo = 0, hi = nt - 1;
    while (lo < hi) {
        const int md = (lo + hi) >> 1;
        if (cnt[md] > ci) hi = md; else lo = md + 1;
    }
    const int loc = ci - (lo ? cnt[lo - 1] : 0);
    *nx = T.nx0 + ((rbase + lo) >> 1);
    *px = (rbase + lo) & 1;
    *ny = ny0[lo] + (loc >> 1);
    *py = loc & 1;
}

// The staged record of one image (see the top of the file).
KB_HD KbRirImg kb_rir_image(const KbRirParams& p, const double* R, int nx, int px, int ny, int py, int nz, int pz,
                            int fl, double tau, double r) {
    const double pi = 3.14159265358979323846;
    const double g = kb_rir_powi(R[6], kb_rir_iabs(nx - px)) * kb_rir_powi(R[7], kb_rir_iabs(nx)) *
                     kb_rir_powi(R[8], kb_rir_iabs(ny - py)) * kb_rir_powi(R[9], kb_rir_iabs(ny)) *
                     kb_rir_powi(R[10], kb_rir_iabs(nz - pz)) * kb_rir_powi(R[11], kb_rir_iabs(nz)) / (4.0 * pi * r);
    const double f = tau - fl;                           // exact
    const int up = f >= 0.5 ? 1 : 0;
    const double e = f - up;                             // exact, in [-1/2, 1/2)
#if defined(__CUDA_ARCH__)
    const double s = sinpi(e);
#else
    const double s = std::sin(pi * e);
#endif
    const double A = e == 0.0 ? -g : g * s / pi;         // e = 0: the tap g w[half] = (-g) ws[half]
    KbRirImg m;
    m.n0 = fl;
    m.nch = fl + up + (p.W - 1) / 2;
    m.e = (float)e;
    m.A = (float)(up ? -A : A);
    return m;
}

KB_HD float kb_rir_fmul(float a, float b) {
#if defined(__CUDA_ARCH__)
    return __fmul_rn(a, b);
#else
    return a * b;
#endif
}

// Inclusive prefix sum of a[0 .. nt) in place (Hillis-Steele through tmp).
KB_RIR_FN void kb_rir_scan(int* a, int* tmp, int nt) {
    for (int d = 1; d < nt; d <<= 1) {
        KB_RIR_THREADS { tmp[tid] = a[tid] + (tid >= d ? a[tid - d] : 0); }
        KB_RIR_SYNC;
        KB_RIR_THREADS { a[tid] = tmp[tid]; }
        KB_RIR_SYNC;
    }
}

// Row r of the group: (nx, px) and the range of its columns (ny, py).  Returns the column count.
KB_HD int kb_rir_row(const KbRirTile& T, int r, int* ny0) {
    const double* R = T.rec;
    const int nx = T.nx0 + (r >> 1), px = r & 1;
    const double dx = kb_rir_d(nx, px, R[0], R[3], T.mx);
    const double dx2 = kb_rir_mul(dx, dx);
    if (dx2 > T.rhi2) return 0;
    const double rho = sqrt(T.rhi2 - dx2);
    int lo, hi;
    kb_rir_nrange(R[1], R[4], T.my, -rho, rho, &lo, &hi);
    *ny0 = lo;
    return 2 * (hi - lo + 1);
}

KB_RIR_FN void kb_rir_tile(const KbRirParams& p, char* smem, long long tile) {
    const int nt = 32 * p.nw;
    const KbRirSmem S = kb_rir_smem(nt);
    KbRirImg* img = reinterpret_cast<KbRirImg*>(smem + S.img);
    float* ws = reinterpret_cast<float*>(smem + S.ws);
    float* acc = reinterpret_cast<float*>(smem + S.acc);
    int* cnt = reinterpret_cast<int*>(smem + S.cnt);
    int* tmp = reinterpret_cast<int*>(smem + S.tmp);
    int* ny0 = reinterpret_cast<int*>(smem + S.ny0);

    const long long col = tile / p.n_tt;
    const int tt = (int)(tile - col * p.n_tt);
    const long long b = col / p.M;
    const int mi = (int)(col - b * p.M);
    KbRirTile T;
    T.rec = p.rec + b * KB_RIR_REC;
    const double* mic = p.mic + (b * p.M + mi) * 3;
    T.mx = mic[0]; T.my = mic[1]; T.mz = mic[2];
    T.max_order = (int)T.rec[12];
    const int start = (int)T.rec[13];
    const int t0 = tt * nt;
    const int a0 = start + t0;
    const int a1 = start + (t0 + nt < p.L ? t0 + nt : p.L);        // absolute samples [a0, a1)
    T.nlo = a0 - p.W + 1;
    T.nhi = a1 - 1;
    // the shell's radii, widened by a part in 1e9 (the exact test is on tau)
    const double rlo = T.nlo > 0 ? (double)T.nlo * p.c / p.fs * (1.0 - 1e-9) : 0.0;
    T.rhi = (double)a1 * p.c / p.fs * (1.0 + 1e-9);
    T.rlo2 = rlo * rlo;
    T.rhi2 = T.rhi * T.rhi;
    int nx1;
    kb_rir_nrange(T.rec[0], T.rec[3], T.mx, -T.rhi, T.rhi, &T.nx0, &nx1);
    T.nrows = 2 * (nx1 - T.nx0 + 1);

    KB_RIR_THREADS {
        acc[tid] = 0.0f;
        for (int k = tid; k < p.W; k += nt) ws[k] = p.ws[k];
    }
    KB_RIR_SYNC;
    for (int rbase = 0; rbase < T.nrows; rbase += nt) {
        // rows of this group: column counts, scanned
        KB_RIR_THREADS {
            int n0 = 0;
            cnt[tid] = rbase + tid < T.nrows ? kb_rir_row(T, rbase + tid, &n0) : 0;
            ny0[tid] = n0;
        }
        KB_RIR_SYNC;
        kb_rir_scan(cnt, tmp, nt);
        const int ncols = cnt[nt - 1];
        for (int cbase = 0; cbase < ncols; cbase += nt) {
            // image counts of the batch's columns (one per thread), scanned in the chunk's first 2 nt ints: the chunk
            // is not in use between walks
            int* iscr = reinterpret_cast<int*>(img);
            KB_RIR_THREADS {
                const int ci = cbase + tid;
                int n = 0;
                if (ci < ncols) {
                    int nx, px, ny, py;
                    kb_rir_column_of(T, cnt, ny0, nt, rbase, ci, &nx, &px, &ny, &py);
                    n = kb_rir_column(p, T, nx, px, ny, py, [](int, int, int, int, int, int, int, double, double) {});
                }
                iscr[nt + tid] = n;
            }
            KB_RIR_SYNC;
            kb_rir_scan(iscr + nt, iscr, nt);
            KB_RIR_THREADS { tmp[tid] = iscr[nt + tid]; }      // inclusive image offsets of the batch's columns
            KB_RIR_SYNC;
            const int total = tmp[nt - 1];
            for (int base = 0; base < total; base += KB_RIR_CAP) {
                const int n_img = total - base < KB_RIR_CAP ? total - base : KB_RIR_CAP;
                KB_RIR_SYNC;
                // write the images of [base, base + n_img) into the chunk, in enumeration order
                KB_RIR_THREADS {
                    const int ci = cbase + tid;
                    const int end = tmp[tid], beg = tid ? tmp[tid - 1] : 0;
                    if (ci < ncols && end > base && beg < base + n_img) {
                        int nx, px, ny, py;
                        kb_rir_column_of(T, cnt, ny0, nt, rbase, ci, &nx, &px, &ny, &py);
                        int j = beg;
                        kb_rir_column(p, T, nx, px, ny, py,
                                      [&](int ax, int apx, int ay, int apy, int az, int apz, int fl, double tau,
                                          double r) {
                                          const int idx = j++ - base;
                                          if (idx >= 0 && idx < n_img)
                                              img[idx] = kb_rir_image(p, T.rec, ax, apx, ay, apy, az, apz, fl, tau, r);
                                      });
                    }
                }
                KB_RIR_SYNC;
                // every thread adds the taps of the chunk's images on its sample, in chunk order
                KB_RIR_THREADS {
                    const int ta = a0 + tid;
                    const int wlo = a0 + (tid & ~31);              // the warp's first sample
                    float v = acc[tid];
                    for (int i = 0; i < n_img; ++i) {
                        const KbRirImg m = img[i];
                        if ((unsigned)(m.n0 - (wlo - p.W + 1)) >= (unsigned)(p.W + 31)) continue;   // misses the warp
                        const int k = ta - m.n0;
                        if ((unsigned)k >= (unsigned)p.W) continue;
                        const int jj = ta - m.nch;
                        if (m.e == 0.0f && jj != 0) continue;
                        const float d = m.e == 0.0f ? 1.0f : kb_sub(kb_rir_i2f(jj), m.e);
                        v = kb_add(v, kb_rir_fmul(kb_rir_fmul(m.A, ws[k]), kb_rir_rcp(d)));
                    }
                    acc[tid] = v;
                }
            }
            KB_RIR_SYNC;
        }
        KB_RIR_SYNC;
    }
    KB_RIR_THREADS {
        const int t = t0 + tid;
        if (t < p.L) p.out[b * p.o_sb + (long long)mi * p.o_sm + (long long)t * p.o_st] = acc[tid];
    }
}
