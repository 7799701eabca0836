// Register-resident FFT of compile-time size R in {2,4,8,16,32}: radix-4 passes, plus one radix-2 pass first
// when log2(R) is odd.  Fully unrolled: every index is a compile-time constant after unrolling, so the array lives
// in registers on the GPU.  Forward transform (kernel exp(-2 pi i jk/R)); the input is in natural order and the
// result for frequency k is left at position kb_brev<R>(k) (bit-reversed order).
//
// The passes are the decimation-in-time butterflies (a, b) -> (a + w b, a - w b), which put the twiddle on a
// butterfly input so that it contracts into the additions: with w = c - i s and |c| >= |s|,
//     w b = c u,  u = (b.re + (s/c) b.im, b.im - (s/c) b.re),   a +- w b = fma(+-c, u, a)
// (and the mirror form with c/s when |s| > |c|): 6 FP32 instructions per twiddled butterfly instead of the 8 of a
// rounded complex product followed by two complex additions.  w = 1 and w = -i cost 4 additions.  The value at
// position p of the textbook bit-reversed-input DIT network is kept in v[kb_brev<R>(p)], which makes the input
// natural-order and the output bit-reversed.  kb_fft<R, H> runs the passes from butterfly half-size H on, so a caller
// may do the first radix-2 pass itself (kb_col_window_dft32 fuses the window into it).
#pragma once
#include "kb_common.h"

// cos(2 pi t / 32), t = 0..16
KB_HD constexpr float kb_cos32_q(int t) {
    return t == 0 ? 1.0f
         : t == 1 ? 0.98078528040323044913f
         : t == 2 ? 0.92387953251128675613f
         : t == 3 ? 0.83146961230254523708f
         : t == 4 ? 0.70710678118654752440f
         : t == 5 ? 0.55557023301960222474f
         : t == 6 ? 0.38268343236508977173f
         : t == 7 ? 0.19509032201612826785f
         : 0.0f;
}
KB_HD constexpr float kb_cos32(int t) { return t <= 8 ? kb_cos32_q(t) : -kb_cos32_q(16 - t); }
KB_HD constexpr float kb_sin32(int t) { return t <= 8 ? kb_cos32_q(8 - t) : kb_cos32_q(t - 8); }
// tan(2 pi t / 32), t = 1..3 (the ratio s/c of the twiddles with |c| > |s|; the others reduce to these by symmetry)
KB_HD constexpr float kb_tan32(int t) {
    return t == 1 ? 0.19891236737965800691f
         : t == 2 ? 0.41421356237309504880f
         : 0.66817863791929891999f;
}

template <int R>
KB_HD constexpr int kb_brev(int k) {
    int r = 0;
    for (int b = 1; b < R; b <<= 1) {
        r = (r << 1) | (k & 1);
        k >>= 1;
    }
    return r;
}

// (a, b) <- (a + w b, a - w b), w = exp(-2 pi i t / 32), t in [0, 16).  `t` is a compile-time constant after
// unrolling, so the branch chain folds away.
KB_HD void kb_bfly32(cpx& a, cpx& b, int t) {
    if (t == 0) {
        const cpx s = cadd(a, b), d = csub(a, b);
        a = s; b = d;
        return;
    }
    if (t == 8) {   // w b = -i b = (b.im, -b.re)
        const cpx s = cmake(kb_add(a.re, b.im), kb_sub(a.im, b.re)), d = cmake(kb_sub(a.re, b.im), kb_add(a.im, b.re));
        a = s; b = d;
        return;
    }
    cpx u;
    float m;
    if (t == 4 || t == 12) {   // w = (-+1 - i)/sqrt2 = m (1 -+ i) with m = cos: u = (b.re +- b.im, b.im -+ b.re)
        u = t == 4 ? cmake(kb_add(b.re, b.im), kb_sub(b.im, b.re)) : cmake(kb_sub(b.re, b.im), kb_add(b.im, b.re));
        m = kb_cos32(t);
    } else if (t < 4 || t > 12) {   // |c| > |s|: w b = c (b.re + r b.im, b.im - r b.re), r = s / c
        const float r = t < 4 ? kb_tan32(t) : -kb_tan32(16 - t);
        u = cmake(kb_fma(r, b.im, b.re), kb_fma(-r, b.re, b.im));
        m = kb_cos32(t);
    } else {                        // |s| > |c|: w b = s (r b.re + b.im, r b.im - b.re), r = c / s
        const float r = t < 8 ? kb_tan32(8 - t) : -kb_tan32(t - 8);
        u = cmake(kb_fma(r, b.re, b.im), kb_fma(r, b.im, -b.re));
        m = kb_sin32(t);
    }
    const cpx s = cmake(kb_fma(m, u.re, a.re), kb_fma(m, u.im, a.im));
    const cpx d = cmake(kb_fma(-m, u.re, a.re), kb_fma(-m, u.im, a.im));
    a = s; b = d;
}

// The passes from butterfly half-size H on: radix-4 over (H, 2H), or radix-2 at H when log2(R / H) is odd.  A
// radix-4 butterfly of size 4H at offset j < H is the four radix-2 butterflies of its two stages, with twiddles
// W_2H^j (twice) and W_4H^j, W_4H^(j + H) = -i W_4H^j.
template <int R, int H = 1>
KB_HD void kb_fft(cpx* v) {
    static_assert(R == 2 || R == 4 || R == 8 || R == 16 || R == 32, "unsupported size");
    if constexpr (H < R) {
        if constexpr (R / H == 2 || R / H == 8 || R / H == 32) {
#pragma unroll
            for (int b0 = 0; b0 < R; b0 += 2 * H) {
#pragma unroll
                for (int j = 0; j < H; ++j)
                    kb_bfly32(v[kb_brev<R>(b0 + j)], v[kb_brev<R>(b0 + j + H)], j * (16 / H));
            }
            kb_fft<R, 2 * H>(v);
        } else {
#pragma unroll
            for (int b0 = 0; b0 < R; b0 += 4 * H) {
#pragma unroll
                for (int j = 0; j < H; ++j) {
                    cpx& x0 = v[kb_brev<R>(b0 + j)];
                    cpx& x1 = v[kb_brev<R>(b0 + j + H)];
                    cpx& x2 = v[kb_brev<R>(b0 + j + 2 * H)];
                    cpx& x3 = v[kb_brev<R>(b0 + j + 3 * H)];
                    kb_bfly32(x0, x1, j * (16 / H));
                    kb_bfly32(x2, x3, j * (16 / H));
                    kb_bfly32(x0, x2, j * (8 / H));
                    kb_bfly32(x1, x3, j * (8 / H) + 8);
                }
            }
            kb_fft<R, 4 * H>(v);
        }
    }
}
