// Kernel bodies of the Griffin-Lim element passes (kapre_griffin_lim in kapre_b200.cu drives the loop):
//   init:     X = S A_0,  A_0 = 1 or exp(2 pi i u(seed, i))
//   project:  A = Y - beta Yprev (A = Y without Yprev),  X = S A / (|A| + 1e-16)   (0 where A = 0)
// S is the magnitude spectrogram, read through its (batch, channel, frame, bin) element strides; X, Y and Yprev are
// the contiguous (B, C, T, F) complex64 buffers of the workspace, so an element's flat index i is its canonical
// index ((b C + c) T + t) F + f.  X may be the same buffer as Yprev: each element is read, then written, by one
// thread.
//
// Random init: u(seed, i) = (mix(seed ^ mix(i)) >> 40) 2^-24, the top 24 bits of a 64-bit hash scaled to [0, 1), with
// mix the splitmix64 step
//   z += 0x9E3779B97F4A7C15;  z = (z ^ (z >> 30)) 0xBF58476D1CE4E5B9;  z = (z ^ (z >> 27)) 0x94D049BB133111EB;  z ^ (z >> 31)
// in uint64 arithmetic.  Because i is canonical, the phases do not depend on the data format or strides of S.
//
// Like the other bodies these are barrier-free per-element functions: the CUDA wrappers call them in a grid-stride
// loop, the CPU emulation (tests/emu, KB_HOST_EMU) calls them for every index in turn.
#pragma once
#include "stft_core.cuh"

#define KB_GL_THREADS 256
#define KB_GL_INIT_ONES 0      // = KAPRE_GL_INIT_ONES
#define KB_GL_INIT_RANDOM 1    // = KAPRE_GL_INIT_RANDOM

struct KbGlParams {
    const float* S;  long long s_sb, s_sc, s_st, s_sf;
    int C, T, F;
    long long n;               // B C T F
    float2* X;                 // output: the next spectrum estimate
    const float2* Y;           // project: STFT of this iteration's waveform
    const float2* Yprev;       // project: the previous iteration's STFT, or null (first iteration, or beta = 0)
    float beta;                // momentum / (1 + momentum)
    int init;                  // KB_GL_INIT_*
    unsigned long long seed;
};

KB_HD unsigned long long kb_gl_mix(unsigned long long z) {
    z += 0x9E3779B97F4A7C15ULL;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
    return z ^ (z >> 31);
}

KB_HD float kb_gl_u(unsigned long long seed, long long i) {
    return (float)(kb_gl_mix(seed ^ kb_gl_mix((unsigned long long)i)) >> 40) * 0x1p-24f;
}

// (sin, cos) of 2 pi u.  2u is exact in float32; the device computes sin / cos of pi * 2u correctly rounded to about
// an ulp, the emulation in double precision.
#if defined(KB_HOST_EMU)
inline void kb_gl_phasor(float u, float* s, float* c) {
    const double a = 3.14159265358979323846 * (double)(2.0f * u);
    *s = (float)std::sin(a);
    *c = (float)std::cos(a);
}
#else
KB_D void kb_gl_phasor(float u, float* s, float* c) { sincospif(2.0f * u, s, c); }
#endif

// Element offset in S of canonical index i; 32-bit divisions while the index fits.
KB_FN long long kb_gl_s_off(const KbGlParams& p, long long i) {
    long long b, c, t, f;
    if (p.n <= 0xffffffffLL) {
        unsigned r = (unsigned)i;
        const unsigned F = (unsigned)p.F, T = (unsigned)p.T, C = (unsigned)p.C;
        f = r % F; r /= F;
        t = r % T; r /= T;
        c = r % C; b = r / C;
    } else {
        long long r = i;
        f = r % p.F; r /= p.F;
        t = r % p.T; r /= p.T;
        c = r % p.C; b = r / p.C;
    }
    return b * p.s_sb + c * p.s_sc + t * p.s_st + f * p.s_sf;
}

KB_FN void kb_gl_init_elem(const KbGlParams& p, long long i) {
    const float s = p.S[kb_gl_s_off(p, i)];
    float re = s, im = 0.0f;
    if (p.init == KB_GL_INIT_RANDOM) {
        float sn, cs;
        kb_gl_phasor(kb_gl_u(p.seed, i), &sn, &cs);
        re = s * cs;
        im = s * sn;
    }
    p.X[i] = make_float2(re, im);
}

KB_FN void kb_gl_project_elem(const KbGlParams& p, long long i) {
    float2 a = p.Y[i];
    if (p.Yprev) {
        const float2 q = p.Yprev[i];
        a.x = fmaf(-p.beta, q.x, a.x);
        a.y = fmaf(-p.beta, q.y, a.y);
    }
    const float g = p.S[kb_gl_s_off(p, i)] / (sqrtf(fmaf(a.x, a.x, a.y * a.y)) + 1e-16f);
    p.X[i] = make_float2(a.x * g, a.y * g);
}
