// Window arithmetic of the streaming pose-graph tracker (loader.cu, mapnet_track_*), shared by its CUDA kernels and
// the host-only test shim (tests/_hosttrack.cpp).
//
// The window of frame c is scripts/eval.py's MF(steps=T, skip, real=True, include_vos=True, no_duplicates=False)
// tuple (dataset_loaders/composite.py:60-75, data/tuples.py mf_indices): slot k holds frame
// clip(c + (k - T/2) * skip, 0, last), T/2 in py2 integer division, and eval.py keeps slot T/2.  The last slot is
// `lag` = (T - 1 - T/2) * skip frames after c, so frame c's window is complete once frame c + lag has arrived, and until
// the sequence ends no slot of a complete window is clipped at `last`: a streamed window is the whole sequence's.  Its
// last slot T-1, optimised, is the zero-lag estimate of frame c + lag.
#pragma once

#if defined(__CUDACC__)
#define TRK_HD __host__ __device__ __forceinline__
#else
#define TRK_HD static inline
#endif

namespace trackcore {

TRK_HD long long lag(int T, int skip) { return (long long)(T - 1 - T / 2) * skip; }

// frames the device rings hold: one call's max_batch new frames plus the (T-1)*skip older ones its windows reach back to
TRK_HD long long ring_frames(int max_batch, int T, int skip) { return (long long)max_batch + (long long)(T - 1) * skip; }

// the frame of slot k of frame c's window in a sequence whose last frame is `last`
TRK_HD long long slot_frame(long long c, int k, int T, int skip, long long last) {
  const long long f = c + (long long)(k - T / 2) * skip;
  return f < 0 ? 0 : (f > last ? last : f);
}

// the first frame whose window is not complete after `seen` frames.  A call that brings `seen` to `seen + n` emits
// frames [first_pending(seen), first_pending(seen + n)); a flush emits [first_pending(seen), seen).
TRK_HD long long first_pending(long long seen, long long lag) { return seen > lag ? seen - lag : 0; }

// Zero-lag calls (mapnet_track_step_now) solve one window per new frame: the window whose last slot is that frame.
// Frame f's is frame (f - lag)'s window, so a call that brings `seen` to `seen + n` solves the windows of centres
// now_first(seen) .. now_first(seen) + n - 1.  A centre below 0 (the first lag frames of a sequence) is a window
// eval.py never builds; slot_frame clips its slots at 0.  From first_pending(seen) on they are the windows a step
// completes, so the first now_lead(seen, n) windows of the call feed only the zero-lag output.
TRK_HD long long now_first(long long seen, long long lag) { return seen - lag; }
TRK_HD long long now_lead(long long seen, long long n, long long lag) {
  return n - (first_pending(seen + n, lag) - first_pending(seen, lag));
}

// slot pair e of a window's VOs: consecutive slots (e, e+1), or with fc every pair i < j in row-major order
TRK_HD void vo_pair(int e, int T, int fc, int* i, int* j) {
  if (!fc) { *i = e; *j = e + 1; return; }
  int a = 0, rem = e;
  while (rem >= T - 1 - a) { rem -= T - 1 - a; ++a; }
  *i = a; *j = a + 1 + rem;
}

// a translation un-normalised as inference._window_errors does it: torch's float64 multiply, then its add, each
// rounded on its own (never a fused multiply-add)
TRK_HD double unnormalize(double t, double s, double m) {
#if defined(__CUDA_ARCH__)
  return __dadd_rn(__dmul_rn(t, s), m);
#else
  const double p = t * s;      // the host shim is compiled with -ffp-contract=off
  return p + m;
#endif
}

}  // namespace trackcore
