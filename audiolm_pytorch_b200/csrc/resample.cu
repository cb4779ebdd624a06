// Band-limited resampling (torchaudio.functional.resample with its defaults: Hann-windowed sinc, 6 zero crossings,
// rolloff 0.99), as called by the reference at soundstream.py:788, hubert_kmeans.py:102, vq_wav2vec.py:70 and
// encodec.py:105.
//
// With the rates reduced by their gcd to o -> n, output j = k n + p (phase p < n) is
//     y[j] = sum_{i < T} K[i, p] x[k o + off[p] + i]        (x = 0 outside [0, L))
// over the compact polyphase table the host builds once per (o, n) (audiolm_pytorch_b200/ops.py: resample_table): only
// the taps whose unclamped filter position lies strictly inside the +-6 zero crossings, T = the most any phase keeps,
// shorter phases padded with zeros.  The table is tap-major ([T, n]) so that the 32 consecutive outputs of a warp,
// which have consecutive phases, read one tap as one coalesced load.  Table and input both go through the read-only
// cache: see DESIGN.md ("Resampling") for the measurement behind that choice.
//
// One thread per output, taps summed in index order with fp32 FMAs and no atomics: a row's output is bitwise the same
// whether it is resampled alone or inside a batch, and whatever output window is asked for.
#include "alm_common.cuh"

namespace alm {
namespace resample {

constexpr int THREADS = 256;

__global__ void __launch_bounds__(THREADS)
resample_kernel(const float* __restrict__ x, long long ldx, long long L, float* __restrict__ y, long long start,
                long long count, int rows, const float* __restrict__ taps, const int* __restrict__ off, int T, int o,
                int n) {
  const long long c = (long long)blockIdx.x * THREADS + threadIdx.x;
  if (c >= count) return;
  const long long j = start + c;
  const long long k = j / n;
  const int p = (int)(j - k * n);
  const long long s = k * o + __ldg(off + p);
  const float* w = taps + p;
  for (int r = blockIdx.y; r < rows; r += gridDim.y) {
    const float* xr = x + (long long)r * ldx;
    float acc = 0.f;
    if (s >= 0 && s + T <= L) {
      const float* xs = xr + s;
#pragma unroll 4
      for (int i = 0; i < T; ++i) acc = fmaf(__ldg(w + (long long)i * n), __ldg(xs + i), acc);
    } else {
#pragma unroll 4
      for (int i = 0; i < T; ++i) {
        const long long q = s + i;
        const float v = (q >= 0 && q < L) ? __ldg(xr + q) : 0.f;
        acc = fmaf(__ldg(w + (long long)i * n), v, acc);
      }
    }
    y[(long long)r * count + c] = acc;
  }
}

}  // namespace resample
}  // namespace alm

extern "C" int alm_resample(const float* x, int64_t ldx, int64_t L, float* y, int64_t start, int64_t count, int rows,
                            const float* taps, const int* off, int T, int o, int n, alm_stream_t stream_) {
  ALM_REQUIRE(x && y && taps && off && rows > 0 && L > 0 && ldx >= L && T > 0 && o > 0 && n > 0, ALM_ERR_ARG);
  ALM_REQUIRE(start >= 0 && count >= 0, ALM_ERR_ARG);
  if (count == 0) return ALM_OK;
  const long long blocks = alm::ceil_div<long long>(count, alm::resample::THREADS);
  ALM_REQUIRE(blocks < (1LL << 31), ALM_ERR_ARG);
  const dim3 grid((unsigned)blocks, (unsigned)(rows < 65535 ? rows : 65535));
  alm::resample::resample_kernel<<<grid, alm::resample::THREADS, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      x, ldx, L, y, start, count, rows, taps, off, T, o, n);
  ALM_CHECK_LAUNCH();
  ALM_LAUNCHED(1);
  return ALM_OK;
}
