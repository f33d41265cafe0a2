// First-stage decoder (AutoencoderKL.decode, ldm/models/autoencoder.py:33-37; Decoder, ldm/modules/
// diffusionmodules/model.py:462-569) -- the pieces that are not idiff_gemm / idiff_groupnorm calls:
//   * latent prologue: z / scale_factor, post_quant_conv (1x1, 4 -> 4), fp32 NCHW -> fp16 NHWC padded to
//     the 64-channel granularity of the conv3x3 kernel's A operand;
//   * row softmax of the single-head mid-block attention (AttnBlock, model.py:150-202): the scores of one
//     image are a [HW, HW] GEMM output (head_dim 512 does not fit the flash kernels' register tiles and the
//     block runs once per image), normalised in place;
//   * image epilogue: the decoder's NCHW output to the uint8 NHWC bytes the reference saves (inference.py:122-125);
//   * encoder epilogue: quant_conv and the seeded sample of the posterior (autoencoder.py:27-31) in one pass.
#include "../../include/idiff_b200.h"
#include "common.cuh"
#include "host.cuh"

namespace idiff {

// grid-stride over pixels; one thread per (pixel): reads C_in <= 8 planes, writes one 128-byte row
__global__ void __launch_bounds__(256)
vae_latent_in_kernel(const float* __restrict__ z, const float* __restrict__ w, const float* __restrict__ bias,
                     float inv_scale, uint4* __restrict__ out, int B, int C, int HW) {
  __shared__ float sw[64], sb[8];
  if (threadIdx.x < C * C) sw[threadIdx.x] = w[threadIdx.x];
  if (threadIdx.x < C) sb[threadIdx.x] = bias[threadIdx.x];
  __syncthreads();
  const long total = (long)B * HW;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int b = (int)(i / HW);
    const int pix = (int)(i - (long)b * HW);
    float zi[8], o[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) zi[c] = (c < C) ? z[((long)b * C + c) * HW + pix] * inv_scale : 0.f;
#pragma unroll
    for (int co = 0; co < 8; ++co) {
      float a = 0.f;
      if (co < C) {
        a = sb[co];
#pragma unroll
        for (int ci = 0; ci < 8; ++ci)
          if (ci < C) a = fmaf(sw[co * C + ci], zi[ci], a);
      }
      o[co] = a;
    }
    uint4* row = out + i * 8;  // 64 halves = 8 x 16 bytes
    row[0] = make_uint4(pack_half2(o[0], o[1]), pack_half2(o[2], o[3]), pack_half2(o[4], o[5]), pack_half2(o[6], o[7]));
    const uint4 zero = make_uint4(0, 0, 0, 0);
#pragma unroll
    for (int q = 1; q < 8; ++q) row[q] = zero;
  }
}

// one CTA per row; the row lives in shared memory as fp32 between the passes
__global__ void __launch_bounds__(256)
softmax_rows_kernel(h16* __restrict__ x, int n, long ld) {
  extern __shared__ float srow[];
  __shared__ float red[8];
  h16* row = x + (long)blockIdx.x * ld;
  const int nv = n >> 3;  // n % 8 == 0
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float m = -INFINITY;
  for (int v = threadIdx.x; v < nv; v += blockDim.x) {
    const uint4 u = reinterpret_cast<const uint4*>(row)[v];
    const uint32_t uu[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = unpack_half2(uu[j]);
      srow[v * 8 + 2 * j] = f.x;
      srow[v * 8 + 2 * j + 1] = f.y;
      m = fmaxf(m, fmaxf(f.x, f.y));
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if (lane == 0) red[warp] = m;
  __syncthreads();
  m = red[0];
#pragma unroll
  for (int i = 1; i < 8; ++i) m = fmaxf(m, red[i]);
  __syncthreads();
  float s = 0.f;
  for (int v = threadIdx.x; v < nv; v += blockDim.x) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float e = exp2_approx((srow[v * 8 + j] - m) * 1.4426950408889634f);
      srow[v * 8 + j] = e;
      s += e;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) red[warp] = s;
  __syncthreads();
  s = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) s += red[i];  // fixed order
  const float inv = 1.0f / s;
  for (int v = threadIdx.x; v < nv; v += blockDim.x) {
    uint32_t o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) o[j] = pack_half2(srow[v * 8 + 2 * j] * inv, srow[v * 8 + 2 * j + 1] * inv);
    reinterpret_cast<uint4*>(row)[v] = make_uint4(o[0], o[1], o[2], o[3]);
  }
}

// inference.py:122-125 for one value: torch.clamp(x, -1, 1) * 0.5 + 0.5 on the device, then * 255 and
// astype(np.uint8) in numpy, all fp32.  x * 0.5 is exact, so one fma rounds like the reference's mul + add; the
// conversion truncates toward zero like the C cast numpy uses.  NaN clamps to -1 (fmaxf returns the other operand).
IDIFF_DEVICE uint32_t image_byte(float x) {
  const float c = fminf(fmaxf(x, -1.f), 1.f);
  return __float2uint_rz(__fmul_rn(__fmaf_rn(c, 0.5f, 0.5f), 255.f));
}

IDIFF_DEVICE float load_f(const float* p) { return *p; }
IDIFF_DEVICE float load_f(const h16* p) { return h2f(*p); }

// four consecutive pixels of one channel plane: one 16-byte (fp32) or 8-byte (16-bit) load
IDIFF_DEVICE void load4(const float* p, float v[4]) {
  const float4 u = *reinterpret_cast<const float4*>(p);
  v[0] = u.x, v[1] = u.y, v[2] = u.z, v[3] = u.w;
}
IDIFF_DEVICE void load4(const h16* p, float v[4]) {
  const uint2 u = *reinterpret_cast<const uint2*>(p);
  const float2 a = unpack_half2(u.x), b = unpack_half2(u.y);
  v[0] = a.x, v[1] = a.y, v[2] = b.x, v[3] = b.y;
}

// One thread per group of four pixels of one image: the three channel planes in (NCHW), the 12 bytes of those pixels
// out (NHWC), which are three aligned 32-bit words.  VEC (HW % 4 == 0): every group is whole and its loads and stores
// are aligned; otherwise the last group of an image may be partial and everything goes element by element.
template <typename T, bool VEC>
__global__ void __launch_bounds__(256)
decode_to_image_kernel(const T* __restrict__ x, uint8_t* __restrict__ out, int B, long HW) {
  constexpr int C = 3;
  const long groups = (HW + 3) / 4;
  const long total = (long)B * groups;
  for (long g = (long)blockIdx.x * blockDim.x + threadIdx.x; g < total; g += (long)gridDim.x * blockDim.x) {
    const long b = g / groups;
    const long p0 = (g - b * groups) * 4;
    const T* src = x + b * C * HW + p0;
    uint8_t* dst = out + (b * HW + p0) * C;
    if (VEC) {
      uint32_t w[C] = {0u, 0u, 0u};  // byte k of the group's output is channel k % 3 of pixel k / 3
#pragma unroll
      for (int c = 0; c < C; ++c) {
        float v[4];
        load4(src + c * HW, v);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int k = j * C + c;
          w[k >> 2] |= image_byte(v[j]) << (8 * (k & 3));
        }
      }
#pragma unroll
      for (int q = 0; q < C; ++q) reinterpret_cast<uint32_t*>(dst)[q] = w[q];
    } else {
      const int n = (int)(HW - p0 < 4 ? HW - p0 : 4);
      for (int j = 0; j < n; ++j)
        for (int c = 0; c < C; ++c) dst[j * C + c] = (uint8_t)image_byte(load_f(src + c * HW + j));
    }
  }
}

// One thread per latent channel c of a group of four pixels p0 .. p0+3 of one image: the eight conv_out planes of those
// pixels in, the mean and logvar rows of quant_conv (1x1, 8 -> 8, fp32 FMAs in input-channel order), the posterior
// sample out.  The noise of element e = c*hw + p of image b is normal e % 4 of group e / 4 of stream kNoisePosterior
// with key seeds[b] and word 2 = index[b] (normals4), so it depends on (seed, index, e) alone; with hw % 4 == 0 one draw
// serves the thread's four pixels.
__global__ void __launch_bounds__(256)
encode_posterior_kernel(const float* __restrict__ h, const float* __restrict__ w, const float* __restrict__ bias,
                        float scale, const unsigned long long* __restrict__ seeds, const int* __restrict__ index,
                        float* __restrict__ z, int B, long hw) {
  constexpr int ZC = 4, MC = 2 * ZC;
  __shared__ float sw[MC * MC], sb[MC];
  if (threadIdx.x < MC * MC) sw[threadIdx.x] = w[threadIdx.x];
  if (threadIdx.x < MC) sb[threadIdx.x] = bias[threadIdx.x];
  __syncthreads();
  const long groups = (hw + 3) / 4;
  const long total = (long)B * ZC * groups;
  for (long g = (long)blockIdx.x * blockDim.x + threadIdx.x; g < total; g += (long)gridDim.x * blockDim.x) {
    const long bc = g / groups;
    const int b = (int)(bc / ZC), c = (int)(bc - (long)b * ZC);
    const long p0 = (g - bc * groups) * 4;
    const int n = (int)(hw - p0 < 4 ? hw - p0 : 4);
    const float* hb = h + (long)b * MC * hw + p0;
    float mean[4], logvar[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) mean[j] = sb[c], logvar[j] = sb[c + ZC];
#pragma unroll
    for (int k = 0; k < MC; ++k) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float v = j < n ? hb[k * hw + j] : 0.f;
        mean[j] = fmaf(sw[c * MC + k], v, mean[j]);
        logvar[j] = fmaf(sw[(c + ZC) * MC + k], v, logvar[j]);
      }
    }
    const uint2 key = philox_key(seeds[b]);
    const uint32_t idx = (uint32_t)index[b];
    float* zb = z + ((long)b * ZC + c) * hw + p0;
    long cached = -1;
    float eps4[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (j >= n) break;
      const long e = c * hw + p0 + j;
      if ((e >> 2) != cached) {
        cached = e >> 2;
        normals4(key, cached, idx, kNoisePosterior, eps4);
      }
      const int q = (int)(e & 3);  // selected, not indexed, so eps4 stays in registers
      const float eps = q == 0 ? eps4[0] : q == 1 ? eps4[1] : q == 2 ? eps4[2] : eps4[3];
      // distributions.py:26-36 then autoencoder.py:31, each operation rounded on its own like the torch expressions
      const float stdv = expf(__fmul_rn(0.5f, fminf(fmaxf(logvar[j], -30.f), 20.f)));
      zb[j] = __fmul_rn(__fadd_rn(mean[j], __fmul_rn(stdv, eps)), scale);
    }
  }
}

}  // namespace idiff

extern "C" int idiff_vae_latent_in(const float* z, const float* w, const float* bias, float inv_scale, void* out,
                                   int batch, int channels, int hw, void* stream) {
  using namespace idiff;
  IDIFF_REQUIRE(z && w && bias && out, "idiff_vae_latent_in: null pointer argument");
  IDIFF_REQUIRE(channels >= 1 && channels <= 8, "idiff_vae_latent_in: 1..8 latent channels supported (got %d)", channels);
  IDIFF_REQUIRE(batch > 0 && hw > 0, "idiff_vae_latent_in: bad shape (batch %d, hw %d)", batch, hw);
  const long total = (long)batch * hw;
  const int blocks = grid_for(total, 256, 8);
  IDIFF_CHECK_CUDA(launch(vae_latent_in_kernel, dim3(blocks), dim3(256), 0, reinterpret_cast<cudaStream_t>(stream), z, w,
                          bias, inv_scale, reinterpret_cast<uint4*>(out), batch, channels, hw));
  return 0;
}

extern "C" int idiff_softmax_rows(void* x, int rows, int n, long ld, void* stream) {
  using namespace idiff;
  IDIFF_REQUIRE(x && rows > 0, "idiff_softmax_rows: bad arguments");
  IDIFF_REQUIRE(n > 0 && n % 8 == 0 && n <= 40960, "idiff_softmax_rows: n=%d must be a multiple of 8, <= 40960", n);
  IDIFF_REQUIRE(ld % 8 == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0, "idiff_softmax_rows: rows must be 16B aligned");
  const size_t smem = (size_t)n * sizeof(float);
  static bool attr_set = false;
  if (!attr_set) {
    IDIFF_CHECK_CUDA(cudaFuncSetAttribute(softmax_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));
    attr_set = true;
  }
  IDIFF_CHECK_CUDA(launch(softmax_rows_kernel, dim3(rows), dim3(256), smem, reinterpret_cast<cudaStream_t>(stream),
                          reinterpret_cast<h16*>(x), n, ld));
  return 0;
}

extern "C" int idiff_decode_to_image(const void* x, int x_fp32, void* out, int batch, long hw, void* stream) {
  using namespace idiff;
  IDIFF_REQUIRE(x && out && batch > 0 && hw > 0, "idiff_decode_to_image: bad arguments");
  const bool vec = hw % 4 == 0 && (reinterpret_cast<uintptr_t>(x) & (x_fp32 ? 15 : 7)) == 0 &&
                   (reinterpret_cast<uintptr_t>(out) & 3) == 0;
  const long total = (long)batch * ((hw + 3) / 4);
  const int blocks = grid_for(total, 256, 16);
  const cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  uint8_t* o = reinterpret_cast<uint8_t*>(out);
  if (x_fp32) {
    const float* xf = reinterpret_cast<const float*>(x);
    IDIFF_CHECK_CUDA(vec ? launch(decode_to_image_kernel<float, true>, dim3(blocks), dim3(256), 0, s, xf, o, batch, hw)
                         : launch(decode_to_image_kernel<float, false>, dim3(blocks), dim3(256), 0, s, xf, o, batch, hw));
  } else {
    const h16* xh = reinterpret_cast<const h16*>(x);
    IDIFF_CHECK_CUDA(vec ? launch(decode_to_image_kernel<h16, true>, dim3(blocks), dim3(256), 0, s, xh, o, batch, hw)
                         : launch(decode_to_image_kernel<h16, false>, dim3(blocks), dim3(256), 0, s, xh, o, batch, hw));
  }
  return 0;
}

extern "C" int idiff_encode_posterior(const float* h, const float* w, const float* bias, float scale,
                                      const unsigned long long* seeds, const int* index, float* z, int batch, long hw,
                                      void* stream) {
  using namespace idiff;
  IDIFF_REQUIRE(h && w && bias && seeds && index && z, "idiff_encode_posterior: null pointer argument");
  IDIFF_REQUIRE(batch > 0 && hw > 0, "idiff_encode_posterior: bad shape (batch %d, hw %ld)", batch, hw);
  const long total = (long)batch * 4 * ((hw + 3) / 4);
  const int blocks = grid_for(total, 256, 16);
  IDIFF_CHECK_CUDA(launch(encode_posterior_kernel, dim3(blocks), dim3(256), 0, reinterpret_cast<cudaStream_t>(stream),
                          h, w, bias, scale, seeds, index, z, batch, hw));
  return 0;
}
