// render.cuh -- the frame rasteriser the env render kernels share (sm_90a): palette and geometry, filled disc / rectangle / line primitives,
// a 3x5 bitmap digit font, and the band loop that writes a frame's pixel rows.  Included by the env kernels (lbf_env.cu, rware_env.cu,
// matrix_env.cu).  Semantics: DESIGN.md
// §4.8; oracle: tests/render_ref.py.
//
// Integer arithmetic only, so that a numpy restatement reproduces every frame bit for bit.  A frame of a rows x cols board with g-pixel cells is
// H = 1 + rows*(g+1) by W = 1 + cols*(g+1) RGB pixels: 1-px black grid lines at every multiple of g+1, cell (row, col) covers the g x g pixels
// after them.  Shapes are placed in cell-local coordinates (lx, ly) in [0, g); a centre (cx, cy) is a point on the pixel grid (a pixel corner),
// and a pixel belongs to a disc when its centre (lx + 1/2, ly + 1/2) is within the radius, measured in half pixels.
#pragma once
#include "common.cuh"

namespace marl {
namespace render {

struct Rgb { uint8_t r, g, b; };

__device__ constexpr Rgb kWhite{255, 255, 255}, kBlack{0, 0, 0};

// ---- Level-Based Foraging (our own geometry and palette) ----
constexpr int kLbfCell = 50;                       // px per cell
constexpr int kLbfFoodR = 16, kLbfAgentR = 20;     // discs centred on the cell centre (25, 25)
constexpr int kLbfBadgeC = 37;                     // level badge: centre (37, 37), the cell's lower right
constexpr int kLbfBadgeR = 11, kLbfBadgeLine = 2;  // radius; outline width (black ring of radii 9..11)
__device__ constexpr Rgb kLbfFood{197, 58, 50}, kLbfAgent{46, 104, 190};

// ---- multi-robot warehouse (colours and sizes recalled from upstream's pyglet renderer; its sprites, fonts and anti-aliasing are not
// reproduced) ----
constexpr int kRwCell = 30;                        // px per cell (recalled)
constexpr int kRwShelfPad = 2;                     // shelf rectangle inset on every side (recalled)
constexpr int kRwAgentR = kRwCell / 3;             // agent disc radius, centred on the cell centre (15, 15) (recalled)
constexpr int kRwDirLine = 2;                      // direction line width, from the centre to the disc's edge
__device__ constexpr Rgb kRwGoal{60, 60, 60};                 // (recalled)
__device__ constexpr Rgb kRwShelf{72, 61, 139}, kRwShelfRequested{0, 128, 128};   // (recalled)
__device__ constexpr Rgb kRwAgent{255, 140, 0}, kRwAgentLoaded{255, 0, 0};        // (recalled)
__device__ constexpr Rgb kRwDir{0, 0, 0};                     // (recalled)

// ---- matrix games (our own: upstream has no rgb_array renderer): one row per player, one column per action ----
constexpr int kMxCell = 40;                        // px per cell
__device__ constexpr Rgb kMxChosen{46, 104, 190};  // fills the cell of each player's previous action

// ---- digits: 3x5 glyphs, bit 14 - (3*row + col) set for an inked pixel, drawn kFontScale px per glyph pixel, kDigitGap px apart ----
constexpr int kFontScale = 2, kDigitGap = 2;
static __constant__ uint16_t kFont[10] = {0x7b6f, 0x2c97, 0x73e7, 0x73cf, 0x5bc9, 0x79cf, 0x79ef, 0x7249, 0x7bef, 0x7bcf};

__host__ __device__ constexpr int frame_side(int cells, int g) { return 1 + cells * (g + 1); }

__device__ __forceinline__ bool in_disc(int lx, int ly, int cx, int cy, int r) {
  const int dx = 2 * (lx - cx) + 1, dy = 2 * (ly - cy) + 1;
  return dx * dx + dy * dy <= 4 * r * r;
}
__device__ __forceinline__ bool in_rect(int lx, int ly, int x0, int y0, int x1, int y1) { return lx >= x0 && lx < x1 && ly >= y0 && ly < y1; }
// Axis-parallel line from corner (x0, y0) to corner (x1, y1), w px wide and centred on it
__device__ __forceinline__ bool on_line(int lx, int ly, int x0, int y0, int x1, int y1, int w) {
  if (x0 == x1) return in_rect(lx, ly, x0 - w / 2, y0 < y1 ? y0 : y1, x0 - w / 2 + w, y0 < y1 ? y1 : y0);
  return in_rect(lx, ly, x0 < x1 ? x0 : x1, y0 - w / 2, x0 < x1 ? x1 : x0, y0 - w / 2 + w);
}
// Is (lx, ly) an inked pixel of `value` (0..999) written in decimal, the text box centred on corner (cx, cy)?
__device__ __forceinline__ bool in_number(int lx, int ly, int value, int cx, int cy) {
  const int nd = value >= 100 ? 3 : value >= 10 ? 2 : 1;
  const int dw = 3 * kFontScale, dh = 5 * kFontScale, tw = nd * dw + (nd - 1) * kDigitGap;
  const int tx = lx - (cx - tw / 2), ty = ly - (cy - dh / 2);
  if (tx < 0 || tx >= tw || ty < 0 || ty >= dh) return false;
  const int k = tx / (dw + kDigitGap), col = tx - k * (dw + kDigitGap);
  if (col >= dw) return false;
  int d = value;
  for (int i = nd - 1; i > k; --i) d /= 10;
  const int bit = (ty / kFontScale) * 3 + col / kFontScale;
  return (kFont[d % 10] >> (14 - bit)) & 1u;
}

// ---- frame bands: one CTA writes the whole pixel rows [y0, y1) of one frame ----
constexpr int kRenderThreads = 256;
constexpr int kBandBytes = 24576;   // staged pixel bytes per CTA; holds a row of the widest frame (RWARE, 255 columns: 23 718 B)

__host__ __device__ inline int band_rows(int W) { const int r = kBandBytes / (3 * W); return r < 1 ? 1 : r; }

// paint(x, y) -> Rgb of frame pixel (x, y).  The band is staged in band_s (kBandBytes + 16, 16-byte aligned) at the destination's address
// phase modulo 16, so the interior goes out as 16-byte stores and only the two ends as bytes.
template <typename Paint>
__device__ void render_band(uint8_t* frame, int W, int y0, int y1, uint8_t* band_s, const Paint& paint) {
  uint8_t* dst = frame + (size_t)y0 * W * 3;
  const int phase = (int)((uintptr_t)dst & 15), npx = (y1 - y0) * W, nbytes = 3 * npx;
  for (int p = threadIdx.x; p < npx; p += blockDim.x) {
    const int yy = p / W, x = p - yy * W;
    const Rgb c = paint(x, y0 + yy);
    uint8_t* b = band_s + phase + 3 * p;
    b[0] = c.r; b[1] = c.g; b[2] = c.b;
  }
  __syncthreads();
  const int head = (16 - phase) & 15;
  const int nw = nbytes > head ? (nbytes - head) >> 4 : 0, tail0 = nw ? head + 16 * nw : 0;
  const uint4* src = reinterpret_cast<const uint4*>(band_s + phase + head);
  uint4* dw = reinterpret_cast<uint4*>(dst + head);
  for (int i = threadIdx.x; i < nw; i += blockDim.x) dw[i] = src[i];
  for (int i = threadIdx.x; i < (nw ? head : 0); i += blockDim.x) dst[i] = band_s[phase + i];
  for (int i = tail0 + threadIdx.x; i < nbytes; i += blockDim.x) dst[i] = band_s[phase + i];
}

// Host: frames [n][H][W][3] of envs [env_first, env_first + n) of handle h, one CTA per (env, band).
template <typename Hd, typename Dev, typename St>
int launch_render(const Hd* h, const char* who, void (*kernel)(Dev, St, int, uint8_t*, int, int), int env_first, int n, uint8_t* frames, int H,
                  int W, void* stream) {
  MARL_REQUIRE(h != nullptr && frames != nullptr, "%s: NULL argument", who);
  MARL_REQUIRE(n >= 1 && env_first >= 0 && env_first <= h->E - n, "%s: envs [%d, %lld) are not a non-empty range inside [0, %d)", who, env_first,
               (long long)env_first + n, h->E);
  MARL_CUDA_TRY(cudaSetDevice(h->device));
  const int rows = band_rows(W);
  kernel<<<dim3((unsigned)n, (unsigned)((H + rows - 1) / rows)), kRenderThreads, 0, (cudaStream_t)stream>>>(h->dev, h->st, env_first, frames, H, W);
  MARL_CUDA_TRY(cudaGetLastError());
  return MARL_OK;
}

}  // namespace render
}  // namespace marl
