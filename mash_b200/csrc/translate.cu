// translate.cu -- six-frame translation of a nucleotide chunk for the translated screen.
//
// Replaces the translation half of hashSequence with trans == true (reference CommandScreen.cpp:500-530, translate and
// aaFromCodon :617-809, reverseComplement Sketch.cpp:1071-1106).  The chunk becomes six peptide strings written back to back,
// each followed by one 0 byte: translate(seq + f) for f = 0, 1, 2, then translate(revcomp(seq) + f) for f = 0, 1, 2, frame f
// holding (len - f) / 3 amino acids.  A stop codon, or a codon with a byte outside {A,C,G,T} (upper-cased unless preserve_case;
// on the reverse strand 'U' complements to 'A' as in the reference's table), is written as 0, which lies outside the protein
// alphabet, so the byte scan kernel that follows skips every window holding one -- the reference's '*' test (:541).
#include "common.cuh"
#include "sketch_core.cuh"

namespace mashgpu {

constexpr int TR_THREADS = 256;
constexpr int TR_BASES = 48;                             // bases per thread: 3 vectors of 16 = 16 codon starts per frame and strand
constexpr int TR_CTA_BASES = TR_THREADS * TR_BASES;
constexpr int TR_CTA_CODONS = TR_CTA_BASES / 3;          // codons per frame per CTA

// Standard genetic code (NCBI table 1), index 16 b0 + 4 b1 + b2 with A0 C1 G2 T3; '*' = stop
__constant__ char c_codon_aa[65] = "KNKNTTTTRSRSIIMIQHQHPPPPRRRRLLLLEDEDAAAAGGGGVVVV*Y*YSSSS*CWCLFLF";

struct TrFrames {
    uint64_t base[6];     // output offset of forward frames 0..2, then reverse frames 0..2
    uint64_t n[3];        // amino acids per frame: (len - f) / 3, the same on both strands
};

uint64_t translated_length(uint64_t len)
{
    uint64_t t = 0;
    for (int f = 0; f < 3; f++) t += 2 * ((len > (uint64_t)f ? (len - f) / 3 : 0) + 1);
    return t;
}

// One thread: 48 consecutive bases p (plus the next two), i.e. the codon on bases p..p+2 of each p.  On the forward strand that
// codon is codon p / 3 of frame p % 3.  On the reverse strand it is, complemented and reversed, codon q = len - 3 - p of
// revcomp(seq): codon q / 3 of frame q % 3.  The thread's 48 starts fall into three classes p % 3 of 16 consecutive codons each,
// and every class lands in one forward and one reverse frame, so each class is packed into one 16-byte vector per strand.  The
// CTA stages its 6 x 4096 codons in shared memory and writes each frame out with coalesced byte stores (frame offsets are not
// aligned).  Codons that would run past the end of the chunk have a forward index >= n and a negative reverse index: clipped.
__global__ void __launch_bounds__(TR_THREADS) translate6_kernel(const uint8_t *__restrict__ seq, uint64_t len, int preserve_case, int aligned,
                                                                uint8_t *__restrict__ out, const __grid_constant__ TrFrames fr)
{
    __shared__ uint8_t lut[256];          // bits 0-1 forward code, bit 2 not a forward base, bits 4-5 complement code, bit 6 no complement
    __shared__ uint8_t aa[64];
    __shared__ __align__(16) uint8_t stage[6][TR_CTA_CODONS];
    const int t = threadIdx.x;
    {
        const int u = (!preserve_case && t > 96 && t < 123) ? t - 32 : t;     // CommandScreen.cpp:500-506
        const int f = u == 'A' ? 0 : u == 'C' ? 1 : u == 'G' ? 2 : u == 'T' ? 3 : 4;
        const int r = (u == 'A' || u == 'G') ? 3 - f : u == 'C' ? 2 : (u == 'T' || u == 'U') ? 0 : 4;
        lut[t] = (uint8_t)(f | (r << 4));
    }
    if (t < 64) aa[t] = c_codon_aa[t] == '*' ? 0 : (uint8_t)c_codon_aa[t];
    __syncthreads();

    const uint64_t P0 = (uint64_t)blockIdx.x * TR_CTA_BASES;
    const uint64_t P = P0 + (uint64_t)t * TR_BASES;
    const long long qb0 = (long long)len - 3 - (long long)P0;               // reverse codon index q of base P0
    const int rb = (int)(((qb0 % 3) + 3) % 3);                                // q % 3 of this thread's class 0 (48 | 3: the same for all)
    if (P < len) {
        uint32_t w[13];
        if (aligned) {
#pragma unroll
            for (int v = 0; v < 3; v++) {
                uint4 q = make_uint4(0, 0, 0, 0);
                if (P + 16 * v < len) q = __ldg(reinterpret_cast<const uint4 *>(seq + P + 16 * v));     // readable up to len rounded up to 16
                w[4 * v] = q.x; w[4 * v + 1] = q.y; w[4 * v + 2] = q.z; w[4 * v + 3] = q.w;
            }
            w[12] = (P + 48 < len ? seq[P + 48] : 0u) | ((P + 49 < len ? seq[P + 49] : 0u) << 8);
        } else {
#pragma unroll
            for (int i = 0; i < 13; i++) {
                uint32_t x = 0;
#pragma unroll
                for (int b = 0; b < 4; b++)
                    if (4 * i + b < TR_BASES + 2 && P + 4 * i + b < len) x |= (uint32_t)seq[P + 4 * i + b] << (8 * b);
                w[i] = x;
            }
        }
        uint32_t l[TR_BASES + 2];
#pragma unroll
        for (int j = 0; j < TR_BASES + 2; j++) l[j] = lut[(w[j >> 2] >> (8 * (j & 3))) & 0xFFu];
        uint32_t fw[3][4], rw[3][4];
#pragma unroll
        for (int c = 0; c < 3; c++)
#pragma unroll
            for (int i = 0; i < 4; i++) fw[c][i] = rw[c][i] = 0;
#pragma unroll
        for (int j = 0; j < TR_BASES; j++) {
            const uint32_t a = l[j], b = l[j + 1], c = l[j + 2], any = a | b | c;
            const uint32_t fa = (any & 4u) ? 0u : aa[((a & 3u) << 4) | ((b & 3u) << 2) | (c & 3u)];
            const uint32_t ra = (any & 64u) ? 0u : aa[(c & 0x30u) | ((b & 0x30u) >> 2) | ((a & 0x30u) >> 4)];
            const int cls = j % 3, i = j / 3, ri = 15 - i;           // reverse: codon index falls as p rises
            fw[cls][i >> 2] |= fa << (8 * (i & 3));
            rw[cls][ri >> 2] |= ra << (8 * (ri & 3));
        }
#pragma unroll
        for (int c = 0; c < 3; c++) {
            *reinterpret_cast<uint4 *>(&stage[c][16 * t]) = make_uint4(fw[c][0], fw[c][1], fw[c][2], fw[c][3]);
            const int r = (rb - c + 3) % 3;
            *reinterpret_cast<uint4 *>(&stage[3 + r][16 * (TR_THREADS - 1 - t)]) = make_uint4(rw[c][0], rw[c][1], rw[c][2], rw[c][3]);
        }
    }
    __syncthreads();
    const uint64_t first_f = P0 / 3;
    const long long qlast = qb0 - (long long)(TR_THREADS - 1) * TR_BASES;    // q of the CTA's last thread's first base
#pragma unroll
    for (int f = 0; f < 3; f++) {
        for (int i = t; i < TR_CTA_CODONS; i += TR_THREADS) {
            const uint64_t idx = first_f + i;
            if (idx < fr.n[f]) out[fr.base[f] + idx] = stage[f][i];
        }
    }
#pragma unroll
    for (int r = 0; r < 3; r++) {
        const int c = (rb - r + 3) % 3;
        const long long first_r = (qlast - c - r) / 3 - 15;                      // exact division: qlast - c == r (mod 3)
        for (int i = t; i < TR_CTA_CODONS; i += TR_THREADS) {
            const long long idx = first_r + i;
            if (idx >= 0 && (uint64_t)idx < fr.n[r]) out[fr.base[3 + r] + idx] = stage[3 + r][i];
        }
    }
    if (blockIdx.x == 0 && t < 6) out[fr.base[t] + fr.n[t % 3]] = 0;            // frame terminators
}

int translate_enqueue(mashgpu_ctx *ctx, const void *d_chunk, uint64_t len, int preserve_case, uint8_t *d_pep, cudaStream_t st)
{
    TrFrames fr;
    uint64_t o = 0;
    for (int f = 0; f < 3; f++) fr.n[f] = len > (uint64_t)f ? (len - f) / 3 : 0;
    for (int s = 0; s < 6; s++) { fr.base[s] = o; o += fr.n[s % 3] + 1; }
    const uint64_t blocks = len ? (len + TR_CTA_BASES - 1) / TR_CTA_BASES : 1;      // an empty chunk still gets its six terminators
    if (blocks > 0x7FFFFFFFull) return fail(ctx, MASHGPU_ERR_UNSUPPORTED, "chunk of %llu bases too large to translate", (unsigned long long)len);
    const int aligned = ((uintptr_t)d_chunk & 15) == 0;
    time_begin(ctx, ctx->translate_events, st);
    translate6_kernel<<<(unsigned)blocks, TR_THREADS, 0, st>>>(static_cast<const uint8_t *>(d_chunk), len, preserve_case, aligned, d_pep, fr);
    time_end(ctx, ctx->translate_events, st);
    ctx->kernel_launches++;
    ctx->translate_launches++;
    MG_CUDA(ctx, cudaGetLastError());
    return MASHGPU_OK;
}

}  // namespace mashgpu

using namespace mashgpu;

extern "C" int mashgpu_translate6(mashgpu_ctx *ctx, const void *d_seq, uint64_t len, int preserve_case, uint8_t *d_out)
{
    if (!ctx) return MASHGPU_ERR_INVALID;
    if (!d_seq || !d_out) return fail(ctx, MASHGPU_ERR_INVALID, "NULL argument");
    MG_CUDA(ctx, cudaSetDevice(ctx->device));
    MG_TRY(translate_enqueue(ctx, d_seq, len, preserve_case, d_out, ctx->stream));
    MG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return MASHGPU_OK;
}
