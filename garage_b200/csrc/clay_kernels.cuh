// clay_kernels.cuh -- Clay(k, m) encode / verify / decode / single-shard repair on sm_90a (DESIGN.md sections 2.4
// and 4.6).  Included by garage_ec.cu after rs_kernels.cuh: it reuses StripePlan, plan_kernel's plans over the
// RS(k+s, m) base code, xtime4 and the apply modes.
#pragma once

namespace garage_ec {

// A work item is one 16-byte column: the same 16 bytes of every layer of every node of one stripe, an independent
// codeword of the layered code.  It lives in shared memory as [layer][node][4 words] (alpha * (n'|1) * 16 bytes,
// 68 KB for alpha = 256 and n' = 16), and the threads of the CTA walk (layer, word) units of it.
constexpr uint32_t kClayColBytes = 16;
constexpr int kClayThreads = 256;
constexpr uint32_t kClayInvGamma = 0x8e;  // 2^-1 in GF(2^8)/0x11D
constexpr uint32_t kClayInvDet = 0xa7;    // (1 + 2*2)^-1 = 5^-1

// Words per layer in shared memory: the n' nodes' 16 bytes, with the node count made odd.  A warp's units are 8
// consecutive layers x 4 words; an odd pitch of 16-byte slots puts those 8 layers on 8 different bank quads (with
// n' = 16 and no padding they all fell on the same 4 banks: 8-way conflicts on every access).
__host__ __device__ constexpr uint32_t clay_layer_words(uint32_t nodes) { return 4 * (nodes | 1); }

struct ClayParams {
    const uint8_t *src;            // data shard j of stripe s at src + s*src_pitch + j*stride
    uint8_t *dst;                  // parity shard i of stripe s at dst + s*dst_pitch + (par_off + i)*stride
    unsigned long long src_pitch, dst_pitch;
    const uint32_t *shard_len;     // device, nullable (=> stride); must be a multiple of 16*alpha
    uint32_t *mismatch;            // kModeVerify
    const StripePlan *plan;        // kModePlan: plan_kernel's plan of the base code for the stripe
    const uint8_t *present;        // kModePlan: the caller's map, k+m per stripe
    const uint8_t *want;           // kModePlan: nullable
    int32_t *status;               // kModePlan: nullable; a malformed shard_len gets GARAGE_EC_E_INVALID
    uint32_t present_is_bad;       // kModePlan: `present` holds scrub's bad flags
    uint32_t stride, n, k, m, s, q, t, alpha, ips, par_off;
    uint32_t qpow[9];              // q^y
    uint8_t coef[kMaxM * kMaxK];   // uniform modes: the base parity rows, coef[i*(k+s) + j]
};

__device__ __forceinline__ uint32_t gf_mul4(uint32_t v, uint32_t c)
{
    uint32_t r = 0;
    for (; c; c >>= 1, v = xtime4(v))
        if (c & 1) r ^= v;
    return r;
}

// Per-stripe remap of the caller's present / want maps (k+m shards) onto the n' nodes of the base code, for
// plan_kernel.  Decode: present = the virtual nodes and the first k present shards, want = every other node.
// Repair (exactly one shard absent and wanted): present = every node outside the lost node's column, want = the column.
// The rule is clay_read_set (gf256.h), which the HOST paths use to choose what they upload.
__global__ void __launch_bounds__(256) clay_prep_kernel(const __grid_constant__ ClayParams p, uint8_t *present2,
                                                        uint8_t *want2)
{
    const uint32_t N = p.q * p.t, tot = p.k + p.m;
    for (uint32_t st = blockIdx.x * blockDim.x + threadIdx.x; st < p.n; st += gridDim.x * blockDim.x) {
        uint64_t pm = 0, wm = 0;
        for (uint32_t i = 0; i < tot; i++) {
            const bool pr = (p.present[(size_t)st * tot + i] != 0) != (p.present_is_bad != 0);
            pm |= (uint64_t)pr << i;
            wm |= (uint64_t)(!p.want || p.want[(size_t)st * tot + i] != 0) << i;
        }
        uint64_t rd = 0;
        const bool ok = clay_read_set((int)p.k, (int)p.m, pm, wm, &rd);
        const uint64_t absent = ((1ull << tot) - 1) & ~pm, w = absent & wm;
        uint64_t P2 = 0, W2 = 0;  // node masks
        auto nodes = [&](uint64_t shards) {
            uint64_t r = 0;
            for (; shards; shards &= shards - 1) r |= 1ull << clay_node((int)p.k, (int)p.s, ctz64(shards));
            return r;
        };
        const uint64_t virt = ((1ull << p.s) - 1) << p.k, alln = (1ull << N) - 1;
        if (!ok || !w) {
            P2 = virt | nodes(pm);  // unrecoverable (fewer than k+s rows), or nothing to rebuild
        } else if (popc64(absent) == 1) {
            const uint32_t y0 = (uint32_t)clay_node((int)p.k, (int)p.s, ctz64(absent)) / p.q;
            W2 = ((1ull << p.q) - 1) << (y0 * p.q);
            P2 = alln & ~W2;
        } else {
            P2 = virt | nodes(rd);
            W2 = alln & ~P2;
        }
        for (uint32_t a = 0; a < N; a++) {
            present2[(size_t)st * N + a] = (uint8_t)((P2 >> a) & 1);
            want2[(size_t)st * N + a] = (uint8_t)((W2 >> a) & 1);
        }
    }
}

// Encode (E = the parity column, survivors = data and virtual nodes, coefficients = P), verify (the same, compared
// with the stored parities) and, with a plan (kModePlan), decode of up to m absent shards or the repair of one.
//   decode: load the survivors; uncouple present pairs; then in layers of increasing score (the number of erased
//     nodes that are the layer's "dot" in their column) uncouple the present nodes paired with an erased one, from
//     the erased partner's U decoded one score earlier, and solve the erased U with the base-code plan; finally
//     couple and write the wanted shards.
//   repair of node f = (x0, y0): only the alpha/q layers with digit y0 = x0 are loaded; uncouple every node outside
//     column y0 (pairs stay inside those layers), solve the q nodes of column y0, and emit f's bytes of all q layers
//     that share the other digits.
template <int MODE>
__global__ void __launch_bounds__(kClayThreads) clay_apply_kernel(const __grid_constant__ ClayParams p)
{
    extern __shared__ __align__(16) uint32_t buf[];  // [layer][node][4]
    __shared__ uint8_t s_coef[kMaxM][kMaxK];
    __shared__ uint8_t s_surv[kMaxK], s_eidx[kMaxM];
    __shared__ unsigned long long s_E;
    __shared__ uint32_t s_out, s_ne, s_skip, s_repair, s_f, s_mm;
    const uint32_t tid = threadIdx.x, N = p.q * p.t, kb = p.k + p.s, tot = p.k + p.m;
    const uint32_t lp = clay_layer_words(N);
    const uint32_t total = p.n * p.ips;
    for (uint32_t it = blockIdx.x; it < total; it += gridDim.x) {
        const uint32_t st = it / p.ips, c = it - st * p.ips;
        const uint32_t L = p.shard_len ? __ldg(p.shard_len + st) : p.stride;
        const uint32_t sub = L / p.alpha;
        if (tid == 0) {
            uint32_t skip = 0;
            const bool bad = L % (kClayColBytes * p.alpha) != 0 || L > p.stride;
            s_mm = 0;
            s_repair = 0;
            s_f = 0;
            if (MODE == kModePlan) {
                const StripePlan *pl = p.plan + st;
                uint32_t absent = 0, w = 0;
                for (uint32_t i = 0; i < tot; i++) {
                    const bool pr = (p.present[(size_t)st * tot + i] != 0) != (p.present_is_bad != 0);
                    if (!pr) {
                        absent |= 1u << i;
                        if (!p.want || p.want[(size_t)st * tot + i]) w |= 1u << i;
                    }
                }
                if (bad) {
                    if (c == 0 && p.status) p.status[st] = -1;  // GARAGE_EC_E_INVALID
                    skip = 1;
                } else if (pl->unrecoverable || !pl->key_out || !w) {
                    skip = 1;
                } else {
                    s_E = pl->key_out;
                    s_ne = pl->nrows;
                    s_out = w;
                    s_repair = __popc(absent) == 1 ? 1u : 0u;
                    s_f = (uint32_t)clay_node((int)p.k, (int)p.s, __ffs(absent) - 1);
                }
            } else if (bad) {
                if (MODE == kModeVerify && c == 0) atomicOr(p.mismatch + st, (1u << p.m) - 1);
                skip = 1;
            } else {
                s_E = ((1ull << p.m) - 1) << kb;
                s_ne = p.m;
                s_out = ((1u << p.m) - 1) << p.k;
            }
            if (!skip && c * kClayColBytes >= sub) skip = 1;
            s_skip = skip;
        }
        __syncthreads();
        if (s_skip) {
            __syncthreads();
            continue;
        }
        // plan rows: survivors and coefficients of the erased nodes (uniform modes: the identity survivors and P)
        const uint32_t ne = s_ne;
        if (MODE == kModePlan) {
            const StripePlan *pl = p.plan + st;
            for (uint32_t i = tid; i < kb; i += blockDim.x) s_surv[i] = pl->surv[i];
            for (uint32_t i = tid; i < ne; i += blockDim.x) s_eidx[i] = pl->out_idx[i];
            for (uint32_t i = tid; i < ne * kb; i += blockDim.x) s_coef[i / kb][i % kb] = pl->coef[i / kb][i % kb];
        } else {
            for (uint32_t i = tid; i < kb; i += blockDim.x) s_surv[i] = (uint8_t)i;
            for (uint32_t i = tid; i < ne; i += blockDim.x) s_eidx[i] = (uint8_t)(kb + i);
            for (uint32_t i = tid; i < ne * kb; i += blockDim.x) s_coef[i / kb][i % kb] = p.coef[i];
        }
        const unsigned long long E = s_E;
        const bool repair = s_repair != 0;
        const uint32_t fa = s_f, x0 = fa % p.q, y0 = fa / p.q;
        // layers held: all alpha, or (repair) the alpha/q with digit y0 = x0, slot r <-> layer zr(r)
        const uint32_t nl = repair ? p.alpha / p.q : p.alpha;
        const uint32_t qy0 = p.qpow[y0], qy1 = p.qpow[y0 + 1];
        auto zr = [&](uint32_t r) { return repair ? (r / qy0) * qy1 + x0 * qy0 + r % qy0 : r; };
        auto rz = [&](uint32_t z) { return repair ? (z / qy1) * qy0 + z % qy0 : z; };
        auto digit = [&](uint32_t z, uint32_t y) { return (z / p.qpow[y]) % p.q; };
        auto slot = [&](uint32_t r, uint32_t a, uint32_t w) -> uint32_t & { return buf[r * lp + a * 4 + w]; };
        auto shard_ptr = [&](uint32_t i) -> uint8_t * {
            return i < p.k ? const_cast<uint8_t *>(p.src) + (size_t)st * p.src_pitch + (size_t)i * p.stride
                           : p.dst + (size_t)st * p.dst_pitch + (size_t)(p.par_off + i - p.k) * p.stride;
        };
        const size_t col = (size_t)c * kClayColBytes;
        // ---- load: the survivors (repair: every node but f), virtual nodes as zeros
        for (uint32_t u = tid; u < N * nl; u += blockDim.x) {
            const uint32_t a = u / nl, r = u - a * nl;
            const int sh = clay_shard((int)p.k, (int)p.s, (int)a);
            const bool load = repair ? a != fa : !((E >> a) & 1);
            uint4 v = make_uint4(0, 0, 0, 0);
            if (sh >= 0 && load) v = ldg_stream(shard_ptr((uint32_t)sh) + (size_t)zr(r) * sub + col);
            if (sh < 0 || load) *reinterpret_cast<uint4 *>(&slot(r, a, 0)) = v;
        }
        __syncthreads();
        // ---- uncouple the pairs whose two members are both known: each pair once, from its lower layer
        for (uint32_t u = tid; u < nl * 4; u += blockDim.x) {
            const uint32_t r = u >> 2, w = u & 3, z = zr(r);
            for (uint32_t a = 0; a < N; a++) {
                const uint32_t x = a % p.q, y = a / p.q;
                if (repair ? y == y0 : ((E >> a) & 1)) continue;
                const uint32_t zy = digit(z, y);
                if (zy == x) continue;
                const uint32_t b = zy + y * p.q;
                if (!repair && ((E >> b) & 1)) continue;
                const uint32_t zp = z + x * p.qpow[y] - zy * p.qpow[y];
                if (zp < z) continue;
                const uint32_t rp = rz(zp), ca = slot(r, a, w), cb = slot(rp, b, w);
                slot(r, a, w) = gf_mul4(ca ^ xtime4(cb), kClayInvDet);
                slot(rp, b, w) = gf_mul4(cb ^ xtime4(ca), kClayInvDet);
            }
        }
        __syncthreads();
        // base-code solve of one layer word: out[i] = XOR_j coef[i][j] * U[surv[j]]
        auto solve = [&](uint32_t r, uint32_t w, uint32_t (&o)[kMaxM / 2]) {
#pragma unroll
            for (int i = 0; i < kMaxM / 2; i++) o[i] = 0;
            for (uint32_t j = 0; j < kb; j++) {
                uint32_t v = slot(r, s_surv[j], w);
                for (int bit = 0; bit < 8; bit++, v = xtime4(v)) {
#pragma unroll
                    for (int i = 0; i < kMaxM / 2; i++)
                        if ((uint32_t)i < ne && ((s_coef[i][j] >> bit) & 1)) o[i] ^= v;
                }
            }
        };
        if (repair) {
            // ---- solve column y0 in every held layer and emit f at the q layers sharing the other digits
            uint8_t *fp = shard_ptr((uint32_t)clay_shard((int)p.k, (int)p.s, (int)fa)) + col;
            for (uint32_t u = tid; u < nl * 4; u += blockDim.x) {
                const uint32_t r = u >> 2, w = u & 3, z = zr(r);
                uint32_t o[kMaxM / 2];
                solve(r, w, o);
                for (uint32_t x = 0; x < p.q; x++) {
                    const uint32_t zx = z + x * qy0 - x0 * qy0;
                    uint32_t v;
                    if (x == x0) {
                        v = o[x];
                    } else {
                        const uint32_t cg = slot(r, x + y0 * p.q, w);
                        const uint32_t uf = gf_mul4(cg ^ o[x], kClayInvGamma);
                        v = uf ^ xtime4(o[x]);
                    }
                    *reinterpret_cast<uint32_t *>(fp + (size_t)zx * sub + 4 * w) = v;
                }
            }
            __syncthreads();
            continue;
        }
        // ---- decode by score: the erased partners' U of score sc-1 are known when score sc runs
        for (uint32_t sc = 0; sc <= p.t; sc++) {
            for (uint32_t u = tid; u < nl * 4; u += blockDim.x) {
                const uint32_t z = u >> 2, w = u & 3;
                uint32_t score = 0;
                for (unsigned long long e = E; e; e &= e - 1) {
                    const uint32_t a = (uint32_t)(__ffsll((long long)e) - 1);
                    score += digit(z, a / p.q) == a % p.q;
                }
                if (score != sc) continue;
                for (uint32_t a = 0; a < N; a++) {
                    if ((E >> a) & 1) continue;
                    const uint32_t x = a % p.q, y = a / p.q, zy = digit(z, y), b = zy + y * p.q;
                    if (zy == x || !((E >> b) & 1)) continue;
                    const uint32_t zp = z + x * p.qpow[y] - zy * p.qpow[y];
                    slot(z, a, w) ^= xtime4(slot(zp, b, w));
                }
                uint32_t o[kMaxM / 2];
                solve(z, w, o);
#pragma unroll
                for (int i = 0; i < kMaxM / 2; i++)
                    if ((uint32_t)i < ne) slot(z, s_eidx[i], w) = o[i];
            }
            __syncthreads();
        }
        // ---- couple the wanted erased shards and write (verify: compare) them
        uint32_t mm = 0;
        for (uint32_t u = tid; u < nl * 4; u += blockDim.x) {
            const uint32_t z = u >> 2, w = u & 3;
            for (uint32_t om = s_out; om; om &= om - 1) {
                const uint32_t i = (uint32_t)(__ffs(om) - 1), a = (uint32_t)clay_node((int)p.k, (int)p.s, (int)i);
                const uint32_t x = a % p.q, y = a / p.q, zy = digit(z, y);
                uint32_t v = slot(z, a, w);
                if (zy != x) v ^= xtime4(slot(z + x * p.qpow[y] - zy * p.qpow[y], zy + y * p.q, w));
                uint32_t *gp = reinterpret_cast<uint32_t *>(shard_ptr(i) + (size_t)z * sub + col) + w;
                if (MODE == kModeVerify) {
                    if (*gp != v) mm |= 1u << (i - p.k);
                } else {
                    *gp = v;
                }
            }
        }
        if (MODE == kModeVerify) {
            mm = __reduce_or_sync(0xffffffffu, mm);
            if (mm && (tid & 31) == 0) atomicOr(&s_mm, mm);
        }
        __syncthreads();
        if (MODE == kModeVerify && tid == 0 && s_mm) atomicOr(p.mismatch + st, s_mm);
    }
}

}  // namespace garage_ec
