// parallel-cnn_b200/csrc/persist_kernels.cu -- the whole training loop as ONE persistent kernel (k_train_persist below):
// `nsteps` consecutive mini-batch steps without returning to the host, the gradient reduction, the SGD update, the
// multi-GPU exchange and the parameter broadcast all inside the kernel.  Round 1 synchronised the steps with two fenced
// grid barriers; this version is a dataflow over thread-block clusters, asynchronous distributed-shared-memory stores and
// tagged words in L2.
#include "fused_body.cuh"

using namespace pcnn_fused;

namespace {

constexpr int XS_MAXC = 40;          // clusters per rank the direct exchange has room for (an H100 holds 16 clusters of 8)
// most GPUs the direct exchange serves: each GPU stores (N - 1) x 0.6 MB per step into its peers, which grows with N while the
// L2 hop it saves does not.  Multi-GPU step times have not been measured on H100; 2 is the world size the scheme was built for.
constexpr int PCNN_DIRECT_MAX_WORLD = 2;
static size_t p2p_inbox_bytes() { return (size_t)2 * PCNN_MAX_PEERS * NPACK * sizeof(uint2); }
static size_t p2p_xslots_bytes() { return (size_t)2 * PCNN_MAX_PEERS * XS_MAXC * NPACK * sizeof(unsigned long long); }

struct PersistArgs {
    const void *images;
    const uint8_t *labels;
    long long n_total;
    float *params;            // global packed parameters, updated in place every step
    float *grads;             // packed gradient (+ error sum) of the most recent step
    long long *cursor;        // in/out: global sample position
    double *err_total;
    float *step_err;          // ring [STEP_ERR_CAP]
    int *step_idx;            // in/out: ring position
    int *abort_flag;
    int B, nsteps, rank, world, rank_local;
    float dt;
    // peer exchange (world > 1)
    uint2 *inbox;             // local  [2][world][NPACK] words {value bits, step id}
    uint2 *peer_inbox[PCNN_MAX_PEERS];
    unsigned step_base;       // id of the step before the first one of this launch (ids are unique per context lifetime)
    // flag-in-data buffers of the dataflow kernel (k_train_persist)
    llword *slots_ll;         // [grid][NPACK] tagged partial gradients
    llword *params_ll;        // [NPACK] tagged parameters: tag X = the parameters step X trains with
    unsigned xstep_base;      // same for the peer exchange (advances only on distributed launches)
    // direct exchange (2 GPUs): every cluster's share owner also stores its share into the peers' copies of this array,
    // [2 parities][PCNN_MAX_PEERS source ranks][XS_MAXC clusters][NPACK] tagged words in IPC-mapped memory; the owners then
    // gather ranks x clusters slots in one go and the separate exchange hop disappears
    llword *xslots;
    llword *peer_xslots[PCNN_MAX_PEERS];
    int direct;
    // host streaming (pcnn_learn_host): sample i may be read once ready[pcnn_chunk_of(ready_chunks, i)] == ready_tag
    const unsigned *ready;
    unsigned ready_tag;
    pcnn_chunking ready_chunks;   // sample -> chunk (pcnn_chunk_of)
    int early;                // 1: request the next step's first image a whole step ahead (images read across PCIe)
    int fresh;                // bit 0: start at sample 0 / step 0 instead of the device-side counters; bit 1: err_total = 0
    float *step_err_host;     // optional mapped pinned array [nsteps]: per-step error sums written straight to the host
    double *done_host;        // optional mapped pinned {double error sum, unsigned tag}: written after the LAST step, so the
    unsigned done_tag;        //   host can return as soon as the results are there instead of waiting for the stream
    long long *trace;         // optional [PCNN_TRACE_STEPS][6] globaltimer stamps written by CTA 0 (pcnn_persist_trace)
};

__device__ __forceinline__ long long globaltimer_ns() {
    long long v;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(v));
    return v;
}

// {value, step id} words of the peer exchange: one 8-byte volatile access each way (bypasses L1, single-copy atomic)
__device__ __forceinline__ void st_ll(uint2 *p, float value, unsigned id) {
    asm volatile("st.volatile.global.v2.u32 [%0], {%1, %2};" ::"l"(p), "r"(__float_as_uint(value)), "r"(id) : "memory");
}
// tagged 64-bit words in PEER-visible memory (system scope: the writer is another GPU)
__device__ __forceinline__ void ll_store_sys(llword *p, float v, unsigned tag) {
    asm volatile("{ .reg .b64 t; mov.b64 t, {%1, %2}; st.relaxed.sys.global.u64 [%0], t; }" ::"l"(p), "r"(__float_as_uint(v)), "r"(tag)
                 : "memory");
}
__device__ __forceinline__ void ll_load_sys(const llword *p, float &v, unsigned &tag) {
    unsigned lo;
    asm volatile("{ .reg .b64 t; ld.relaxed.sys.global.u64 t, [%2]; mov.b64 {%0, %1}, t; }" : "=r"(lo), "=r"(tag) : "l"(p) : "memory");
    v = __uint_as_float(lo);
}
__device__ __forceinline__ uint2 ld_ll(const uint2 *p) {
    uint2 v;
    asm volatile("ld.volatile.global.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(p) : "memory");
    return v;
}

// =====================================================================================================================
// k_train_persist -- the dataflow version: thread-block clusters, asynchronous distributed-shared-memory stores and
// tagged words through L2; no grid barrier, no cluster barrier and no fence inside the step loop.
//
// Inside a cluster (CS = 8 CTAs) data is PUSHED into the consumer's shared memory with st.async, which signals the
// consumer's mbarrier with the byte count (the mechanism of a bulk copy): the consumer just waits on its own mbarrier.
// Between clusters data moves through L2 as tagged 64-bit words {fp32 value, step id} (fused_body.cuh: ll_store /
// ll_load) that the consumer polls until they carry the id it expects.  Per step X every CTA (cluster rank r)
//   1. polls share r (1/CS) of the tagged parameters (tag X) and pushes it into S.params of all CS CTAs; waits until its
//      own S.params is complete (mbarrier, 9,376 bytes),
//   2. runs forward + backward over its images,
//   3. reduces its register accumulators and pushes piece q of the packed gradient to cluster rank q (S.recv[r]),
//   4. waits for the CS pieces of ITS share (mbarrier), adds them in rank order and writes them, tagged X, to the
//      cluster's slot in L2,
//   5. as OWNER of a chunk of the packed vector: gathers that chunk from all cluster slots (tag X), adds them in slot
//      order, [N > 1: exchanges the chunk with the peer GPUs, rank order], updates its parameters -- which it keeps in
//      registers for the whole launch -- and publishes them with tag X + 1.
// Buffer reuse needs no extra synchronisation: a CTA can only reach the next use of a buffer after it has received the
// parameters tagged X + 1, i.e. after every owner has read all cluster slots of step X, i.e. after every CTA of every
// cluster has consumed what was pushed to it in step X.
// Determinism: rank order, slot order and phase order are fixed -> bit-identical reruns and replicas.
// =====================================================================================================================
// phase boundaries of one step as seen by CTA 0: 0 step start, 1 parameters resident, 2 images done, 3 cluster slot
// written, 4 owned chunk gathered, 5 parameters published
// dataflow kernel: CTA 0 stamps every step (row s of the trace), and at step PCNN_TRACE_STEPS / 2 EVERY CTA stamps its own
// row (8 values: the 6 phase stamps, its SM id, spare) behind them -- the spread over CTAs is the skew the owners wait for
#define PCNN_TRACE2(k)                                                  \
    do {                                                                \
        if (t == 0) {                                                   \
            const long long now__ = globaltimer_ns();                   \
            if (tr0) tr0[(k)] = now__;                                  \
            if (tr1) tr1[(k)] = now__;                                  \
        }                                                               \
    } while (0)

constexpr long long POLL_BUDGET = 4000000000LL;   // cycles a single wait may take before the launch is aborted

// Budget of one wait.  Once any wait has given up (here or in another CTA: global abort flag) every later wait of this CTA
// returns at once (shared-memory flag), so an aborted launch drains in milliseconds instead of hanging the GPU.  No CTA
// ever leaves the step loop early: the hardware cluster barriers need all of them.
struct PollGuard {
    long long t0;
    unsigned n;
    int *abort_flag;
    volatile int *local;
    __device__ __forceinline__ PollGuard(int *f, int *cta_flag) {
        t0 = clock64();
        n = 0;
        abort_flag = f;
        local = cta_flag;
    }
    // true: give up
    __device__ __forceinline__ bool expired(int code) {
        if ((++n & 255u) != 0) return false;
        if (*local) return true;
        if (*(volatile int *)abort_flag) { *local = 1; return true; }
        if (clock64() - t0 > POLL_BUDGET) { *(volatile int *)abort_flag = code; *local = 1; return true; }
        return false;
    }
};

// mbarrier wait that gives up with the launch (same budget as the polling loops)
__device__ __forceinline__ void mbar_wait_guarded(unsigned long long *bar, unsigned parity, PollGuard &guard) {
    for (;;) {
        unsigned done;
        asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                     : "=r"(done)
                     : "r"(smem_u32(bar)), "r"(parity)
                     : "memory");
        if (done || guard.expired(1)) return;
    }
}

// share `rank` of the packed vector among CS cluster ranks: [rank * SH, rank * SH + len), SH even (moved in pairs)
template <int CS> struct Share {
    static constexpr int SH = ((NPACK + CS - 1) / CS + 1) & ~1;
    __device__ __forceinline__ static int len(unsigned rank) {
        const int b = (int)rank * SH;
        return b >= NPACK ? 0 : (b + SH > NPACK ? NPACK - b : SH);
    }
};

// Step 1: poll this rank's share of the tagged parameters and push every pair into S.params of ALL CTAs of the cluster;
// then wait until this CTA's own S.params has received all NPACK floats (thread 0 armed the mbarrier for them).
template <typename InT, int CS, int NTH>
__device__ __forceinline__ void fetch_params_cluster(FusedSmem<InT> &S, const llword *pll, unsigned tag, unsigned crank, unsigned parity,
                                                     int *abort_flag) {
    static_assert(NPACK % 2 == 0, "pairs");
    const int sb = (int)crank * Share<CS>::SH, sl = Share<CS>::len(crank);
    PollGuard guard(abort_flag, &S.aborted);
    for (int i = threadIdx.x; i < sl / 2; i += NTH) {
        float v0, v1;
        unsigned g0, g1;
        for (;;) {
            ll_load2(pll + sb + 2 * i, v0, g0, v1, g1);
            if ((g0 == tag && g1 == tag) || guard.expired(1)) break;
        }
        float *dst = S.params + sb + 2 * i;
        if (CS == 1) {
            *reinterpret_cast<float2 *>(dst) = make_float2(v0, v1);       // published by the image pass's first block barrier
        } else {
#pragma unroll
            for (unsigned q = 0; q < (unsigned)CS; ++q) dsmem_st_async_f2(dsmem_addr(dst, q), v0, v1, dsmem_addr(&S.params_bar, q));
        }
    }
    if (CS > 1) mbar_wait_guarded(&S.params_bar, parity, guard);
}

// gradient piece sink of the CTA epilogue: entry p goes to the cluster rank that owns its share
template <typename InT, int CS> struct PushSink {
    FusedSmem<InT> *S;
    unsigned crank;
    __device__ __forceinline__ void operator()(int p, float v) const {
        if (CS == 1) {
            S->recv[p] = v;
            return;
        }
        const unsigned q = (unsigned)p / (unsigned)Share<CS>::SH;
        const int i = p - (int)q * Share<CS>::SH;
        dsmem_st_async_f32(dsmem_addr(S->recv + (int)crank * Share<CS>::SH + i, q), v, dsmem_addr(&S->grads_bar, q));
    }
};

// thread 0: wait until the host-streamed chunk holding `src` has landed (pcnn_learn_host), then make the DMA-written
// bytes visible to the async proxy that the bulk copy reads through.  The gate's constants live in shared memory.
template <typename InT> struct ChunkGate {
    FusedSmem<InT> *S;
    __device__ __forceinline__ void operator()(const void *src) const {
        const unsigned *ready = S->gate_ready;
        if (!ready) return;
        const long long sample = (reinterpret_cast<const InT *>(src) - reinterpret_cast<const InT *>(S->gate_images)) / PCNN_IMG;
        const unsigned *f = ready + pcnn_chunk_of(S->gate_chunks, sample);
        const unsigned want = S->gate_tag;
        PollGuard guard(S->gate_abort, &S->aborted);
        while (*(const volatile unsigned *)f != want)
            if (guard.expired(3)) break;
        asm volatile("fence.proxy.async.global;" ::: "memory");
    }
};

// Steps 2 and 3 of a step: forward + backward over this CTA's images b = c, c + G, ... < nb (IPC = 2: image 2c + half of
// each half), then the CTA reduction whose results are pushed piece-wise to the cluster ranks.  Returns the advanced
// image counter of this thread's half.
template <typename InT, int CS, int IPC>
__device__ __forceinline__ int step_images(FusedSmem<InT> &S, ImageSmem<InT> &H, PairXchg *X, const ThreadId &id, int half,
                                           const InT *img_base, const uint8_t *lab_base, int c, int G, int nb, int li, unsigned crank,
                                           long long *trace_row, long long *trace_row2) {
    const ChunkGate<InT> gate{&S};
    if (IPC == 2 || nb <= G) {
        // at most one image per CTA half (batch <= images the grid holds side by side, the usual case): the specialised
        // single-image step; the image was prepared (landed + converted) while the CTA was waiting for the parameters
        const int ci = c * IPC + half;
        image_step_single<IPC>(S, H, X, id, half, li, ci < nb, PushSink<InT, CS>{&S, crank});
        if (threadIdx.x == 0 && (trace_row || trace_row2)) {
            const long long now = globaltimer_ns();
            if (trace_row) trace_row[2] = now;
            if (trace_row2) trace_row2[2] = now;
        }
        return ci < nb ? li + 1 : li;
    }
    li = image_steps_multi(S, id, img_base, lab_base, c, G, nb, li, gate, PushSink<InT, CS>{&S, crank});
    if (id.t == 0 && (trace_row || trace_row2)) {
        const long long now = globaltimer_ns();
        if (trace_row) trace_row[2] = now;
        if (trace_row2) trace_row2[2] = now;
    }
    return li;
}

// The fp32 staging buffers of a CTA half start as zeros.  A half without an image still reads its buffer in the c1 weight
// gradient of image_step_single (as a product with dpc = 0), and leftover shared memory may hold NaN (0 x NaN = NaN).  From
// then on only bulk copies of pixels and the u8 conversion write them.  The fence orders these stores before the bulk copies.
// Not inlined: the launch prologue then leaves the register allocation of the step loop alone.
__device__ __noinline__ void zero_staging(float *imgf, int t) {
    for (int i = t; i < 2 * PCNN_IMG; i += NT) imgf[i] = 0.0f;
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// two-image CTA (IPC = 2): image 0's buffers and everything the CTA shares, image 1's buffers, the hand-over area
template <typename InT> struct PairSmem {
    FusedSmem<InT> s;
    ImageSmem<InT> h1;
    PairXchg x;
};
template <typename InT, int IPC> constexpr size_t persist_smem_bytes() {
    return IPC == 1 ? sizeof(FusedSmem<InT>) : sizeof(PairSmem<InT>);
}

// DIRECT (2 GPUs, see PersistArgs::xslots) is compile-time: as a run-time flag the generalised slot addressing of the owner gather
// is paid by every configuration, one GPU included (compare builds with scripts/step_ab_raw.py).
// IPC: images per CTA trained side by side.  1: one 224-thread CTA per image, two CTAs per SM.  2: one 448-thread CTA per SM
// whose halves (threads half * 224 ...) train images 2c and 2c + 1; the CTA's once-per-step work (parameter fetch, gradient
// pushes, cluster slot, barriers) is then done once per SM instead of twice (image_step_single).
template <typename InT, int CS, bool DIRECT, int IPC>
__global__ void __launch_bounds__(NT * IPC, IPC == 1 ? FUSED_CTAS_PER_SM : 1) k_train_persist(const PersistArgs a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    constexpr int NTH = NT * IPC;
    FusedSmem<InT> &S = *reinterpret_cast<FusedSmem<InT> *>(smem_raw);
    PairSmem<InT> &PS = *reinterpret_cast<PairSmem<InT> *>(smem_raw);      // IPC = 2 only
    const int half = IPC == 1 ? 0 : (int)threadIdx.x / NT;
    ImageSmem<InT> &H = half == 0 ? static_cast<ImageSmem<InT> &>(S) : PS.h1;
    PairXchg *X = IPC == 1 ? nullptr : &PS.x;
    const ThreadId id((int)threadIdx.x - half * NT);                         // thread within its image's 224
    const int t = threadIdx.x;
    const int G = gridDim.x, c = blockIdx.x;
    const int ci = c * IPC + half;                                           // this half's image of the batch
    const InT *images = reinterpret_cast<const InT *>(a.images);
    const ChunkGate<InT> gate{&S};
    if (t == 0) {
        S.gate_images = a.images;
        S.gate_ready = a.ready;
        S.gate_chunks = a.ready_chunks;
        S.gate_abort = a.abort_flag;
        S.gate_tag = a.ready_tag;
        S.aborted = 0;
    }

    // cluster geometry (CS = 1: launched without a cluster dimension, every CTA is its own cluster)
    const unsigned crank = CS == 1 ? 0u : cluster_ctarank();
    const int NC = G / CS;                                // clusters = slots
    const int my_sb = (int)crank * Share<CS>::SH, my_sl = Share<CS>::len(crank);
    llword *cslot = a.slots_ll + (long long)(CS == 1 ? (unsigned)c : cluster_idx()) * NPACK;
    // owner geometry: this CTA owns packed entries [e0, e0 + cnt); thread t owns entry e0 + t (wide chunks: + i * NTH)
    const int chunk = (NPACK + G - 1) / G;
    const int e0 = c * chunk;
    const int cnt = e0 >= NPACK ? 0 : (e0 + chunk > NPACK ? NPACK - e0 : chunk);
    const int PH = chunk >= NT ? 1 : NT / chunk;         // slot phases when the chunk is narrower than the CTA
    constexpr int KB = 8;                                // slot words one thread keeps in flight
    const int NV = DIRECT ? NC * a.world : NC;           // slots an owner gathers: clusters (x ranks with the direct exchange)
    const int PHG = PH < (NV + KB - 1) / KB ? PH : (NV + KB - 1) / KB;   // phases in use: thread (e, ph) adds slots ph, ph + PHG, ...

    long long cursor = (a.fresh & 1) ? 0 : *a.cursor;
    const int step_idx0 = (a.fresh & 1) ? 0 : *a.step_idx;
    const long long stride = a.rank_local ? (long long)a.B : (long long)a.B * a.world;
    auto shard = [&](long long cur, long long &base, int &nb) {
        base = cur + (a.rank_local ? 0 : (long long)a.rank * a.B);
        const long long avail = a.n_total - base;
        nb = avail <= 0 ? 0 : (avail < a.B ? (int)avail : a.B);
    };
    long long base;
    int nb;
    shard(cursor, base, nb);

    if (CS > 1 && cluster_nctarank() != (unsigned)CS) {
        // launched without the cluster dimension this instantiation is built for (seen under profilers that re-issue the
        // launch): every CTA takes this exit, nothing has been signalled yet
        if (t == 0) *(volatile int *)a.abort_flag = 4;
        return;
    }
    zero_staging(&H.imgf[0][0], id.t);      // ordered before the first bulk copy by the barrier that ends init_barriers
    init_barriers(S, IPC == 1 ? nullptr : &PS.h1);
    if (CS > 1) cluster_sync_all();   // every CTA's mbarriers are initialised before a peer may signal them
    int li = 0;                 // running image counter of this half (staging buffer + mbarrier phase)
    if (id.t == 0 && ci < nb) {
        const InT *src = images + (base + ci) * PCNN_IMG;
        gate(src);
        issue_image(H, 0, src);
    }
    __syncwarp();   // lane 0 rejoins its warp (see image_pass)

    // launch prologue: owners read their parameters once (they live in registers from here on) and publish them for
    // the first step
    float w0 = 0.0f;            // chunk < NT (the usual case): the one parameter this thread owns
#pragma unroll 1
    for (int e = t; e < cnt; e += NTH) {
        const int p = e0 + e;
        const float w = p < NPARAM ? __ldcg(a.params + p) : 0.0f;
        if (e == t) w0 = w;
        ll_store(a.params_ll + p, w, a.step_base + 1u);
    }

    for (int s = 0; s < a.nsteps; ++s) {
        const unsigned tag = a.step_base + (unsigned)s + 1u;
        long long *tr0 = (a.trace && c == 0 && s < PCNN_TRACE_STEPS) ? a.trace + s * 6 : nullptr;
        long long *tr1 = (a.trace && s == PCNN_TRACE_STEPS / 2) ? a.trace + PCNN_TRACE_STEPS * 6 + c * 8 : nullptr;
        if (tr1 && t == 0) {
            unsigned smid;
            asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
            tr1[6] = (long long)smid;
        }
        PCNN_TRACE2(0);
        // ---- 1. this step's parameters: my share L2 -> shared memory of the whole cluster.  Thread 0 arms both
        //         mbarriers of the step: all NPACK parameters, and CS pieces of my gradient share
        if (CS > 1 && t == 0) {
            mbar_expect_tx(&S.params_bar, NPACK * 4);
            mbar_expect_tx(&S.grads_bar, (unsigned)(CS * my_sl * 4));
        }
        __syncwarp();
        // the step's first image has been in flight since the previous step: land + convert it while the owners publish
        if (ci < nb) image_prepare(S, H, id, li, a.labels + base + ci);
        fetch_params_cluster<InT, CS, NTH>(S, a.params_ll, tag, crank, (unsigned)s & 1u, a.abort_flag);
        PCNN_TRACE2(1);

        // Images in pinned HOST memory (pcnn_learn_host): the NEXT step's first image is requested now, a whole step ahead, so that
        // the PCIe latency disappears behind the step; the other staging buffer is free (one image per CTA half and step;
        // with more, the in-step prefetch chain owns it).  Device-resident data keep the late request (no PCIe latency to hide).
        const bool early_issue = a.early != 0 && nb <= G * IPC;
        if (early_issue && id.t == 0 && s + 1 < a.nsteps) {
            long long ecur = cursor + stride;
            if (ecur >= a.n_total) ecur = 0;
            long long ebase;
            int enb;
            shard(ecur, ebase, enb);
            if (ci < enb) issue_image(H, (ci < nb ? li + 1 : li) & 1, images + (ebase + ci) * PCNN_IMG);
        }
        __syncwarp();

        // ---- 2. forward + backward over this CTA's images, 3. CTA reduction, pieces pushed to the cluster ranks
        li = step_images<InT, CS, IPC>(S, H, X, id, half, images + base * PCNN_IMG, a.labels + base, c, G, nb, li, crank,
                                       tr0, tr1);

        // ---- 4. my share: the CS pieces (rank order) -> tagged cluster slot
        {
            PollGuard guard(a.abort_flag, &S.aborted);
            if (CS > 1) mbar_wait_guarded(&S.grads_bar, (unsigned)s & 1u, guard);
            else __syncthreads();
            for (int i = t; i < my_sl; i += NTH) {
                float g = 0.0f;
#pragma unroll
                for (int q = 0; q < CS; ++q) g += S.recv[q * Share<CS>::SH + i];
                ll_store(cslot + my_sb + i, g, tag);
                if (DIRECT) {            // the peers' owners gather this cluster's share straight from their own memory
                    const unsigned xt = a.xstep_base + (unsigned)s + 1u;
                    const long long off = ((((long long)(xt & 1u) * PCNN_MAX_PEERS + a.rank) * XS_MAXC + (CS == 1 ? c : (int)cluster_idx())) * NPACK) + my_sb + i;
                    for (int r = 0; r < a.world; ++r)
                        if (r != a.rank) ll_store_sys(a.peer_xslots[r] + off, g, xt);
                }
            }
        }
        PCNN_TRACE2(3);

        // position of the next step; its first image is prefetched while the gradient is being reduced
        long long ncur = cursor + stride;
        if (ncur >= a.n_total) ncur = 0;
        long long nbase;
        int nnb;
        shard(ncur, nbase, nnb);
        const bool more = s + 1 < a.nsteps;
        if (id.t == 0 && more && ci < nnb && !early_issue) {
            const InT *src = images + (nbase + ci) * PCNN_IMG;
            gate(src);
            issue_image(H, li & 1, src);
        }
        __syncwarp();

        // ---- 4. owner: gather my chunk from all slots in slot order; 5. [N > 1: exchange with the peer GPUs], update,
        //         publish the next step's parameters
        const float step = a.dt / (float)effective_global_batch(cursor, true, a.n_total, a.B, a.world, a.rank_local);
        const unsigned xtag = a.xstep_base + (unsigned)s + 1u;
        // entry p: local sum g, parameter value before the step w_old; returns the updated parameter
        auto finalize = [&](int p, float g, float w_old) -> float {
            if (a.world > 1 && !DIRECT) {
                // "low-latency" push: every 8-byte inbox word carries {value, step id}; one NVLink one-way latency per step.
                // Every polling round then requests the words of ALL ranks still missing at once; the ranks' values are
                // added in rank order, so all GPUs compute bit-identical sums.
                const int par = (int)(xtag & 1u);
                for (int q = 0; q < a.world; ++q)
                    st_ll(a.peer_inbox[q] + ((long long)par * a.world + a.rank) * NPACK + p, g, xtag);
                const uint2 *w0p = a.inbox + (long long)par * a.world * NPACK + p;
                uint2 v[PCNN_MAX_PEERS];
                unsigned pending = (1u << a.world) - 1u;
                PollGuard guard(a.abort_flag, &S.aborted);
                while (pending) {
#pragma unroll
                    for (int q = 0; q < PCNN_MAX_PEERS; ++q)
                        if ((pending >> q) & 1u) v[q] = ld_ll(w0p + (long long)q * NPACK);
#pragma unroll
                    for (int q = 0; q < PCNN_MAX_PEERS; ++q)
                        if (((pending >> q) & 1u) && v[q].y == xtag) pending &= ~(1u << q);
                    if (pending && guard.expired(2)) break;
                }
                g = 0.0f;
#pragma unroll
                for (int q = 0; q < PCNN_MAX_PEERS; ++q)
                    if (q < a.world) g += __uint_as_float(v[q].x);
            }
            a.grads[p] = g;
            float w = 0.0f;
            if (p < NPARAM) {
                w = updated_entry(w_old, p, g, step);
                a.params[p] = w;
            } else {
                const double tot = (s == 0 && (a.fresh & 2)) ? (double)g : *a.err_total + (double)g;
                *a.err_total = tot;
                a.step_err[(step_idx0 + s) & (STEP_ERR_CAP - 1)] = g;
                if (a.step_err_host) a.step_err_host[s] = g;
                // an aborted launch never reports completion: the host then falls back to a stream synchronisation + abort check
                if (a.done_host && s + 1 == a.nsteps && *(volatile int *)a.abort_flag == 0) {   // same thread as the per-step stores
                    *(volatile double *)a.done_host = tot;
                    __threadfence_system();
                    *(volatile unsigned *)(a.done_host + 1) = a.done_tag;
                }
            }
            ll_store(a.params_ll + p, w, tag + 1u);
            return w;
        };
        if (chunk < NT) {
            const int e = t % chunk, ph = t / chunk;
            float sum = 0.0f;
            if (e < cnt && ph < PHG) {
                PollGuard guard(a.abort_flag, &S.aborted);
                if (DIRECT) {
                    // virtual slot v = (source rank, cluster): this GPU's own clusters live in slots_ll (local tag), the peers' in
                    // xslots (exchange tag); every GPU adds them in the same (rank, cluster) order -> bit-identical replicas
                    const int par = (int)(xtag & 1u);
                    auto slot_word = [&](int v, const llword *&ptr, unsigned &want, bool &remote) {
                        const int q = v / NC, k = v - q * NC;
                        remote = q != a.rank;
                        ptr = remote ? a.xslots + ((((long long)par * PCNN_MAX_PEERS + q) * XS_MAXC + k) * NPACK) + e0 + e
                                     : a.slots_ll + (long long)k * NPACK + e0 + e;
                        want = remote ? xtag : tag;
                    };
                    for (int k0 = ph; k0 < NV; k0 += KB * PHG) {
                        float v[KB];
                        unsigned pend = 0;
#pragma unroll
                        for (int u = 0; u < KB; ++u) {
                            v[u] = 0.0f;
                            if (k0 + u * PHG < NV) pend |= 1u << u;
                        }
                        while (pend) {
                            unsigned g[KB], want[KB];
#pragma unroll
                            for (int u = 0; u < KB; ++u)
                                if ((pend >> u) & 1u) {
                                    const llword *ptr;
                                    bool remote;
                                    slot_word(k0 + u * PHG, ptr, want[u], remote);
                                    if (remote) ll_load_sys(ptr, v[u], g[u]);
                                    else ll_load(ptr, v[u], g[u]);
                                }
#pragma unroll
                            for (int u = 0; u < KB; ++u)
                                if (((pend >> u) & 1u) && g[u] == want[u]) pend &= ~(1u << u);
                            if (pend && guard.expired(1)) break;
                        }
#pragma unroll
                        for (int u = 0; u < KB; ++u) sum += v[u];              // slot order within the phase
                    }
                } else {
                    const llword *sp = a.slots_ll + e0 + e;
                    for (int k0 = ph; k0 < NC; k0 += KB * PHG) {
                        float v[KB];
                        unsigned pend = 0;
#pragma unroll
                        for (int u = 0; u < KB; ++u) {
                            v[u] = 0.0f;
                            if (k0 + u * PHG < NC) pend |= 1u << u;
                        }
                        while (pend) {
                            unsigned g[KB];
#pragma unroll
                            for (int u = 0; u < KB; ++u)
                                if ((pend >> u) & 1u) ll_load(sp + (long long)(k0 + u * PHG) * NPACK, v[u], g[u]);
#pragma unroll
                            for (int u = 0; u < KB; ++u)
                                if (((pend >> u) & 1u) && g[u] == tag) pend &= ~(1u << u);
                            if (pend && guard.expired(1)) break;
                        }
#pragma unroll
                        for (int u = 0; u < KB; ++u) sum += v[u];              // slot order within the phase
                    }
                }
            }
            if (ph < PHG) S.part[ph * chunk + e] = sum;
            __syncthreads();
            PCNN_TRACE2(4);
            if (t < cnt) {
                float g = S.part[t];
                for (int q = 1; q < PHG; ++q) g += S.part[q * chunk + t];      // phase order
                w0 = finalize(e0 + t, g, w0);
            }
        } else {                                                               // G <= 10: a thread owns several entries
            PCNN_TRACE2(4);
#pragma unroll 1
            for (int e = t; e < cnt; e += NTH) {
                const int p = e0 + e;
                const llword *sp = a.slots_ll + p;
                PollGuard guard(a.abort_flag, &S.aborted);
                float acc = 0.0f;
                for (int k = 0; k < NC; ++k) {
                    float v;
                    unsigned g;
                    for (;;) {
                        ll_load(sp + (long long)k * NPACK, v, g);
                        if (g == tag || guard.expired(1)) break;
                    }
                    acc += v;
                }
                // the parameter is re-read: this thread itself stored it one step earlier
                finalize(p, acc, p < NPARAM ? __ldcg(a.params + p) : 0.0f);
            }
        }
        __syncwarp();
        PCNN_TRACE2(5);
        cursor = ncur;
        base = nbase;
        nb = nnb;
    }
    if (c == 0 && t == 0) {
        *a.cursor = cursor;
        *a.step_idx = step_idx0 + a.nsteps;
    }
    if (CS > 1) cluster_sync_all();     // no CTA leaves while a cluster peer may still push into its shared memory
}

constexpr int PERSIST_CS = 8;            // cluster size of the dataflow kernel (1 = fallback without clusters)
// cluster sizes of the two-image kernel, preferred first: at one CTA per SM a cluster needs that many SMs of one GPC.  An
// H100 80GB HBM3 keeps 120 such CTAs co-resident in clusters of 4 (or 8) -- up to 240 images -- and 128 and more in clusters
// of 2 (a batch of 256).  Where both fit, clusters of 4 are faster (fewer cluster slots to gather).
constexpr int PAIR_CS[2] = {4, 2};

template <typename InT> int persist_cap(int *out) {
    int m = 1 << 30;
    const void *fns[3] = {(const void *)k_train_persist<InT, PERSIST_CS, false, 1>, (const void *)k_train_persist<InT, PERSIST_CS, true, 1>,
                          (const void *)k_train_persist<InT, 1, false, 1>};
    for (const void *fn : fns) {
        int per_sm = 0;
        cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(FusedSmem<InT>));
        if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, NT, sizeof(FusedSmem<InT>));
        if (e != cudaSuccess) return pcnn_fail_cuda(e, "persistent kernel occupancy", __FILE__, __LINE__);
        if (per_sm < m) m = per_sm;
    }
    *out = m;
    return PCNN_OK;
}

// CTAs of IPC images each that can be co-resident when the grid is launched as clusters of CSZ (0 when they cannot be
// scheduled)
template <typename InT, int IPC, int CSZ> int cluster_cap(int sm_count) {
    if constexpr (IPC == 2) {      // the single-image variants are set up by persist_cap
        const void *fns[2] = {(const void *)k_train_persist<InT, CSZ, false, 2>, (const void *)k_train_persist<InT, CSZ, true, 2>};
        for (const void *fn : fns)
            if (cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)persist_smem_bytes<InT, 2>()) != cudaSuccess) {
                cudaGetLastError();
                return 0;
            }
    }
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)(CSZ * sm_count));            // any multiple of the cluster size
    cfg.blockDim = dim3(NT * IPC);
    cfg.dynamicSmemBytes = persist_smem_bytes<InT, IPC>();
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = CSZ;
    at[0].val.clusterDim.y = 1;
    at[0].val.clusterDim.z = 1;
    cfg.attrs = at;
    cfg.numAttrs = 1;
    int n = 0;
    if (cudaOccupancyMaxActiveClusters(&n, k_train_persist<InT, CSZ, false, IPC>, &cfg) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return n * CSZ;
}

template <typename InT> const void *persist_fn(int cs, bool direct, int ipc) {
    if (ipc == 2 && cs == PAIR_CS[0])
        return direct ? (const void *)k_train_persist<InT, PAIR_CS[0], true, 2> : (const void *)k_train_persist<InT, PAIR_CS[0], false, 2>;
    if (ipc == 2)
        return direct ? (const void *)k_train_persist<InT, PAIR_CS[1], true, 2> : (const void *)k_train_persist<InT, PAIR_CS[1], false, 2>;
    if (cs > 1)
        return direct ? (const void *)k_train_persist<InT, PERSIST_CS, true, 1> : (const void *)k_train_persist<InT, PERSIST_CS, false, 1>;
    return (const void *)k_train_persist<InT, 1, false, 1>;
}

}  // namespace

int pcnn_persist_configure(pcnn_ctx *ctx) {
    int a = 0, b = 0, rc;
    if ((rc = persist_cap<uint8_t>(&a))) return rc;
    if ((rc = persist_cap<float>(&b))) return rc;
    int per_sm = a < b ? a : b;
    if (per_sm > FUSED_CTAS_PER_SM) per_sm = FUSED_CTAS_PER_SM;
    ctx->persist_cap = per_sm * ctx->sm_count;
    if (ctx->persist_cap > MAX_SLOTS) ctx->persist_cap = MAX_SLOTS;
    {
        const int u = cluster_cap<uint8_t, 1, PERSIST_CS>(ctx->sm_count), f = cluster_cap<float, 1, PERSIST_CS>(ctx->sm_count);
        int cap = u < f ? u : f;
        if (cap > ctx->persist_cap) cap = ctx->persist_cap;
        ctx->persist_cluster_cap = cap - cap % PERSIST_CS;
    }
    {
        const int u = cluster_cap<uint8_t, 2, PAIR_CS[0]>(ctx->sm_count), f = cluster_cap<float, 2, PAIR_CS[0]>(ctx->sm_count);
        const int cap = u < f ? u : f;
        ctx->persist_pair_cap[0] = cap - cap % PAIR_CS[0];
    }
    {
        const int u = cluster_cap<uint8_t, 2, PAIR_CS[1]>(ctx->sm_count), f = cluster_cap<float, 2, PAIR_CS[1]>(ctx->sm_count);
        const int cap = u < f ? u : f;
        ctx->persist_pair_cap[1] = cap - cap % PAIR_CS[1];
    }
    PCNN_CUDA(cudaMalloc((void **)&ctx->d_slots_ll, (size_t)MAX_SLOTS * NPACK * sizeof(llword)));
    PCNN_CUDA(cudaMalloc((void **)&ctx->d_params_ll, (size_t)NPACK * sizeof(llword)));
    PCNN_CUDA(cudaMemset(ctx->d_slots_ll, 0, (size_t)MAX_SLOTS * NPACK * sizeof(llword)));
    PCNN_CUDA(cudaMemset(ctx->d_params_ll, 0, (size_t)NPACK * sizeof(llword)));
    return PCNN_OK;
}

// Grid, cluster size and images per CTA of the dataflow kernel for a per-rank batch of B.  When the batch outnumbers the
// SMs, single-image CTAs would share SMs and do their once-per-step work (parameter fetch, gradient pushes, cluster slot,
// barriers) twice per SM: then one two-image CTA per SM, ceil(B / 2) of them rounded up to whole clusters, in the first of
// the PAIR_CS cluster sizes at which the device keeps that grid co-resident.  Otherwise one image per CTA while the device can hold them, rounded up to whole clusters
// (CTAs without an image still take part in the reduction); clusters of PERSIST_CS whenever the device can keep that grid
// co-resident, otherwise single CTAs.
static void persist_geometry(const pcnn_ctx *ctx, int B, int *grid, int *cs, int *ipc) {
    const int capc = ctx->persist_force_cluster == 1 ? 0 : ctx->persist_cluster_cap;
    *ipc = 1;
    if (B > ctx->sm_count && ctx->persist_force_cluster != 1) {
        for (int k = 0; k < 2; ++k) {
            const int g = ((B + 1) / 2 + PAIR_CS[k] - 1) / PAIR_CS[k] * PAIR_CS[k];
            if (g <= ctx->persist_pair_cap[k]) { *grid = g; *cs = PAIR_CS[k]; *ipc = 2; return; }
        }
    }
    const int want = B < ctx->persist_cap ? B : ctx->persist_cap;
    if (capc >= PERSIST_CS) {
        int g = ((want + PERSIST_CS - 1) / PERSIST_CS) * PERSIST_CS;
        if (g > capc) g = capc;
        // a grid slightly smaller than the batch only means some CTAs take two images; never give up more than 1/8
        if (g >= want || g * 8 >= want * 7) { *grid = g; *cs = PERSIST_CS; return; }
    }
    *grid = want;
    *cs = 1;
}

// nsteps cursor-driven steps of batch B over split `s` in one cooperative launch.  `gate` (optional) makes the kernel wait
// for host-streamed chunks; `step_err_host` (optional, mapped pinned) receives every step's error sum.
int pcnn_persist_run(pcnn_ctx *ctx, const pcnn_split_binding &s, int B, long nsteps, const pcnn_persist_gate *gate,
                     float *step_err_host, int fresh, double *done_host, unsigned done_tag) {
    PCNN_REQUIRE(ctx->persist_cap > 0, PCNN_ERR_STATE, "persistent kernel cannot be co-resident on this device");
    PCNN_REQUIRE(ctx->world == 1 || ctx->p2p_ready, PCNN_ERR_STATE, "persistent multi-GPU steps need pcnn_p2p_attach");
    while (nsteps > 0) {
        const int k = nsteps > 1000000 ? 1000000 : (int)nsteps;   // bounds one launch (and the ids it consumes)
        // tags are unique per context lifetime; long before the 32-bit ids wrap, start over on cleared buffers
        if (ctx->ll_step_id > 0xF0000000u) {
            PCNN_CUDA(cudaMemsetAsync(ctx->d_slots_ll, 0, (size_t)MAX_SLOTS * NPACK * sizeof(llword), ctx->stream));
            PCNN_CUDA(cudaMemsetAsync(ctx->d_params_ll, 0, (size_t)NPACK * sizeof(llword), ctx->stream));
            ctx->ll_step_id = 0;
        }
        PCNN_REQUIRE(ctx->world == 1 || ctx->p2p_step_id <= 0xF0000000u, PCNN_ERR_STATE,
                     "peer-exchange step ids exhausted: pcnn_p2p_detach and attach again on all ranks");
        PersistArgs a{};
        a.images = s.images;
        a.labels = s.labels;
        a.n_total = s.n;
        a.params = ctx->d_params;
        a.grads = ctx->d_grads;
        a.cursor = ctx->d_cursor;
        a.err_total = ctx->d_err_total;
        a.step_err = ctx->d_step_err;
        a.step_idx = ctx->d_step_idx;
        a.abort_flag = ctx->d_abort;
        a.B = B;
        a.nsteps = k;
        a.rank = ctx->rank;
        a.world = ctx->world;
        a.rank_local = s.rank_local ? 1 : 0;
        a.dt = ctx->lr;
        a.inbox = ctx->p2p_inbox;
        for (int q = 0; q < PCNN_MAX_PEERS; ++q) {
            a.peer_inbox[q] = ctx->p2p_peer_inbox[q];
            a.peer_xslots[q] = ctx->p2p_peer_inbox[q] ? reinterpret_cast<llword *>(reinterpret_cast<char *>(ctx->p2p_peer_inbox[q]) + p2p_inbox_bytes()) : nullptr;
        }
        a.xslots = ctx->p2p_inbox ? reinterpret_cast<llword *>(reinterpret_cast<char *>(ctx->p2p_inbox) + p2p_inbox_bytes()) : nullptr;
        a.trace = ctx->d_trace;
        a.slots_ll = ctx->d_slots_ll;
        a.params_ll = ctx->d_params_ll;
        a.step_base = ctx->ll_step_id;
        a.xstep_base = ctx->p2p_step_id;
        // k + 1 ids per launch: the parameters published after the last step (tag base + k + 1) must never look like the
        // first step's parameters of the next launch (pcnn_set_params may have changed them in between)
        ctx->ll_step_id += (unsigned)k + 1u;
        if (ctx->world > 1) ctx->p2p_step_id += (unsigned)k;      // identical on all ranks: same launches after attach
        if (gate) {
            a.ready = gate->flags;
            a.ready_tag = gate->tag;
            a.ready_chunks = gate->chunks;
        }
        a.early = (s.host_resident && !gate) ? 1 : 0;
        a.fresh = fresh;
        fresh = 0;                                                 // a split longer than one launch continues
        a.step_err_host = step_err_host;
        if (step_err_host) step_err_host += k;
        if (nsteps == k) {            // the last launch of this run reports completion
            a.done_host = done_host;
            a.done_tag = done_tag;
        }
        void *args[] = {&a};
        cudaError_t e;
        {
            int grid = 0, cs = 1, ipc = 1;
            persist_geometry(ctx, B, &grid, &cs, &ipc);
            // 2 GPUs: the cluster shares go straight into the peer's memory and the owners gather ranks x clusters slots (one
            // NVLink hop replaces an L2 hop + the separate exchange).  With more GPUs the per-step NVLink volume of that scheme
            // ((N - 1) x 0.6 MB per GPU) grows and the owners exchange their 9.4 KB of sums instead (PCNN_DIRECT_MAX_WORLD)
            a.direct = (ctx->world >= 2 && ctx->world <= PCNN_DIRECT_MAX_WORLD && cs > 1 && grid / cs <= XS_MAXC && grid > 16 &&
                        !ctx->persist_no_direct) ? 1 : 0;
            const bool u8 = s.pixel_type == PCNN_U8;
            const void *fn = u8 ? persist_fn<uint8_t>(cs, a.direct != 0, ipc) : persist_fn<float>(cs, a.direct != 0, ipc);
            cudaLaunchConfig_t cfg = {};
            cfg.gridDim = dim3((unsigned)grid);
            cfg.blockDim = dim3((unsigned)(NT * ipc));
            cfg.dynamicSmemBytes = ipc == 2 ? (u8 ? persist_smem_bytes<uint8_t, 2>() : persist_smem_bytes<float, 2>())
                                            : (u8 ? persist_smem_bytes<uint8_t, 1>() : persist_smem_bytes<float, 1>());
            cfg.stream = ctx->stream;
            cudaLaunchAttribute at[2];
            int na = 0;
            // co-residency of the whole grid is what the polling loops rely on: cooperative launch guarantees it
            // (the launch fails instead of deadlocking when the grid does not fit)
            if (!ctx->persist_no_coop) {
                at[na].id = cudaLaunchAttributeCooperative;
                at[na].val.cooperative = 1;
                ++na;
            }
            if (cs > 1) {
                at[na].id = cudaLaunchAttributeClusterDimension;
                at[na].val.clusterDim.x = (unsigned)cs;
                at[na].val.clusterDim.y = 1;
                at[na].val.clusterDim.z = 1;
                ++na;
            }
            cfg.attrs = at;
            cfg.numAttrs = (unsigned)na;
            e = cudaLaunchKernelExC(&cfg, fn, args);
            if (e != cudaSuccess && cs > 1 && !ctx->persist_no_coop) {
                // a driver that refuses cooperative + cluster launches: the grid was sized by cudaOccupancyMaxActiveClusters,
                // so it is co-resident on an otherwise idle device; remember the choice
                cudaGetLastError();
                ctx->persist_coop_refused = true;
                ctx->persist_no_coop = true;
                cfg.attrs = at + 1;
                cfg.numAttrs = 1;
                e = cudaLaunchKernelExC(&cfg, fn, args);
            }
            ctx->persist_last_cluster = cs;
            ctx->persist_last_grid = grid;
            ctx->persist_last_direct = a.direct;
            ctx->persist_last_ipc = ipc;
        }
        if (e != cudaSuccess) return pcnn_fail_cuda(e, "launch of k_train_persist", __FILE__, __LINE__);
        ctx->launches += 1;
        ctx->persist_used = true;
        nsteps -= k;
    }
    return PCNN_OK;
}

// blocking check of the persistent kernel's abort flag (call after a stream synchronisation)
int pcnn_persist_check(pcnn_ctx *ctx) {
    if (!ctx->persist_used) return PCNN_OK;
    int flag = 0;
    PCNN_CUDA(cudaMemcpy(&flag, ctx->d_abort, sizeof(int), cudaMemcpyDeviceToHost));
    if (flag) {
        cudaMemset(ctx->d_abort, 0, sizeof(int));
        pcnn_set_error("persistent training kernel aborted: %s wait exceeded its cycle budget",
                       flag == 2 ? "peer-GPU exchange" : (flag == 3 ? "host-streamed chunk" :
                       (flag == 4 ? "launched without its cluster dimension; no" : "slot / parameter")));
        return PCNN_ERR_STATE;
    }
    return PCNN_OK;
}

// ------------------------------------------------------------------------------------------ peer memory plumbing
struct p2p_layout {
    static size_t inbox_bytes() { return p2p_inbox_bytes() + p2p_xslots_bytes(); }      // everything a peer may write into
};

extern "C" int pcnn_p2p_export(pcnn_ctx *ctx, void *handle_out, size_t *handle_bytes) {
    PCNN_REQUIRE(ctx && handle_out && handle_bytes, PCNN_ERR_ARG, "pcnn_p2p_export: NULL argument");
    pcnn_device_guard g(ctx->device);
    if (!ctx->p2p_base) {
        PCNN_CUDA(cudaMalloc(&ctx->p2p_base, p2p_layout::inbox_bytes()));
        PCNN_CUDA(cudaMemset(ctx->p2p_base, 0, p2p_layout::inbox_bytes()));
    }
    cudaIpcMemHandle_t h;
    PCNN_CUDA(cudaIpcGetMemHandle(&h, ctx->p2p_base));
    memcpy(handle_out, &h, sizeof(h));
    *handle_bytes = sizeof(h);
    return PCNN_OK;
}

extern "C" int pcnn_p2p_attach(pcnn_ctx *ctx, const void *handles, int rank, int world) {
    PCNN_REQUIRE(ctx && handles, PCNN_ERR_ARG, "pcnn_p2p_attach: NULL argument");
    PCNN_REQUIRE(world >= 1 && world <= PCNN_MAX_PEERS && rank >= 0 && rank < world, PCNN_ERR_ARG,
                 "pcnn_p2p_attach: bad rank %d / world %d (at most %d peers)", rank, world, PCNN_MAX_PEERS);
    PCNN_REQUIRE(ctx->p2p_base, PCNN_ERR_STATE, "pcnn_p2p_attach: call pcnn_p2p_export first");
    PCNN_REQUIRE(!ctx->p2p_ready, PCNN_ERR_STATE, "pcnn_p2p_attach: already attached");
    PCNN_REQUIRE(ctx->world == 1 || (ctx->world == world && ctx->rank == rank), PCNN_ERR_STATE,
                 "pcnn_p2p_attach: rank/world disagree with pcnn_comm_init_rank");
    pcnn_device_guard g(ctx->device);
    const cudaIpcMemHandle_t *hs = reinterpret_cast<const cudaIpcMemHandle_t *>(handles);
    for (int q = 0; q < world; ++q) {
        void *base = ctx->p2p_base;
        if (q != rank) {
            cudaIpcMemHandle_t h;
            memcpy(&h, hs + q, sizeof(h));
            PCNN_CUDA(cudaIpcOpenMemHandle(&base, h, cudaIpcMemLazyEnablePeerAccess));
            ctx->p2p_mapped[q] = base;
        }
        ctx->p2p_peer_inbox[q] = reinterpret_cast<uint2 *>(base);
    }
    ctx->p2p_inbox = ctx->p2p_peer_inbox[rank];
    // exchange ids restart at every attach: all ranks then issue the same distributed launches and agree on them; the
    // caller must barrier between attach and the first distributed step (a peer may still be clearing its inbox)
    PCNN_CUDA(cudaStreamSynchronize(ctx->stream));
    PCNN_CUDA(cudaMemset(ctx->p2p_base, 0, p2p_layout::inbox_bytes()));
    ctx->p2p_step_id = 0;
    ctx->rank = rank;
    ctx->world = world;
    ctx->p2p_ready = true;
    for (auto &kv : ctx->graphs) cudaGraphExecDestroy(kv.second);
    ctx->graphs.clear();
    return PCNN_OK;
}

extern "C" int pcnn_p2p_detach(pcnn_ctx *ctx) {
    PCNN_REQUIRE(ctx, PCNN_ERR_ARG, "pcnn_p2p_detach: ctx is NULL");
    pcnn_device_guard g(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    for (int q = 0; q < PCNN_MAX_PEERS; ++q) {
        if (ctx->p2p_mapped[q]) cudaIpcCloseMemHandle(ctx->p2p_mapped[q]);
        ctx->p2p_mapped[q] = nullptr;
        ctx->p2p_peer_inbox[q] = nullptr;
    }
    if (ctx->p2p_ready && !ctx->nccl_comm) { ctx->rank = 0; ctx->world = 1; }
    ctx->p2p_ready = false;
    return PCNN_OK;
}

// Phase timestamps (ns, %globaltimer) of the first PCNN_TRACE_STEPS steps of the NEXT persistent launches as seen by
// CTA 0: enable with host_out == NULL (allocates and clears the device buffer), read back with host_out != NULL.
extern "C" int pcnn_persist_trace(pcnn_ctx *ctx, long long *host_out, int cap_steps) {
    PCNN_REQUIRE(ctx, PCNN_ERR_ARG, "pcnn_persist_trace: ctx is NULL");
    pcnn_device_guard g(ctx->device);
    const size_t bytes = ((size_t)PCNN_TRACE_STEPS * 6 + (size_t)MAX_SLOTS * 8) * sizeof(long long);
    if (!host_out) {
        if (!ctx->d_trace) PCNN_CUDA(cudaMalloc((void **)&ctx->d_trace, bytes));
        PCNN_CUDA(cudaMemsetAsync(ctx->d_trace, 0, bytes, ctx->stream));
        return PCNN_OK;
    }
    PCNN_REQUIRE(ctx->d_trace, PCNN_ERR_STATE, "pcnn_persist_trace: tracing was not enabled");
    PCNN_CUDA(cudaStreamSynchronize(ctx->stream));
    const int n = cap_steps < PCNN_TRACE_STEPS ? cap_steps : PCNN_TRACE_STEPS;
    PCNN_CUDA(cudaMemcpy(host_out, ctx->d_trace, (size_t)n * 6 * sizeof(long long), cudaMemcpyDeviceToHost));
    return PCNN_OK;
}

// per-CTA stamps of step PCNN_TRACE_STEPS / 2 of the traced launch: rows of 8 (6 phase stamps, SM id, spare)
extern "C" int pcnn_persist_trace_ctas(pcnn_ctx *ctx, long long *host_out, int cap_ctas) {
    PCNN_REQUIRE(ctx && host_out, PCNN_ERR_ARG, "pcnn_persist_trace_ctas: NULL argument");
    PCNN_REQUIRE(ctx->d_trace, PCNN_ERR_STATE, "pcnn_persist_trace_ctas: tracing was not enabled");
    pcnn_device_guard g(ctx->device);
    PCNN_CUDA(cudaStreamSynchronize(ctx->stream));
    const int n = cap_ctas < MAX_SLOTS ? cap_ctas : MAX_SLOTS;
    PCNN_CUDA(cudaMemcpy(host_out, ctx->d_trace + PCNN_TRACE_STEPS * 6, (size_t)n * 8 * sizeof(long long), cudaMemcpyDeviceToHost));
    return PCNN_OK;
}

extern "C" int pcnn_persist_info(pcnn_ctx *ctx, int *out6) {
    PCNN_REQUIRE(ctx && out6, PCNN_ERR_ARG, "pcnn_persist_info: NULL argument");
    out6[0] = ctx->persist_last_grid;
    out6[1] = ctx->persist_last_cluster;
    out6[2] = ctx->persist_cap;
    out6[3] = ctx->persist_cluster_cap;
    out6[4] = PERSIST_CS;
    out6[5] = (ctx->persist_no_coop ? 0 : 1) | (ctx->persist_last_direct ? 2 : 0) | (ctx->persist_last_ipc == 2 ? 4 : 0);
    return PCNN_OK;
}

extern "C" int pcnn_persist_tune(pcnn_ctx *ctx, int max_cluster) {
    PCNN_REQUIRE(ctx, PCNN_ERR_ARG, "pcnn_persist_tune: ctx is NULL");
    PCNN_REQUIRE(max_cluster >= 0 && max_cluster <= 31, PCNN_ERR_ARG,
                 "pcnn_persist_tune: bit mask of 1 (no clusters), 2 (clusters without the cooperative attribute), 4 (host copies before the "
                 "launch), 8 (two-stage exchange also on 2 GPUs), 16 (pinned host images are staged, not pulled by the kernel)");
    ctx->persist_no_direct = (max_cluster & 8) != 0;
    ctx->persist_force_cluster = (max_cluster & 1) ? 1 : 0;
    // the mask is the whole state of the knobs (tune(0) restores the defaults); the automatic causes are kept on their own
    ctx->persist_no_coop = (max_cluster & 2) != 0 || ctx->persist_coop_refused;
    ctx->hs_copies_first = (max_cluster & 4) != 0 || ctx->launch_blocking_env;
    ctx->hs_no_pull = (max_cluster & 16) != 0;
    return PCNN_OK;
}

extern "C" int pcnn_set_step_mode(pcnn_ctx *ctx, int mode) {
    PCNN_REQUIRE(ctx, PCNN_ERR_ARG, "pcnn_set_step_mode: ctx is NULL");
    PCNN_REQUIRE(mode >= PCNN_MODE_AUTO && mode <= PCNN_MODE_PERSISTENT, PCNN_ERR_ARG, "pcnn_set_step_mode: bad mode %d", mode);
    ctx->step_mode = mode;
    return PCNN_OK;
}
