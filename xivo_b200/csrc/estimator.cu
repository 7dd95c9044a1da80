// Estimator-level C ABI (include/xivo_b200_estimator.h): a Batch of independent estimators that
// advance in lock-step.  The host state machines (estimator_host.cpp.inc, tracker_host.cpp.inc) decide; every numeric hot
// loop runs in the CUDA kernels of tracker_kernels.cu / ekf_kernels.cu, batched over sequences.

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstring>
#include <deque>
#include <mutex>
#include <optional>
#include <stdexcept>

#include "../../include/xivo_b200_estimator.h"
#include "ctx.h"
#include "estimator.h"
#include "homography.h"
#include "png.cuh"
#include "prof.h"
#include "workpool.h"

namespace xb {
// Host wall-clock phases go into the same profile report as the kernels ("host:<phase>").
struct HostScope {
  const char* name;
  std::chrono::steady_clock::time_point t0;
  explicit HostScope(const char* n) : name(n), t0(std::chrono::steady_clock::now()) {}
  ~HostScope() {
    if (!Prof::get().enabled.load(std::memory_order_relaxed)) return;
    if (name[0] == 'x' && name[1] == '_') {
      if (Prof::get().fine.load(std::memory_order_relaxed))
        Prof::get().fine_tab.add(name, (unsigned long long)std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - t0).count());
      return;
    }
    Prof::get().add_host(name, std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count());
  }
};
}  // namespace xb

#include "estimator_host.cpp.inc"
#include "tracker_host.cpp.inc"

namespace xb {
extern std::atomic<unsigned long long> g_launches;
// How pinned host frames reach the frame ring: 0 = one gather launch whose SMs read the host memory over PCIe,
// 1 = one cudaMemcpyAsync per frame on the copy engine.  Results are identical; which is faster depends on the
// host's PCIe path, so it is a run-time setting (xivo_set_frame_ingest; initial value from XIVO_ZEROCOPY).
// Default: the copy engine (with the tables of every phase fetched by kernels, DMA frames delay them least).
static std::atomic<int> g_frame_ingest{(getenv("XIVO_ZEROCOPY") && getenv("XIVO_ZEROCOPY")[0] == '1') ? 0 : 1};

// A host table and its device copy, n elements each.  A View does not own them: its tables live inside a Mirror blob (one upload /
// download of the blob then covers several tables).
template <typename T>
struct View {
  T* h = nullptr;
  T* d = nullptr;
  size_t n = 0;
  cudaError_t up(cudaStream_t st, size_t count = 0, size_t off = 0) {
    Prof::get().h2d += (count ? count : n) * sizeof(T);
    return cudaMemcpyAsync(d + off, h + off, (count ? count : n) * sizeof(T), cudaMemcpyHostToDevice, st);
  }
  cudaError_t down(cudaStream_t st, size_t count = 0, size_t off = 0) {
    Prof::get().d2h += (count ? count : n) * sizeof(T);
    return cudaMemcpyAsync(h + off, d + off, (count ? count : n) * sizeof(T), cudaMemcpyDeviceToHost, st);
  }
};

// Pinned host mirror + device array, both zeroed, owned.  fetchable: the host copy is also mapped into the device address space (hd),
// so that its upload can be a kernel that reads it over PCIe (Batch::up_blob).
template <typename T>
struct Mirror : View<T> {
  using View<T>::h;
  using View<T>::d;
  using View<T>::n;
  T* hd = nullptr;
  Mirror() = default;
  Mirror(const Mirror&) = delete;
  Mirror& operator=(const Mirror&) = delete;
  ~Mirror() { release(); }
  void release() {
    if (h) cudaFreeHost(h);
    if (d) cudaFree(d);
    h = d = hd = nullptr;
    n = 0;
  }
  // releases what it held; on failure the mirror is left empty
  bool alloc(size_t count, bool fetchable = false) {
    release();
    if (!count) return true;
    const size_t bytes = count * sizeof(T);
    if (cudaHostAlloc(reinterpret_cast<void**>(&h), bytes, fetchable ? cudaHostAllocMapped : cudaHostAllocDefault) != cudaSuccess) {
      h = nullptr;
      return false;
    }
    memset(h, 0, bytes);
    if ((fetchable && cudaHostGetDevicePointer(reinterpret_cast<void**>(&hd), h, 0) != cudaSuccess) ||
        cudaMalloc(reinterpret_cast<void**>(&d), bytes) != cudaSuccess)
      d = nullptr;
    if (!d || cudaMemset(d, 0, bytes) != cudaSuccess) {
      release();
      return false;
    }
    n = count;
    return true;
  }
};

// Several tables back to back in one fetchable Mirror blob, each padded to a multiple of `pad` bytes, the blob to 16-byte units
// (fetch_kernel's loads).  put() returns a table's offset; with a base (h, d) it also points the table's view there.
struct BlobLayout {
  size_t pad, off = 0;
  unsigned char *h = nullptr, *d = nullptr;
  template <typename T>
  size_t put(View<T>& v, size_t count) {
    const size_t o = off;
    off += (count * sizeof(T) + pad - 1) / pad * pad;
    if (h) { v.h = reinterpret_cast<T*>(h + o); v.d = reinterpret_cast<T*>(d + o); v.n = count; }
    return o;
  }
};
// Allocates blob b for the tables that tables(BlobLayout&) puts, in that order, and binds their views.
template <typename Tables>
static bool carve(Mirror<unsigned char>& b, Tables tables, size_t pad = 16) {
  BlobLayout size{pad};
  tables(size);
  if (!b.alloc((size.off + 15) & ~(size_t)15, true)) return false;
  BlobLayout bind{pad, 0, b.h, b.d};
  tables(bind);
  return true;
}

// Owners of a non-blocking stream and of a timing-free event.
struct Stream {
  cudaStream_t s = nullptr;
  Stream() { cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking); }
  Stream(const Stream&) = delete;
  Stream& operator=(const Stream&) = delete;
  ~Stream() { if (s) cudaStreamDestroy(s); }
  operator cudaStream_t() const { return s; }
};
struct Event {
  cudaEvent_t e = nullptr;
  Event() { cudaEventCreateWithFlags(&e, cudaEventDisableTiming); }
  Event(const Event&) = delete;
  Event& operator=(const Event&) = delete;
  ~Event() { if (e) cudaEventDestroy(e); }
  operator cudaEvent_t() const { return e; }
};

// Completion of a stream without CUDA calls in the wait loop: the driver thread asks the stream to write a ticket number into mapped
// pinned memory behind everything enqueued so far (cuStreamWriteValue32, fetched from the driver at run time; a one-thread kernel where
// the driver lacks it) and then polls that word.  Why: every runtime call of a driver thread contends with the calls of the other
// batches' drivers (the runtime serialises them), and threads spinning on cudaEventQuery slow the issuing threads down further.
typedef CUresult (*StreamWriteValue32Fn)(CUstream, CUdeviceptr, cuuint32_t, unsigned int);
static StreamWriteValue32Fn stream_write_value32() {
  static StreamWriteValue32Fn fn = [] {
    const char* off = getenv("XIVO_NO_STREAM_MEMOPS");
    if (off && off[0] == '1') return (StreamWriteValue32Fn) nullptr;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuStreamWriteValue32", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) { cudaGetLastError(); p = nullptr; }
    return reinterpret_cast<StreamWriteValue32Fn>(p);
  }();
  return fn;
}
// Upload of a host-written table blob by the SMs: 16-byte loads from the mapped pinned copy, stores to the device copy.  Why not the
// copy engine: the frames of a step travel by DMA, and a small cudaMemcpyAsync issued behind that burst waits for it in the engine's
// FIFO, while a kernel that reads the table in place does not queue behind the burst.
// Four loads in flight per thread: the reads cross PCIe (2-3 us each on an idle link, far more while a frame burst holds it), so the
// number of round trips, not the byte count, is what a table upload costs.
__global__ void __launch_bounds__(256) fetch_kernel(const uint4* __restrict__ src, uint4* __restrict__ dst, unsigned n16) {
  const unsigned tile = 4u * blockDim.x;
  for (unsigned base = blockIdx.x * tile; base < n16; base += gridDim.x * tile) {
    uint4 v[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const unsigned i = base + k * blockDim.x + threadIdx.x;
      if (i < n16) v[k] = __ldcv(src + i);
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const unsigned i = base + k * blockDim.x + threadIdx.x;
      if (i < n16) dst[i] = v[k];
    }
  }
}
__global__ void ticket_kernel(unsigned* flag, unsigned value) {
  *flag = value;
  __threadfence_system();
}
struct StreamTicket {
  unsigned* h = nullptr;  // mapped pinned word the stream writes
  unsigned* d = nullptr;  // its device address
  unsigned next = 0;      // last ticket handed out
  StreamTicket() = default;
  StreamTicket(const StreamTicket&) = delete;
  StreamTicket& operator=(const StreamTicket&) = delete;
  ~StreamTicket() { if (h) cudaFreeHost(h); }
  bool alloc() {
    if (cudaHostAlloc(reinterpret_cast<void**>(&h), 64, cudaHostAllocMapped) != cudaSuccess) {
      h = nullptr;
      return false;
    }
    memset(h, 0, 64);
    return cudaHostGetDevicePointer(reinterpret_cast<void**>(&d), h, 0) == cudaSuccess;
  }
  bool reached(unsigned t) const { return (int)(*reinterpret_cast<volatile unsigned*>(h) - t) >= 0; }
};

class Batch {
 public:
  cudaStream_t st1 = nullptr;  // image-tracker stream: the context's stream
  // Per-sequence host logic is independent across sequences: run it on the process-wide worker pool
  // (workpool.h).  CUDA calls stay on the calling thread.
  // An exception thrown by the host state machine (std::out_of_range of a container lookup, std::bad_alloc) must neither reach a
  // worker thread's top frame (std::terminate) nor unwind the publishing frame while workers still hold the job: it is caught per
  // item, recorded, and reported by the next first_error() as a sticky batch error.  On an isolating handle it is a failure of the
  // item's sequence instead (owner(i): idx[i] where the items are sequences, the caller's mapping where they are positions in a list
  // of sequences, -1 where an item belongs to no one sequence and its failure stays the handle's).
  std::atomic<int> pfor_bad{0};
  std::mutex pfor_mu;
  std::string pfor_msg;
  void pfor_record(int seq, const char* what) {
    if (isolate && seq >= 0) {  // only the item of this sequence writes its estimator
      fail_sequence(seq, XIVO_ERR_STATE, std::string("host state machine threw: ") + what);
      return;
    }
    std::lock_guard<std::mutex> lk(pfor_mu);
    if (!pfor_bad.load()) { pfor_msg = what; pfor_bad.store(1); }
  }
  template <typename Fn, typename Owner>
  void pfor(const std::vector<int>& idx, Fn fn, Owner owner) {
    WorkPool::get().pfor((int)idx.size(), [&](int i) {
      try { fn(idx[i], i); }
      catch (const std::exception& ex) { pfor_record(owner(i), ex.what()); }
      catch (...) { pfor_record(owner(i), "unknown exception"); }
    });
  }
  template <typename Fn>
  void pfor(const std::vector<int>& idx, Fn fn) {
    pfor(idx, fn, [&](int i) { return idx[i]; });
  }
  int first_error(const std::vector<int>& idx) {
    if (pfor_bad.load()) return fail(XIVO_ERR_STATE, "host state machine threw: " + pfor_msg);
    for (int b : idx)
      if (est[b]->error) return fail(est[b]->error, est[b]->error_msg);
    return 0;
  }

  // ---- failure isolation (xivo_batch_isolate_failures) -------------------------------------
  // Off: the first error of any sequence ends the call mid-frame for every sequence, and the handle refuses what follows.  On: a
  // sequence's own failure (its estimator's sticky error, an exception of one of its pool items, one of its per-sequence capacities)
  // takes that sequence out of the rest of the frame and out of every later call until it is reset; only a handle-wide failure (CUDA,
  // a shared buffer's capacity) fails the handle (dead).
  bool isolate = false;
  int dead = 0;
  std::string dead_msg;
  void fail_sequence(int b, int code, const std::string& m) {
    Estimator& e = *est[b];
    if (e.error) return;
    e.error = code;
    e.error_msg = m;
  }
  bool seq_failed(int b) const { return isolate && est[b]->error != 0; }
  int n_failed() const {
    int n = 0;
    for (int b = 0; b < B; ++b) n += est[b]->error != 0;
    return n;
  }
  // the sequences whose messages a call takes: every one, except the failed ones of an isolating handle
  std::vector<int> live_sequences() const {
    std::vector<int> v;
    for (int b = 0; b < B; ++b)
      if (!seq_failed(b)) v.push_back(b);
    return v;
  }
  // Every per-sequence entry that a kernel of the rest of this frame reads is zeroed for sequence b (counts, packed-list extents,
  // tracker kinds, pyramid and FAST selectors), so no launch reads its stale entries; the other sequences' offsets stay where they are.
  // Called only while no upload of these host mirrors is in flight (right after a host phase, which follows a wait).
  void quiesce(int b) {
    nfeat.h[b] = 0; nopsJ.h[b] = 0; firstJ.h[b] = 0;
    nsel.h[b] = 0; nopsU.h[b] = 0; firstU.h[b] = 0;
    if (!img_ready) return;
    npts.h[b] = 0; tkind.h[b] = 0; tneed.h[b] = 0; tnnew.h[b] = 0;
    off_cur.h[b] = ~0ull; fast_off.h[b] = ~0ull; frame_ptr.h[b] = nullptr;
    if (desc_on) { nkps.h[b] = 0; nq.h[b] = 0; }
  }
  // Isolating handle: the failed sequences leave `list` and are quiesced.  No-op otherwise.
  void prune(std::vector<int>& list) {
    if (!isolate) return;
    size_t k = 0;
    for (int b : list) {
      if (est[b]->error) quiesce(b);
      else list[k++] = b;
    }
    list.resize(k);
  }
  // Where a host phase of the frame ends: first_error without isolation, prune with it (a handle-wide pool failure still ends the call).
  int settle(std::vector<int>& list) {
    if (!isolate) return first_error(list);
    prune(list);
    return pool_error();
  }
  int pool_error() { return pfor_bad.load() ? fail(XIVO_ERR_STATE, "host state machine threw: " + pfor_msg) : 0; }
  // A message call of an isolating handle: refused once the handle has failed; afterwards a handle-wide failure (rc < 0) fails it, and
  // XIVO_SEQ_FAILED reports sequences that failed during the call.  Without isolation rc passes through.
  int begin_call(const char* what) { return isolate ? refuse_if_failed(what) : 0; }
  int end_call(int rc, int failed_before) {
    if (!isolate) return rc;
    if (rc < 0) {
      if (!dead) { dead = rc; dead_msg = xivo_last_error(); }
      return rc;
    }
    return n_failed() > failed_before ? XIVO_SEQ_FAILED : rc;
  }
  int set_isolation(bool on) {
    if (int rc = refuse_if_failed("isolate_failures")) return rc;
    if (!on && n_failed()) return fail(XIVO_ERR_STATE, "isolate_failures: a sequence has failed; reset it before turning isolation off");
    isolate = on;
    return 0;
  }
  xivo_ctx* ctx;
  int B, N, maxops, max_sub;
  int cov_tc = 0;  // covariance downdate on the tensor cores ("covariance_update": "tf32x3")
  bool use_1pt = false;       // filter-level 1-point RANSAC: the gate phase also returns diag(P), two extra device phases on demand
  DevBuf<double> dP0;         // P_ backup of OnePointRANSAC (BackupState / RestoreState), allocated at the first use
  std::vector<std::vector<Feature*>> table_order;  // per sequence: index space of the device feature table of this frame
  TcOperands tcops;  // its TF32 operand buffers + tensor maps (ekf_cov_tc2_kernel); XIVO_TC_V1=1 keeps the first formulation
  DevBuf<uint32_t> dKt32, dHP32;
  EkfLayout lay;
  std::vector<std::unique_ptr<Estimator>> est;
  // EKF device state
  DevBuf<double> dP, dHP, dKt, dErr;
  DevBuf<FeatJac> dJac;
  Mirror<CameraParams> cam;
  Mirror<double> R, mh, pack;
  View<double> X, groups, fx, fxp;
  View<int> fref, fsind, nfeat, sel, nsel;
  // Host-written tables go down as ONE copy per phase: each phase owns a pinned + device blob, its tables are views into it, and the
  // variable-length table (sub-filter inputs, packed edit list, packed stage records) sits last so that only its used part is copied.
  Mirror<unsigned char> blobS, blobJ, blobU, blobI[2];
  size_t blobS_fixed = 0, blobJ_fixed = 0, blobU_fixed = 0, blobI_fixed = 0;  // bytes in front of the variable-length table
  View<EditOp> opsJ, opsU;              // packed edit lists: filter b owns [first[b], first[b] + nops[b])
  View<int> nopsJ, firstJ, nopsU, firstU;
  View<SubfilterIn> sub_in;
  Mirror<SubfilterOut> sub_out;
  View<ImuStep> stg[2];  // packed Runge-Kutta sub-step records of all filters, two staging halves used alternately
  View<int> stg_first[2], stg_n[2];
  int stg_half = 0;
  unsigned stg_busy[2] = {0, 0};  // st2 ticket after which the half may be refilled (0 = free)
  Mirror<ImuConst> icst;
  Mirror<double> pmm0;      // B x 23 x 23: initial motion covariance of every filter (cov_init_kernel)
  Json cfg0;                // the creation config: what a reset sequence gets when it is given none
  bool sim_depths = false;  // xivo_init_with_sim_depths was called: a reset sequence inherits it
  unsigned reset_busy = 0;  // st2 ticket after which the host mirrors of the last reset's uploads may be rewritten (0 = free)
  StreamTicket tk1, tk2, tkc;  // completion flags of st1 / st2 / st_copy
  // The covariance side (IMU propagation, slot edits, Jacobians, update) runs on its own stream so that it
  // overlaps the image tracker's kernels and host phases, which use ctx->stream.
  Stream st2;
  // Frames are uploaded on their own stream: the message heap releases a frame several messages after it was
  // pushed, so its copy overlaps the tracking of the frame released now.  ring_ev[slot] orders the two.
  Stream st_copy;
  std::vector<Event> ring_ev;
  // tracker device state (allocated at the first image)
  bool img_ready = false;
  int rows = 0, cols = 0, cn = 0, ring_n = 0, max_pts = 0, max_kp = 0;
  PyrDesc pd;
  DevBuf<uint8_t> dRing;  // B x ring_n x img_bytes
  DevBuf<uint8_t> dPyr;   // B x 2 x pd.total
  std::vector<int> ring_next, prev_slot;
  // xivo_batch_visual_meas_png: pinned staging [frame table | IDAT payloads] + its device copy, the decoder's scratch of filtered scanlines
  // and the per-frame status words; all grown on demand to what a call needs
  Mirror<unsigned char> png_stage;
  DevBuf<uint8_t> png_scratch;
  Mirror<int> png_status;
  // xivo_batch_prefetch_frames: host pointers and ring slots of the frames whose upload is already in flight on st_copy
  struct Prefetched { std::vector<const uint8_t*> ptr; std::vector<int> slot; };
  std::deque<Prefetched> pref;  // oldest first; at most two (the frame about to be consumed and the one after it)
  View<unsigned long long> off_prev, off_cur;
  View<uint8_t*> frame_ptr;                    // ring slot of the frame being tracked (written in place by the normalisation)
  View<const uint8_t*> ingest_ptr;             // sources of a device-resident ingest
  View<unsigned long long> ingest_off;
  Mirror<unsigned char> blobG;                 // [ingest_ptr | ingest_off]: one copy per gather launch
  View<float> pts0, pts1;
  Mirror<float> lkerr;
  Mirror<uint8_t> lkst;
  View<int> npts;
  Mirror<int> kpcount;
  Mirror<unsigned> kp;
  // TMA pyramid passes (pyrdown_tma_kernel): tensor maps over the frame ring (level-0 source) and over the pyramid levels
  bool tma_pyr = false;
  CUtensorMap tm_ring;
  CUtensorMap tm_lvl[kMaxPyrLevels];
  bool tm_lvl_ok[kMaxPyrLevels] = {false};
  bool tma_fast = false;  // FAST tiles by TMA (fast_pair_tma_kernel): tensor map over the level-0 images of the pyramid buffer
  CUtensorMap tm_fast;
  View<int> ring_img, pyr_img;  // per sequence: image index of the new frame inside the ring map / of the current pyramid inside the level maps
  // device-side tracker decisions (track_accept_kernel / track_select_kernel)
  bool dev_decide = false;
  View<int> tkind, tneed, tnnew;
  View<uint8_t> tstat;
  View<unsigned> tnewkp;
  View<unsigned long long> fast_off;  // FAST selector: pyramid offset of the sequences that may need a detection
  // descriptor path (tracker.cpp:231-292, :341-460, :530-565): BRIEF-32 at the tracked positions and at the detected keypoints, Hamming
  // nearest neighbours for the cross-checked matcher.  Allocated when the tracker extracts descriptors; decisions then stay on the host.
  bool desc_on = false;
  Mirror<uint8_t> descT, validT;        // B x max_pts (x 32): descriptors at this frame's LK positions
  Mirror<float> kpxy;                   // B x max_kp x 2: detected keypoints in selection order (mask- and border-filtered, sorted)
  Mirror<int> nkps, nq;                 // B
  Mirror<uint8_t> descK, validK, qdesc; // B x max_kp x 32 / B x max_kp / B x max_pts x 32 (queries: descriptors of dropped / existing tracks)
  Mirror<int> bestT_idx, bestT_dist, bestQ_idx, bestQ_dist;  // nearest keypoint of every query; nearest query of every keypoint
  // every table of the tracker phase lives in ONE blob: [inputs | pts1 (in/out) | outputs], so the phase costs one H2D and one D2H call
  Mirror<unsigned char> tt;
  size_t tt_up_bytes = 0, tt_down_off = 0, tt_down_bytes = 0;

  Batch(xivo_ctx* c, const Json& cfg, int nseq, EkfLayout l, bool tracker_only) : ctx(c), B(nseq), lay(l), cfg0(cfg) {
    N = lay.N();
    st1 = ctx->stream;
    for (int b = 0; b < B; ++b) {
      est.emplace_back(new Estimator(cfg, lay, tracker_only));
      est.back()->compact_records = true;  // imu_cov_propagate rebuilds the intermediate Runge-Kutta stages itself
    }
    cov_tc = est[0]->c.cov_update_tf32x3 ? 1 : 0;
    const bool tc2 = cov_tc && !(getenv("XIVO_TC_V1") && getenv("XIVO_TC_V1")[0] == '1');
    if (!tracker_only) {  // an update of 2 * max_features rows must fit the kernels' resident shared-memory working sets (kernels.h)
      const int gain_f = ekf_gain_max_rows(true) / 2, tc2_f = ekf_cov_tc2_max_rows() / 2;
      if (lay.F > gain_f)
        throw std::runtime_error("max_features = " + std::to_string(lay.F) + " exceeds " + std::to_string(gain_f) +
                                 ", the most the gain kernel's shared-memory Cholesky holds");
      if (tc2 && lay.F > tc2_f)
        throw std::runtime_error("max_features = " + std::to_string(lay.F) + " exceeds " + std::to_string(tc2_f) +
                                 ", the most the \"tf32x3\" covariance downdate holds (XIVO_TC_V1=1 selects the first tensor-core kernel, "
                                 "which has no such limit)");
    }
    use_1pt = est[0]->c.use_1pt_RANSAC;
    table_order.resize(B);
    maxops = 4 * (lay.F + lay.G) + 16;
    max_sub = est[0]->tc.num_features_max + 8;
    const size_t nB = (size_t)B, nF = (size_t)B * lay.F;
    bool ok = dP.alloc(nB * N * N) && dHP.alloc(nF * 2 * N) && dKt.alloc(nF * 2 * N) && dErr.alloc(nB * N) && dJac.alloc(nF);
    ok = ok && cam.alloc(B) && R.alloc(B) && mh.alloc(nF + nB * N) && pack.alloc(nB * (2 * N + 529)) && sub_out.alloc(nB * max_sub) &&
         icst.alloc(B) && pmm0.alloc(nB * 529) && tk1.alloc() && tk2.alloc() && tkc.alloc();
    // the per-phase upload blobs and the table views inside them; the variable-length table last
    ok = ok && carve(blobS, [&](BlobLayout& t) {  // sub-filter phase
           t.put(X, nB * kPoseDoubles);
           blobS_fixed = t.put(sub_in, nB * max_sub);
         });
    ok = ok && carve(blobJ, [&](BlobLayout& t) {  // Jacobian / gate phase
           t.put(nfeat, nB); t.put(nopsJ, nB); t.put(firstJ, nB); t.put(fref, nF); t.put(fsind, nF); t.put(fxp, nF * 2); t.put(fx, nF * 3);
           t.put(groups, nB * lay.G * kGroupDoubles);
           blobJ_fixed = t.put(opsJ, nB * maxops);
         });
    ok = ok && carve(blobU, [&](BlobLayout& t) {  // update phase
           t.put(nsel, nB); t.put(nopsU, nB); t.put(firstU, nB); t.put(sel, nF);
           blobU_fixed = t.put(opsU, nB * maxops);
         });
    for (int h = 0; h < 2; ++h)  // IMU sub-step records, two staging halves
      ok = ok && carve(blobI[h], [&](BlobLayout& t) {
             t.put(stg_first[h], nB); t.put(stg_n[h], nB);
             blobI_fixed = t.put(stg[h], nB * kMaxSteps);
           });
    if (ok && tc2) {
      const size_t words = tc_operand_words(N, 2 * lay.F, B);
      ok = dKt32.alloc(words) && dHP32.alloc(words) && cudaMemset(dKt32.p, 0, words * 4) == cudaSuccess && cudaMemset(dHP32.p, 0, words * 4) == cudaSuccess &&
           tc_operands_init(&tcops, N, 2 * lay.F, B, dKt32.p, dHP32.p) == 0;
    }
    if (!ok) throw std::runtime_error(std::string("device allocation failed: ") + cudaGetErrorString(cudaGetLastError()));
    for (int b = 0; b < B; ++b) set_filter_tables(b);
    cam.up(st1);
    R.up(st1);
    icst.up(st1);
    pmm0.up(st1);
    if (launch_cov_init(st1, N, dP.p, pmm0.d, 0, B)) throw std::runtime_error(std::string("initial covariance: ") + cudaGetErrorString(cudaGetLastError()));
    cudaStreamSynchronize(st1);
  }
  // Host mirrors of sequence b's per-filter device tables (camera, measurement noise, IMU constants, initial motion covariance) from
  // est[b], and the diagonal of its initial covariance: identity with the motion block from the config (estimator.cpp:258-302).
  void set_filter_tables(int b) {
    Estimator& e = *est[b];
    cam.h[b] = e.cam;
    R.h[b] = e.c.R;
    ImuConst& ic = icst.h[b];
    memcpy(ic.g, e.c.g.v, 24);
    for (int i = 0; i < 12; ++i) ic.qimu[i] = e.c.Qimu[i * 12 + i];
    for (int i = 0; i < 23; ++i) ic.qmodel[i] = e.c.Qmodel[i * 23 + i];
    ic.stages_per_step = e.c.integration_method == "PrinceDormand" ? 7 : 4;
    ic.pad = 0;
    memcpy(pmm0.h + (size_t)b * 529, e.Pmm, sizeof(e.Pmm));
    for (int i = 0; i < N; ++i) e.diagP[i] = i < 23 ? e.Pmm[i * 23 + i] : 1.0;
  }

  // ---- sequence lifecycle (xivo_batch_reset_sequence) -------------------------------------
  // Sequence `seq` starts over as a freshly created estimator configured by cfg (null: the handle's creation config); the other
  // sequences, their heaps and their frames in the ring are untouched.  Refused without any change when an earlier call failed, when
  // the config does not parse or when it differs from the handle in a batch-wide setting (batch_incompatibility).
  int reset_sequence(int seq, const Json* cfg) {
    if (int rc = refuse_if_failed("reset_sequence")) return rc;
    std::unique_ptr<Estimator> e;
    try {
      e.reset(new Estimator(cfg ? *cfg : cfg0, lay, est[0]->tracker_only));
    } catch (const std::exception& ex) {
      return fail(XIVO_ERR_ARG, std::string("reset_sequence: bad config: ") + ex.what());
    }
    const std::string key = batch_incompatibility(*est[0], *e);
    if (!key.empty()) return fail(XIVO_ERR_ARG, "reset_sequence: \"" + key + "\" differs from the handle's; it must be the same for every sequence of a batch");
    // the host mirrors of the per-filter tables may be rewritten once the uploads of an earlier reset have left them
    if (reset_busy && !tk2.reached(reset_busy))
      if (int rc = wait(st2)) return rc;
    reset_busy = 0;
    e->compact_records = true;
    e->sim_initialize_depths = sim_depths;
    if (img_ready) {  // what ensure_images gives every estimator at the first image
      e->tracker_set_geometry(rows, cols, !dev_decide);
      prev_slot[seq] = 0;
    }
    est[seq] = std::move(e);  // the old estimator's heap, pending propagation records, edits and tracker state go with it
    table_order[seq].clear();
    drop_prefetches();
    set_filter_tables(seq);
    // Device side on st2, in stream order behind the work already queued for the old sequence (an imu_cov_propagate of a frame the heap
    // has released reads icst and P), ahead of everything the new one enqueues.
    XB_CUDA(cam.up(st2, 1, seq));
    XB_CUDA(R.up(st2, 1, seq));
    XB_CUDA(icst.up(st2, 1, seq));
    XB_CUDA(pmm0.up(st2, 529, (size_t)seq * 529));
    if (int rc = launch_cov_init(st2, N, dP.p, pmm0.d, seq, 1)) return rc;
    g_launches += 1;
    reset_busy = tk2.next + 1;  // the next ticket of st2 lies behind these uploads
    return 0;
  }
  // the members free themselves once no queued work can touch them any more
  ~Batch() {
    cudaStreamSynchronize(st1);
    cudaStreamSynchronize(st2);
    cudaStreamSynchronize(st_copy);
  }

  int fail(int code, const std::string& m) {
    set_error("%s", m.c_str());
    return code;
  }
  // XIVO_ERR_STATE once an earlier call on the handle failed: such a call stops mid-frame for every sequence.  On an isolating handle
  // only a handle-wide failure counts: a failed sequence is that sequence's matter.
  int refuse_if_failed(const char* what) {
    if (pfor_bad.load()) return fail(XIVO_ERR_STATE, std::string(what) + ": an earlier call on this handle failed (" + pfor_msg + "); the handle cannot continue");
    if (isolate) {
      if (dead) return fail(XIVO_ERR_STATE, std::string(what) + ": an earlier call on this handle failed (" + dead_msg + "); the handle cannot continue");
      return 0;
    }
    for (int b = 0; b < B; ++b)
      if (est[b]->error)
        return fail(XIVO_ERR_STATE, std::string(what) + ": an earlier call on this handle failed (sequence " + std::to_string(b) + ": " + est[b]->error_msg +
                                        "); the handle cannot continue");
    return 0;
  }
  std::vector<int> every_sequence() const {
    std::vector<int> all(B);
    for (int s = 0; s < B; ++s) all[s] = s;
    return all;
  }

  // ---- staging helpers -------------------------------------------------------------------
  cudaError_t up_blob(Mirror<unsigned char>& b, size_t bytes, cudaStream_t st) {
    Prof::get().h2d += bytes;
    if (!bytes) return cudaSuccess;
    const unsigned n16 = (unsigned)((bytes + 15) / 16);  // blobs are allocated in 16-byte units
    const unsigned ctas = std::max(1u, std::min(64u, (n16 + 1023) / 1024));
    fetch_kernel<<<ctas, 256, 0, st>>>(reinterpret_cast<const uint4*>(b.hd), reinterpret_cast<uint4*>(b.d), n16);
    g_launches += 1;
    return cudaGetLastError();
  }
  // pack the pending covariance edits of the given sequences into ops (filter b: [first[b], first[b] + nops[b])); *total = entries used
  int stage_edits(const std::vector<int>& act, View<EditOp>& ops, View<int>& first, View<int>& nops, int* total) {
    for (int b = 0; b < B; ++b) { nops.h[b] = 0; first.h[b] = 0; }
    int n = 0;
    for (int b : act) {
      auto& e = est[b]->edits;
      if ((int)e.size() > maxops) {  // one sequence's share of the packed list
        if (!isolate) return fail(XIVO_ERR_STATE, "covariance edit list overflow");
        fail_sequence(b, XIVO_ERR_STATE, "covariance edit list overflow");
        continue;
      }
      first.h[b] = n;
      nops.h[b] = (int)e.size();
      for (size_t i = 0; i < e.size(); ++i) ops.h[(size_t)n + i] = e[i];
      n += (int)e.size();
      e.clear();
    }
    *total = n;
    return 0;
  }
  // Enqueue the covariance algebra of the queued Runge-Kutta sub-step records of the given sequences
  // (imu_cov_propagate_kernel).  Asynchronous: the host already holds the propagated nominal state.
  int integrate(const std::vector<int>& act) {
    HostScope hsi("issue_integrate");
    cudaStream_t st = st2;
    bool any = false;
    for (int b : act) any = any || !est[b]->steps.empty();
    if (!any) return 0;
    // A queue longer than the per-filter staging capacity (an IMU / vision gap of several hundred ms: the reference integrates any dt,
    // estimator.cpp:539-592) goes down in several launches of whole sub-steps each; the kernel composes per launch.
    // sub-steps per launch and filter: the integration method (and with it the stages per sub-step) is a per-sequence setting
    auto chunk = [&](int b) { return kMaxStages / std::max(1, icst.h[b].stages_per_step); };
    std::vector<size_t> cur(B, 0);
    for (;;) {
      const int h = stg_half;
      // the staging half may be refilled once st2 has passed the launch that read it: normally the wait that ended the last frame
      if (stg_busy[h] && !tk2.reached(stg_busy[h])) {
        if (int rc = wait(st)) return rc;
      }
      stg_busy[h] = 0;
      for (int b = 0; b < B; ++b) { stg_n[h].h[b] = 0; stg_first[h].h[b] = 0; }
      int total = 0;
      bool more = false;
      for (int b : act) {
        Estimator& e = *est[b];
        const int n = (int)std::min<size_t>((size_t)chunk(b), e.steps.size() - cur[b]);
        if (n <= 0) continue;
        stg_first[h].h[b] = total;
        stg_n[h].h[b] = n;
        total += n;
      }
      if (!total) break;
      // the records themselves (~5 KB per sequence and frame) are copied by the pool, not by the driver thread alone
      pfor(act, [&](int b, int) {
        const int n = stg_n[h].h[b];
        if (n > 0) memcpy(stg[h].h + stg_first[h].h[b], est[b]->steps.data() + cur[b], sizeof(ImuStep) * n);
      });
      for (int b : act) {
        cur[b] += stg_n[h].h[b];
        more = more || cur[b] < est[b]->steps.size();
      }
      XB_CUDA(up_blob(blobI[h], blobI_fixed + (size_t)total * sizeof(ImuStep), st));
      if (int rc = launch_imu_cov_propagate(st, N, dP.p, stg[h].d, stg_first[h].d, stg_n[h].d, icst.d, B)) return rc;
      stg_busy[h] = tk2.next + 1;  // the next ticket of st2 lies behind this launch
      stg_half ^= 1;
      g_launches += 1;
      {
        int nact = 0;
        for (int b = 0; b < B; ++b) nact += stg_n[h].h[b] > 0;
        // algorithmic bytes: the sub-step records + the motion block read and written + the 23 x (N-23) strip read, 9 rows of it written (twice: mirrored)
        Prof::get().add_work("imu_cov_propagate", total * (double)sizeof(ImuStep) + nact * 8.0 * (2 * 529 + (23 + 18) * (double)(N - 23)));
      }
      if (!more) break;
    }
    for (int b : act) {
      est[b]->steps.clear();
      est[b]->prop_pending = false;
    }
    return 0;
  }
  // apply pending propagation + edits of the given sequences (used before state / P read-back)
  int flush(const std::vector<int>& act) {
    cudaStream_t st = st2;
    if (int rc = integrate(act)) return rc;
    int nops_total = 0;
    if (int rc = stage_edits(act, opsJ, firstJ, nopsJ, &nops_total)) return rc;
    XB_CUDA(up_blob(blobJ, blobJ_fixed + (size_t)nops_total * sizeof(EditOp), st));
    if (int rc = launch_cov_edit(st, N, dP.p, opsJ.d, nopsJ.d, maxops, B, firstJ.d)) return rc;
    g_launches += 1;
    { HostScope hw("wait_flush"); if (int rc = wait(st)) return rc; }
    return 0;
  }

  // Wait until everything enqueued on st1 / st2 so far has completed, without idling the CPU: the stream writes a ticket into mapped
  // host memory (StreamTicket); while it is pending the driver executes items of whatever host jobs the other batches of this process
  // have published.  No CUDA call sits in the loop (a stream query every ~2^16 polls only catches a faulted context).
  int wait(cudaStream_t st) {
    static const bool help = !(getenv("XIVO_HELP") && getenv("XIVO_HELP")[0] == '0');
    StreamTicket& t = st == st2 ? tk2 : st == st_copy ? tkc : tk1;
    const unsigned want = ++t.next;
    std::unique_ptr<HostScope> hx_t(new HostScope("x_i_ticket"));
    if (StreamWriteValue32Fn wv = stream_write_value32()) {
      if (wv(reinterpret_cast<CUstream>(st), reinterpret_cast<CUdeviceptr>(t.d), want, 0) != CUDA_SUCCESS) {
        set_error("cuStreamWriteValue32 failed");
        return XIVO_ERR_CUDA;
      }
    } else {
      ticket_kernel<<<1, 1, 0, st>>>(t.d, want);
      XB_CUDA(cudaGetLastError());
    }
    hx_t.reset();
    unsigned polls = 0;
    while (!t.reached(want)) {
      if (help && WorkPool::get().help_one()) continue;
      cpu_relax();
      if ((++polls & 0xffffu) == 0) {
        const cudaError_t e = cudaStreamQuery(st);
        if (e != cudaSuccess && e != cudaErrorNotReady) { set_error("CUDA error while waiting: %s", cudaGetErrorString(e)); return XIVO_ERR_CUDA; }
      }
    }
    std::atomic_thread_fence(std::memory_order_acquire);  // the copies that precede the ticket in the stream are visible now
    return 0;
  }
  // Bring one frame per sequence into its ring slot (slot_of[s]) on the copy stream.  Device frames and
  // device-accessible host frames (pinned / registered: the SMs read them over PCIe) take one gather launch,
  // which keeps the H2D copy engine's FIFO free for the small latency-critical table uploads of the other
  // phases; pageable host frames fall back to one cudaMemcpyAsync each.
  // Device address of a host frame the SMs can read in place (pinned / registered memory), or null.  The answer is cached per
  // allocation (cuMemGetAddressRange gives its extent): one driver query per pinned pool instead of one runtime call per frame per step.
  struct HostRange { uintptr_t lo, hi; ptrdiff_t dev_minus_host; };
  std::vector<HostRange> host_ranges;
  const uint8_t* mapped_host_pointer(const uint8_t* p, size_t bytes) {
    const uintptr_t a = reinterpret_cast<uintptr_t>(p);
    for (const HostRange& r : host_ranges)
      if (a >= r.lo && a + bytes <= r.hi) return reinterpret_cast<const uint8_t*>(a + r.dev_minus_host);
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, p) != cudaSuccess || at.type == cudaMemoryTypeUnregistered || !at.devicePointer) {
      cudaGetLastError();  // clear the sticky "invalid value" of an unregistered pointer
      return nullptr;
    }
    typedef CUresult (*RangeFn)(CUdeviceptr*, size_t*, CUdeviceptr);
    static RangeFn range_fn = [] {
      void* f = nullptr;
      cudaDriverEntryPointQueryResult q;
      if (cudaGetDriverEntryPoint("cuMemGetAddressRange", &f, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) { cudaGetLastError(); f = nullptr; }
      return reinterpret_cast<RangeFn>(f);
    }();
    const uintptr_t da = reinterpret_cast<uintptr_t>(at.devicePointer);
    CUdeviceptr base = 0;
    size_t size = 0;
    if (range_fn && range_fn(&base, &size, (CUdeviceptr)da) == CUDA_SUCCESS && base && size && da >= (uintptr_t)base && da + bytes <= (uintptr_t)base + size) {
      const ptrdiff_t d = (ptrdiff_t)da - (ptrdiff_t)a;
      if (host_ranges.size() >= 64) host_ranges.clear();
      host_ranges.push_back(HostRange{(uintptr_t)base - d, (uintptr_t)base - d + size, d});
    }
    return static_cast<const uint8_t*>(at.devicePointer);
  }
  // The next ring slot of every sequence in `seqs` (slot_of is indexed by sequence; the others' entries are left alone).
  void fresh_slots(const std::vector<int>& seqs, std::vector<int>& slot_of) {
    for (int s : seqs) {
      const int slot = ring_next[s];
      ring_next[s] = (slot + 1) % ring_n;
      slot_of[s] = slot;
    }
  }
  // pending prefetches are abandoned and their slots handed out again (st_copy is in order: a new upload lands after the abandoned ones)
  void drop_prefetches() {
    if (pref.empty()) return;
    for (int s = 0; s < B; ++s) ring_next[s] = pref.front().slot[s];
    pref.clear();
  }
  // Ring slots of the frame about to be ingested.  If the oldest pending xivo_batch_prefetch_frames call brought exactly these host buffers,
  // their upload is already enqueued (*uploaded = true) and its slots are taken over; otherwise every pending prefetch is abandoned and its
  // slots are handed out again (st_copy is in order: the new upload lands after the abandoned ones).
  // Fresh slots go to the sequences in `seqs` only (a failed sequence of an isolating handle takes none; its prefetched copy is ignored).
  void take_slots(const uint8_t* const* imgs, bool on_device, const std::vector<int>& seqs, std::vector<int>& slot_of, bool* uploaded) {
    bool match = !pref.empty() && !on_device;
    if (match)
      for (int s = 0; s < B; ++s)
        if (pref.front().ptr[s] != imgs[s]) { match = false; break; }
    if (match) {
      slot_of = pref.front().slot;
      pref.pop_front();
      *uploaded = true;
      return;
    }
    drop_prefetches();
    fresh_slots(seqs, slot_of);
    *uploaded = false;
  }
  int prefetch_frames(const uint8_t* const* imgs, size_t ib) {
    if (pref.size() >= 2) return fail(XIVO_ERR_STATE, "prefetch_frames: two prefetched frames are pending already (consume one with a step / visual_meas call first)");
    Prefetched p;
    p.slot.resize(B);
    const std::vector<int> all = every_sequence();
    fresh_slots(all, p.slot);
    if (int rc = upload_frames(imgs, all, p.slot, false, ib)) return rc;
    p.ptr.assign(imgs, imgs + B);
    pref.push_back(std::move(p));
    return 0;
  }
  // The frames of the sequences in `seqs` (imgs[s] into ring slot slot_of[s]) go down on st_copy; the other sequences' entries are not read.
  int upload_frames(const uint8_t* const* imgs, const std::vector<int>& seqs, const std::vector<int>& slot_of, bool on_device, size_t ib) {
    HostScope hsu("issue_upload_frames");
    const bool zero_copy = g_frame_ingest.load(std::memory_order_relaxed) == 0;
    bool gather = on_device || zero_copy;
    const int n = (int)seqs.size();
    if (!n) return 0;
    // compacted [source, ring offset] list of the present frames
    for (int i = 0; i < n; ++i) {
      const int s = seqs[i];
      ingest_off.h[i] = ((size_t)s * ring_n + slot_of[s]) * ib;
      ingest_ptr.h[i] = imgs[s];
      if (!on_device && gather) {
        if (i == 0) host_ranges.clear();  // one real query per call keeps the cache honest if the caller re-pins / frees its pool between steps
        const uint8_t* dp = mapped_host_pointer(imgs[s], ib);
        if (!dp) gather = false;
        else ingest_ptr.h[i] = dp;
      }
    }
    if (!on_device) Prof::get().h2d += (unsigned long long)ib * n;
    if (gather) {
      XB_CUDA(up_blob(blobG, blobG.n, st_copy));  // [sources | ring offsets]
      // host sources: one warp per frame with four loads in flight still fills the link when several batches pull at once, and hogs it
      // less for the other batches' table fetches than wider grids do
      if (int rc = launch_gather_frames(st_copy, ingest_ptr.d, dRing.p, 0, ingest_off.d, ib, n, on_device ? 64 : 1, on_device ? 256 : 32)) return rc;
      g_launches += 1;
    } else {
      // copy engine: runs of consecutive sequences whose sources are evenly spaced (frames of one pinned pool) and whose ring slots agree
      // go down as ONE pitched copy each (far fewer copy calls than one per frame)
      auto next_in_run = [&](int i, int j) { return seqs[j] == seqs[i] + 1 && slot_of[seqs[j]] == slot_of[seqs[i]] && imgs[seqs[j]] > imgs[seqs[i]]; };
      int i = 0;
      while (i < n) {
        int e = i + 1;
        if (e < n && next_in_run(i, e)) {
          const size_t stride = (size_t)(imgs[seqs[e]] - imgs[seqs[i]]);
          if (stride >= ib) {
            while (e + 1 < n && next_in_run(e, e + 1) && (size_t)(imgs[seqs[e + 1]] - imgs[seqs[e]]) == stride) ++e;
            ++e;
            XB_CUDA(cudaMemcpy2DAsync(dRing.p + ingest_off.h[i], (size_t)ring_n * ib, imgs[seqs[i]], stride, ib, (size_t)(e - i), cudaMemcpyHostToDevice,
                                      st_copy));
            i = e;
            continue;
          }
        }
        XB_CUDA(cudaMemcpyAsync(dRing.p + ingest_off.h[i], imgs[seqs[i]], ib, cudaMemcpyHostToDevice, st_copy));
        ++i;
      }
    }
    return ring_uploaded(distinct_slots(seqs, slot_of));
  }
  // the distinct ring slots of the frames of `seqs`
  static std::vector<int> distinct_slots(const std::vector<int>& seqs, const std::vector<int>& slot_of) {
    std::vector<int> used;
    for (int s : seqs)
      if (std::find(used.begin(), used.end(), slot_of[s]) == used.end()) used.push_back(slot_of[s]);
    return used;
  }
  // mark the uploads enqueued on st_copy for ring slot `slot` (call after the last one)
  int ring_uploaded(const std::vector<int>& slots_used) {
    for (int k : slots_used) XB_CUDA(cudaEventRecord(ring_ev[k], st_copy));
    return 0;
  }
  // the caller's frame buffers are free again once THEIR uploads have landed (the events of the ring slots they went to: a prefetched copy
  // of the next frame may already be queued behind them on st_copy and must not be waited for)
  int ingest_done(const std::vector<int>& seqs, const std::vector<int>& slot_of) {
    HostScope hsw("wait_ingest_done");
    for (int k : distinct_slots(seqs, slot_of)) XB_CUDA(cudaEventSynchronize(ring_ev[k]));
    return 0;
  }

  // PNG frames (xivo_batch_visual_meas_png): the host walks the chunks of every sequence's file and packs the IDAT payloads of all of them,
  // with one PngFrameDesc per frame, into the pinned staging blob (in parallel on the worker pool); ONE upload on st_copy, then
  // png_inflate_kernel + png_unfilter_kernel decode straight into the ring slots of the frames and ring_ev[slot] is recorded after them,
  // so the tracker stream orders on the decode like on an upload.  The status words come back on st_copy before any message is pushed:
  // a refused frame (host- or device-detected) leaves ring_next as the call found it and changes no sequence.  Only the frames of the
  // sequences in `seqs` are read (png_data / png_bytes / slot_of are indexed by sequence); the descriptors, the scratch space and the status
  // words cover those frames alone.  slot_of[s] = the slot of sequence s's frame.
  int decode_png_frames(const std::vector<int>& seqs, const uint8_t* const* png_data, const size_t* png_bytes, int channels, std::vector<int>& slot_of) {
    const int n = (int)seqs.size();
    if (!n) return 0;
    std::vector<png::Info> info(n);
    std::vector<const char*> why(n, nullptr);
    std::vector<size_t> zlen(n, 0);
    std::vector<int> idx(n);
    for (int i = 0; i < n; ++i) idx[i] = i;
    {
      HostScope hp("png_parse");
      pfor(idx, [&](int i, int) {
        const int s = seqs[i];
        const char* w = "";
        size_t z = 0;
        if (png::parse(png_data[s], png_bytes[s], info[i], &w, [&](size_t, size_t len) { z += len; })) why[i] = w;
        zlen[i] = z;
      }, [](int) { return -1; });  // the frames go down in one shared decode launch: a failure here is the handle's
      if (pfor_bad.load()) return fail(XIVO_ERR_STATE, "host state machine threw: " + pfor_msg);
    }
    for (int i = 0; i < n; ++i) {
      const std::string frame = "png frame " + std::to_string(seqs[i]);
      if (why[i]) return fail(XIVO_ERR_ARG, frame + ": " + why[i]);
      if (channels == 1 && info[i].channels > 2)
        return fail(XIVO_ERR_ARG, frame + ": 1-channel output needs a grey or grey + alpha PNG (colour type " + std::to_string(info[i].color_type) + ")");
      if (info[i].rows != info[0].rows || info[i].cols != info[0].cols)
        return fail(XIVO_ERR_ARG, frame + " is " + std::to_string(info[i].rows) + " x " + std::to_string(info[i].cols) + ", frame " + std::to_string(seqs[0]) +
                                      " is " + std::to_string(info[0].rows) + " x " + std::to_string(info[0].cols) + ": all sequences of a batch share one geometry");
    }
    if (img_ready && (info[0].rows != rows || info[0].cols != cols))
      return fail(XIVO_ERR_ARG, "png frame " + std::to_string(seqs[0]) + " is " + std::to_string(info[0].rows) + " x " + std::to_string(info[0].cols) +
                                    ", the handle's frames are " + std::to_string(rows) + " x " + std::to_string(cols));
    if (int rc = ensure_images(info[0].rows, info[0].cols, channels)) return rc;
    const size_t ib = (size_t)rows * cols * cn;
    const size_t table = ((size_t)n * sizeof(PngFrameDesc) + 15) & ~(size_t)15;
    std::vector<size_t> zoff(n), soff(n);
    size_t zsum = 0, scratch = 0;
    for (int i = 0; i < n; ++i) {
      zoff[i] = zsum;
      zsum += zlen[i];
      soff[i] = scratch;
      scratch += (size_t)info[i].raw_bytes();
    }
    const size_t stage_bytes = table + zsum;
    // grown to 1.25 x the need: frames of one sequence compress to similar sizes
    if (png_stage.n < stage_bytes && !png_stage.alloc(stage_bytes + stage_bytes / 4)) return fail(XIVO_ERR_CUDA, "png staging allocation failed");
    if (png_scratch.n < scratch && !png_scratch.alloc(scratch + scratch / 4)) return fail(XIVO_ERR_CUDA, "png scratch allocation failed");
    if (png_status.n < (size_t)n && !png_status.alloc(B)) return fail(XIVO_ERR_CUDA, "png status allocation failed");
    // pending prefetches are dropped as for any call with other buffers; ring_next after that is what a refusal restores
    drop_prefetches();
    const std::vector<int> ring_before = ring_next;
    fresh_slots(seqs, slot_of);
    PngFrameDesc* fr = reinterpret_cast<PngFrameDesc*>(png_stage.h);
    {
      HostScope hk("png_pack");
      pfor(idx, [&](int i, int) {
        const int s = seqs[i];
        uint8_t* dst = png_stage.h + table + zoff[i];
        png::Info I;
        const char* w = "";
        png::parse(png_data[s], png_bytes[s], I, &w, [&](size_t off, size_t len) { memcpy(dst, png_data[s] + off, len); dst += len; });
        PngFrameDesc& d = fr[i];
        d.in_off = zoff[i];
        d.in_len = zlen[i];
        d.scratch_off = soff[i];
        d.out_off = ((size_t)s * ring_n + slot_of[s]) * ib;
        d.rows = I.rows;
        d.cols = I.cols;
        d.bpp = I.bpp;
        d.channels = I.channels;
        d.bps = I.bit_depth / 8;
        d.oc = channels;
      }, [](int) { return -1; });
      if (pfor_bad.load()) return fail(XIVO_ERR_STATE, "host state machine threw: " + pfor_msg);
    }
    {
      HostScope hu("png_issue");
      XB_CUDA(png_stage.up(st_copy, stage_bytes));
      if (int rc = launch_png_decode(st_copy, png_stage.d + table, png_scratch.p, dRing.p, reinterpret_cast<const PngFrameDesc*>(png_stage.d), n,
                                     png_status.d))
        return rc;
      XB_CUDA(png_status.down(st_copy, n));
      if (int rc = ring_uploaded(distinct_slots(seqs, slot_of))) return rc;
    }
    { HostScope hw("wait_png"); if (int rc = wait(st_copy)) return rc; }
    for (int i = 0; i < n; ++i)
      if (png_status.h[i] != png::kOk) {
        ring_next = ring_before;
        return fail(XIVO_ERR_ARG, "png frame " + std::to_string(seqs[i]) + ": " + png::status_text(png_status.h[i]));
      }
    return 0;
  }

  // ---- image tracker ---------------------------------------------------------------------
  int ensure_images(int r, int c, int ch) {
    if (img_ready) {
      if (r != rows || c != cols || ch != cn) return fail(XIVO_ERR_ARG, "image geometry changed between frames");
      return 0;
    }
    Estimator& e0 = *est[0];
    if (ch != 1 && ch != 3) return fail(XIVO_ERR_ARG, "images must have 1 or 3 channels");
    if (e0.cam.rows > 0 && e0.cam.cols > 0 && (r != e0.cam.rows || c != e0.cam.cols))  // Tracker::Tracker sizes its mask from camera_cfg (tracker.cpp:119-127)
      return fail(XIVO_ERR_ARG, "image is " + std::to_string(r) + " x " + std::to_string(c) + " but camera_cfg says " + std::to_string(e0.cam.rows) + " x " + std::to_string(e0.cam.cols));
    rows = r; cols = c; cn = ch;
    pd = make_pyr_desc(rows, cols, cn, e0.tc.win_size, e0.tc.max_level);
    ring_n = e0.c.message_buffer_size + 2;
    max_pts = e0.tc.num_features_max + 8;
    max_kp = std::max(4096, std::min(1 << 16, rows * cols / 8));
    const size_t ib = (size_t)rows * cols * cn;
    const size_t nB = (size_t)B, npt = (size_t)B * max_pts, nk = (size_t)B * max_kp;
    bool ok = dRing.alloc(nB * ring_n * ib) && dPyr.alloc(nB * 2 * pd.total);
    // [sources | ring offsets], 8-byte entries back to back
    ok = ok && carve(blobG, [&](BlobLayout& t) { t.put(ingest_ptr, nB); t.put(ingest_off, nB); }, 8);
    ok = ok && lkerr.alloc(npt) && lkst.alloc(npt) && kpcount.alloc(B) && kp.alloc(nk);
    // the accept / select decisions run on the device unless the homography stage (host code between the two) is on, the mask does
    // not fit into shared memory, or XIVO_HOST_TRACKER_DECISIONS=1 asks for the host path (parity tests compare the two)
    {
      const char* hd = getenv("XIVO_HOST_TRACKER_DECISIONS");
      dev_decide = !e0.tc.do_outlier_rejection && !e0.tc.extract_descriptor && track_mask_bytes(rows, cols) <= 200 * 1024 && max_pts <= 1024 && !(hd && hd[0] == '1');
    }
    desc_on = e0.tc.extract_descriptor;
    norm_on = e0.tc.normalize;
    if (ok && norm_on) ok = norm_part.alloc(nB * kNormMaxChunks);
    if (ok && desc_on)
      ok = descT.alloc(npt * 32) && validT.alloc(npt) && kpxy.alloc(nk * 2) && nkps.alloc(B) && nq.alloc(B) && descK.alloc(nk * 32) && validK.alloc(nk) &&
           qdesc.alloc(npt * 32) && bestT_idx.alloc(npt) && bestT_dist.alloc(npt) && bestQ_idx.alloc(nk) && bestQ_dist.alloc(nk);
    // the tracker-phase tables: [inputs | pts1 (in/out) | outputs]; the upload covers inputs + pts1, the read-back pts1 + outputs
    ok = ok && carve(tt, [&](BlobLayout& t) {
           t.put(pts0, npt * 2); t.put(off_cur, nB); t.put(off_prev, nB); t.put(fast_off, nB); t.put(npts, nB); t.put(frame_ptr, nB);
           t.put(ring_img, nB); t.put(pyr_img, nB); t.put(tkind, nB);
           tt_down_off = t.put(pts1, npt * 2);
           tt_up_bytes = t.put(tstat, npt);
           t.put(tneed, nB); t.put(tnnew, nB); t.put(tnewkp, nB * e0.tc.num_features_max);
           tt_down_bytes = t.off - tt_down_off;
         });
    if (!ok) return fail(XIVO_ERR_CUDA, "device allocation for the image tracker failed");
    {  // TMA passes where the geometry allows (XIVO_PYRDOWN_TMA=0 / XIVO_FAST_TMA=0 keep the thread-staged kernels: parity tests compare the two)
      const char* tv = getenv("XIVO_PYRDOWN_TMA");
      const char* gv = getenv("XIVO_PYRDOWN_GENERIC");
      const char* fv = getenv("XIVO_FAST_TMA");
      if (cn == 1 && (cols & 15) == 0 && (pd.total & 15) == 0 && (pd.off[0] & 15) == 0 && !(fv && fv[0] == '0'))
        tma_fast = make_fast_tensor_map(&tm_fast, dPyr.p + pd.off[0], rows, cols, pd.total, (unsigned long long)B * 2) == 0;
      if (cn == 1 && (cols & 15) == 0 && (pd.total & 15) == 0 && pd.n_levels > 1 && !(tv && tv[0] == '0') && !(gv && gv[0] == '1')) {
        if (make_pyr_tensor_map(&tm_ring, dRing.p, rows, cols, ib, (unsigned long long)B * ring_n) == 0) {
          tma_pyr = true;
          for (int l = 1; l + 1 < pd.n_levels; ++l)
            tm_lvl_ok[l] = (pd.cols[l] & 15) == 0 && (pd.off[l] & 15) == 0 &&
                           make_pyr_tensor_map(&tm_lvl[l], dPyr.p + pd.off[l], pd.rows[l], pd.cols[l], pd.total, (unsigned long long)B * 2) == 0;
        }
      }
    }
    ring_next.assign(B, 0);
    ring_ev = std::vector<Event>(ring_n);
    prev_slot.assign(B, 0);
    for (auto& e : est) e->tracker_set_geometry(rows, cols, !dev_decide);
    img_ready = true;
    return 0;
  }

  // The frame of every sequence in `act` (ring slot slots[i]) goes into the free half of the sequence's pyramid buffer: the tracker stream
  // waits for the slots' uploads; off_cur / off_prev / frame_ptr (and the TMA image indices) of the sequences, ~0 / 0 / null for the others.
  int begin_frame(const std::vector<int>& act, const std::vector<int>& slots) {
    const size_t ib = (size_t)rows * cols * cn;
    for (int b = 0; b < B; ++b) { off_cur.h[b] = ~0ull; off_prev.h[b] = 0; npts.h[b] = 0; frame_ptr.h[b] = nullptr; }
    std::vector<char> seen(ring_n, 0);
    for (int k : slots)
      if (!seen[k]) { seen[k] = 1; XB_CUDA(cudaStreamWaitEvent(st1, ring_ev[k], 0)); }
    for (size_t i = 0; i < act.size(); ++i) {
      const int b = act[i];
      const int cur = 1 - prev_slot[b];
      off_cur.h[b] = ((size_t)b * 2 + cur) * pd.total;
      off_prev.h[b] = ((size_t)b * 2 + prev_slot[b]) * pd.total;
      frame_ptr.h[b] = dRing.p + ((size_t)b * ring_n + slots[i]) * ib;  // consumed by the first pyrDown pass
      if (tma_pyr) { ring_img.h[b] = b * ring_n + slots[i]; pyr_img.h[b] = b * 2 + cur; }
    }
    return 0;
  }
  // The pyramid passes of the frames begun by begin_frame: every level (LK), or level 0 only (MATCH: the image FAST and BRIEF read).
  // With tracker_cfg.normalize each of those frames is first normalised in its ring slot (frame_ptr, null for the others): the slot is
  // the library's own copy of the frame whatever the ingest path, so the caller's memory is never written.
  int build_pyramids(bool all_levels) {
    if (norm_on) {
      if (int rc = launch_normalize_minmax(st1, frame_ptr.d, (size_t)rows * cols * cn, B, norm_part.p)) return rc;
      g_launches += 2;
    }
    if (tma_pyr) {
      std::optional<ProfScope> ps;
      if (all_levels) ps.emplace("pyrdown", st1);
      if (int rc = launch_pyrdown_tma(st1, tm_ring, ring_img.d, dPyr.p, 0, off_cur.d, pd, 0, 1, B)) return rc;
      for (int l = 1; all_levels && l + 1 < pd.n_levels; ++l) {
        if (tm_lvl_ok[l]) { if (int rc = launch_pyrdown_tma(st1, tm_lvl[l], pyr_img.d, dPyr.p, 0, off_cur.d, pd, l, 0, B)) return rc; }
        else if (int rc = launch_pyrdown_level(st1, dPyr.p, 0, off_cur.d, pd, B, nullptr, l)) return rc;
      }
    } else if (int rc = all_levels ? launch_build_pyramid(st1, dPyr.p, 0, off_cur.d, pd, B, frame_ptr.d) : launch_pyrdown_level(st1, dPyr.p, 0, off_cur.d, pd, B, frame_ptr.d, 0))
      return rc;
    g_launches += all_levels ? std::max(1, pd.n_levels - 1) : 1;
    return 0;
  }
  // FAST on the level-0 images that sel selects (device pyramid offsets, ~0 = skip), then the keypoint counts and the keypoints of `seqs`.
  int detect_and_fetch(const std::vector<int>& seqs, const unsigned long long* sel) {
    cudaStream_t st = st1;
    const TrackerCfg& tc = est[0]->tc;
    if (int rc = launch_fast_detect(st, dPyr.p, 0, sel, rows, cols, cn, tc.fast_threshold, tc.fast_nonmax, kp.d, max_kp, kpcount.d, B, nullptr,
                                    tma_fast ? &tm_fast : nullptr, pd.total))
      return rc;
    g_launches += 1;
    XB_CUDA(kpcount.down(st));
    { HostScope hw("wait_fastcount"); if (int rc = wait(st)) return rc; }
    for (int b : seqs) {
      const int n = std::min(kpcount.h[b], max_kp);
      if (n) { Prof::get().d2h += sizeof(unsigned) * n; XB_CUDA(cudaMemcpyAsync(kp.h + (size_t)b * max_kp, kp.d + (size_t)b * max_kp, sizeof(unsigned) * n, cudaMemcpyDeviceToHost, st)); }
    }
    HostScope hw("wait_fastkp");
    return wait(st);
  }
  // LK of the staged points (pts0 -> pts1) from the previous to the current pyramid of every sequence with npts > 0
  int track_lk(const std::vector<int>& lk_list) {
    const TrackerCfg& tc = est[0]->tc;
    if (int rc = launch_lk_track(st1, dPyr.p, dPyr.p, 0, off_prev.d, off_cur.d, pd, pts0.d, pts1.d, lkst.d, lkerr.d, npts.d, max_pts, B, tc.win_size, tc.max_iter,
                                 tc.eps, 1, 1e-4))
      return rc;
    g_launches += 1;
    double np_ = 0;
    for (int b : lk_list) np_ += npts.h[b];
    Prof::get().add_work("lk_track", np_ * pd.n_levels * (17.0 * 17.0 + 25.0 * 25.0) * cn);  // §8d: L (17^2+25^2) c bytes / feature
    return 0;
  }
  void swap_pyramids(const std::vector<int>& act) {
    for (int b : act)
      if (off_cur.h[b] != ~0ull) prev_slot[b] = 1 - prev_slot[b];  // std::swap(pyramid, pyramid_)
  }
  // cross-checked matches of sequence b from the nearest-neighbour tables of describe_and_match
  void matches_of(int b, std::vector<std::array<int, 3>>* m) const {
    cross_checked(nq.h[b], bestT_idx.h + (size_t)b * max_pts, bestT_dist.h + (size_t)b * max_pts, bestQ_idx.h + (size_t)b * max_kp, m);
  }

  // BRIEF at the ordered keypoints of `seqs` (level-0 image of the current pyramid: sel_off) and, where a sequence has query descriptors
  // (Estimator::query_feats), the two nearest-neighbour tables of the cross-checked matcher.  One wait.
  int describe_and_match(const std::vector<int>& seqs, const unsigned long long* sel_off_dev) {
    cudaStream_t st = st1;
    bool any_q = false;
    for (int b = 0; b < B; ++b) nq.h[b] = 0;
    for (int b : seqs) {
      const int n = nkps.h[b];
      if (n) XB_CUDA(cudaMemcpyAsync(kpxy.d + (size_t)b * max_kp * 2, kpxy.h + (size_t)b * max_kp * 2, sizeof(float) * 2 * n, cudaMemcpyHostToDevice, st));
      const std::vector<Feature*>& qf = est[b]->query_feats;
      if ((int)qf.size() > max_pts) {  // one sequence's share of the query table
        if (!isolate) return fail(XIVO_ERR_STATE, "descriptor matcher: more query features than max_pts");
        fail_sequence(b, XIVO_ERR_STATE, "descriptor matcher: more query features than max_pts");
        nkps.h[b] = 0;  // BRIEF and both nearest-neighbour passes skip it (the callers prune it after this phase)
        continue;
      }
      nq.h[b] = n ? (int)qf.size() : 0;
      for (int j = 0; j < nq.h[b]; ++j) memcpy(qdesc.h + ((size_t)b * max_pts + j) * 32, qf[j]->descriptor, 32);
      if (nq.h[b]) {
        any_q = true;
        XB_CUDA(cudaMemcpyAsync(qdesc.d + (size_t)b * max_pts * 32, qdesc.h + (size_t)b * max_pts * 32, (size_t)32 * nq.h[b], cudaMemcpyHostToDevice, st));
      }
    }
    XB_CUDA(nkps.up(st)); XB_CUDA(nq.up(st));
    if (int rc = launch_brief(st, dPyr.p, 0, sel_off_dev, rows, cols, cn, kpxy.d, nkps.d, max_kp, descK.d, validK.d, B)) return rc;
    g_launches += 1;
    if (any_q) {
      if (int rc = launch_hamming_nearest(st, qdesc.d, nq.d, max_pts, descK.d, nkps.d, max_kp, bestT_idx.d, bestT_dist.d, B)) return rc;
      if (int rc = launch_hamming_nearest(st, descK.d, nkps.d, max_kp, qdesc.d, nq.d, max_pts, bestQ_idx.d, bestQ_dist.d, B)) return rc;
      g_launches += 2;
    }
    for (int b : seqs) {
      const int n = nkps.h[b];
      if (!n) continue;
      XB_CUDA(cudaMemcpyAsync(descK.h + (size_t)b * max_kp * 32, descK.d + (size_t)b * max_kp * 32, (size_t)32 * n, cudaMemcpyDeviceToHost, st));
      if (nq.h[b]) {
        XB_CUDA(cudaMemcpyAsync(bestT_idx.h + (size_t)b * max_pts, bestT_idx.d + (size_t)b * max_pts, sizeof(int) * nq.h[b], cudaMemcpyDeviceToHost, st));
        XB_CUDA(cudaMemcpyAsync(bestT_dist.h + (size_t)b * max_pts, bestT_dist.d + (size_t)b * max_pts, sizeof(int) * nq.h[b], cudaMemcpyDeviceToHost, st));
        XB_CUDA(cudaMemcpyAsync(bestQ_idx.h + (size_t)b * max_kp, bestQ_idx.d + (size_t)b * max_kp, sizeof(int) * n, cudaMemcpyDeviceToHost, st));
      }
    }
    HostScope hw("wait_describe");
    return wait(st);
  }

  // The rest of Tracker::UpdateLK with the decisions on the device: LK -> accept loop (track_accept_kernel) -> FAST for the sequences
  // the accept kernel flagged -> greedy selection (track_select_kernel) -> ONE read-back of [positions | keep flags | picks].  The host
  // then only replays the decisions on its track list (same order, same feature ids as the host path).
  int tracker_decide_on_device(const std::vector<int>& act, const std::vector<int>& lk_list, const std::vector<int>& kind,
                               std::unique_ptr<HostScope>* hs_issue) {
    cudaStream_t st = st1;
    const TrackerCfg& tc = est[0]->tc;
    Estimator& e0 = *est[0];
    if (e0.mask_half < 0) e0.mask_half = tc.mask_size >> 1;
    const int max_new = tc.num_features_max;
    TrackDecideCfg dc{rows, cols, tc.margin, tc.mask_size >> 1, tc.num_features_min, tc.num_features_max, max_pts, max_kp, max_new,
                      (double)tc.max_pixel_displacement};
    if (!lk_list.empty()) {
      HostScope hx("x_i_trk_lk");
      if (int rc = track_lk(lk_list)) return rc;
    }
    {
      HostScope hx("x_i_trk_accept");
      if (int rc = launch_track_accept(st, dc, tkind.d, npts.d, pts0.d, pts1.d, lkst.d, tstat.d, tneed.d, B, kpcount.d)) return rc;
    }
    std::unique_ptr<HostScope> hx_fs(new HostScope("x_i_trk_fast_select"));
    // FAST on the current level-0 image of every tracked sequence (fast_off); the kernel skips those whose need is 0
    if (int rc = launch_fast_detect(st, dPyr.p, 0, fast_off.d, rows, cols, cn, tc.fast_threshold, tc.fast_nonmax, kp.d, max_kp, kpcount.d, B, tneed.d,
                                    tma_fast ? &tm_fast : nullptr, pd.total, true))
      return rc;
    if (int rc = launch_track_select(st, dc, tkind.d, npts.d, pts1.d, tstat.d, tneed.d, kp.d, kpcount.d, tnewkp.d, tnnew.d, B)) return rc;
    g_launches += 3;
    hx_fs.reset(new HostScope("x_i_trk_d2h"));
    Prof::get().d2h += tt_down_bytes;  // [pts1 | keep flags | need | picks] in one copy
    XB_CUDA(cudaMemcpyAsync(tt.h + tt_down_off, tt.d + tt_down_off, tt_down_bytes, cudaMemcpyDeviceToHost, st));
    hx_fs.reset();
    hs_issue->reset();
    { HostScope hw("wait_lk"); if (int rc = wait(st)) return rc; }
    {
      int ndet = 0;
      for (int b : act) ndet += tneed.h[b] > 0;
      Prof::get().add_work("fast_detect", ndet * 2.0 * rows * cols);  // §8d: 2 W H bytes
    }
    HostScope hs("tracker_accept");
    pfor(act, [&](int b, int) {
      HostScope hx("x_trk_replay");
      est[b]->tracker_replay(kind[b], pts1.h + (size_t)b * max_pts * 2, tstat.h + (size_t)b * max_pts, tneed.h[b], tnewkp.h + (size_t)b * max_new,
                             std::min(tnnew.h[b], max_new));
    });
    swap_pyramids(act);
    return 0;
  }

  // Tracker::UpdateLK (tracker.cpp:463-629) for the sequences in `act` whose message holds ring slot slots[i]; the decisions are the
  // estimators' (tracker_host.cpp.inc) or, without descriptors and homography rejection, the device's (tracker_decide_on_device).
  int tracker_update_lk(const std::vector<int>& act_in, const std::vector<int>& slots) {
    cudaStream_t st = st1;
    std::vector<int> act = act_in, lk_list, det_list, kind(B, 0);
    {
      HostScope hs("tracker_prepare");
      if (int rc = begin_frame(act, slots)) return rc;
      std::atomic<int> overflow{0};
      pfor(act, [&](int b, int) {
        HostScope hx("x_trk_prepare");
        Estimator& e = *est[b];
        kind[b] = e.tracker_lk_begin(pts0.h + (size_t)b * max_pts * 2, pts1.h + (size_t)b * max_pts * 2, max_pts);
        if (kind[b] == Estimator::kTrkOverflow) {  // one sequence's track list
          if (isolate) fail_sequence(b, XIVO_ERR_STATE, "tracker feature list exceeds max_pts");
          else overflow = 1;
        }
        if (kind[b] == Estimator::kTrkLK) npts.h[b] = (int)e.tracks.size();
      });
      if (overflow) return fail(XIVO_ERR_STATE, "tracker feature list exceeds max_pts");
      prune(act);
      for (int b : act) {
        if (kind[b] == Estimator::kTrkFirst) det_list.push_back(b);
        else if (kind[b] == Estimator::kTrkLK) lk_list.push_back(b);
        else { off_cur.h[b] = ~0ull; frame_ptr.h[b] = nullptr; }
      }
    }
    std::unique_ptr<HostScope> hs_issue(new HostScope("issue_tracker"));
    if (dev_decide) {
      // every table of the phase is known now: one upload of the blob [inputs | pts1], then the whole chain
      for (int b = 0; b < B; ++b) { tkind.h[b] = 0; fast_off.h[b] = ~0ull; }
      for (int b : act) {
        tkind.h[b] = kind[b];
        if (kind[b] == Estimator::kTrkFirst || kind[b] == Estimator::kTrkLK) fast_off.h[b] = off_cur.h[b];
      }
      HostScope hx("x_i_trk_h2d");
      XB_CUDA(up_blob(tt, tt_up_bytes, st));
    } else {
      XB_CUDA(off_cur.up(st)); XB_CUDA(off_prev.up(st)); XB_CUDA(npts.up(st)); XB_CUDA(frame_ptr.up(st));
      if (tma_pyr) { XB_CUDA(ring_img.up(st)); XB_CUDA(pyr_img.up(st)); }
    }
    std::unique_ptr<HostScope> hx_pyr(new HostScope("x_i_trk_pyr"));
    if (int rc = build_pyramids(true)) return rc;
    hx_pyr.reset();
    {
      int nact = 0;
      for (int b = 0; b < B; ++b) nact += off_cur.h[b] != ~0ull;
      Prof::get().add_work("pyrdown", nact * (7.0 / 3.0) * rows * cols * cn);  // SURVEY.md §8d: (7/3) W H c bytes
    }
    if (dev_decide) return tracker_decide_on_device(act, lk_list, kind, &hs_issue);
    hs_issue.reset();
    if (!lk_list.empty()) {
      XB_CUDA(pts0.up(st)); XB_CUDA(pts1.up(st));
      if (int rc = track_lk(lk_list)) return rc;
      XB_CUDA(pts1.down(st)); XB_CUDA(lkst.down(st));
      if (desc_on) {  // descriptors at the tracked positions (tracker.cpp:530-545), same stream, same wait
        if (int rc = launch_brief(st, dPyr.p, 0, off_cur.d, rows, cols, cn, pts1.d, npts.d, max_pts, descT.d, validT.d, B)) return rc;
        g_launches += 1;
        XB_CUDA(descT.down(st)); XB_CUDA(validT.down(st));
      }
      { HostScope hw("wait_lk"); if (int rc = wait(st)) return rc; }
      HostScope hs("tracker_accept");
      pfor(lk_list, [&](int b, int) {
        HostScope hx("x_trk_accept");
        const size_t r = (size_t)b * max_pts;
        est[b]->tracker_lk_accept(pts0.h + 2 * r, pts1.h + 2 * r, lkst.h + r, desc_on ? descT.h + 32 * r : nullptr, desc_on ? validT.h + r : nullptr);
      });
      prune(lk_list);
      for (int b : lk_list)
        if (est[b]->detect_budget > 0) det_list.push_back(b);
    }
    if (!det_list.empty()) {
      // FAST on the current level-0 image of the sequences that need new features
      for (int b = 0; b < B; ++b) off_prev.h[b] = ~0ull;  // reuse off_prev as the FAST selector
      for (int b : det_list) off_prev.h[b] = off_cur.h[b];
      XB_CUDA(off_prev.up(st));
      if (int rc = detect_and_fetch(det_list, off_prev.d)) return rc;
      Prof::get().add_work("fast_detect", det_list.size() * 2.0 * rows * cols);  // §8d: 2 W H bytes
      if (desc_on) {  // DetectLK with descriptors: every masked keypoint gets one, dropped tracks may claim a keypoint (tracker.cpp:231-327)
        pfor(det_list, [&](int b, int) {
          nkps.h[b] = est[b]->tracker_order_keypoints(kp.h + (size_t)b * max_kp, std::min(kpcount.h[b], max_kp), true, kpxy.h + (size_t)b * max_kp * 2);
        });
        prune(det_list);
        if (int rc = describe_and_match(det_list, off_prev.d)) return rc;
        prune(det_list);
        HostScope hs("tracker_select");
        pfor(det_list, [&](int b, int) {
          std::vector<std::array<int, 3>> m;
          matches_of(b, &m);
          est[b]->tracker_detect_select_desc(descK.h + (size_t)b * max_kp * 32, m);
        });
      } else {
        HostScope hs("tracker_select");
        pfor(det_list, [&](int b, int) {
          HostScope hx("x_trk_select");
          est[b]->tracker_detect_select(kp.h + (size_t)b * max_kp, std::min(kpcount.h[b], max_kp));
        });
      }
    }
    for (int b : lk_list) est[b]->tracker_lk_finish();
    swap_pyramids(act);
    return 0;
  }

  // Tracker::UpdateMatch (tracker.cpp:341-460): detect without a mask, describe, cross-checked nearest-neighbour matching of the existing
  // features' descriptors against the new keypoints (device); the decisions are the estimators' (tracker_host.cpp.inc).
  int tracker_update_match(const std::vector<int>& act_in, const std::vector<int>& slots) {
    cudaStream_t st = st1;
    std::vector<int> act = act_in;
    if (int rc = begin_frame(act, slots)) return rc;
    XB_CUDA(off_cur.up(st)); XB_CUDA(frame_ptr.up(st));
    if (tma_pyr) { XB_CUDA(ring_img.up(st)); XB_CUDA(pyr_img.up(st)); }
    if (int rc = build_pyramids(false)) return rc;
    if (int rc = detect_and_fetch(act, off_cur.d)) return rc;
    std::atomic<int> overflow{0};
    pfor(act, [&](int b, int) {
      Estimator& e = *est[b];
      nkps.h[b] = e.tracker_match_begin(kp.h + (size_t)b * max_kp, std::min(kpcount.h[b], max_kp), kpxy.h + (size_t)b * max_kp * 2);
      if ((int)e.query_feats.size() > max_pts) {  // one sequence's track list
        if (isolate) fail_sequence(b, XIVO_ERR_STATE, "tracker feature list exceeds max_pts");
        else overflow = 1;
      }
    });
    if (overflow) return fail(XIVO_ERR_STATE, "tracker feature list exceeds max_pts");
    prune(act);
    if (int rc = describe_and_match(act, off_cur.d)) return rc;
    prune(act);
    pfor(act, [&](int b, int) {
      std::vector<std::array<int, 3>> m;
      matches_of(b, &m);
      est[b]->tracker_match_finish(descK.h + (size_t)b * max_kp * 32, m);
    });
    swap_pyramids(act);
    return 0;
  }

  // Estimator::OnePointRANSAC (update.cpp:213-393) for the sequences whose gate found high-innovation inliers: back up P (and the
  // Jacobians), temporary update with the low-innovation rows of J() on the covariance with the high-innovation rows zeroed, Jacobians +
  // Mahalanobis distances of the in-state features at the temporarily absorbed motion state, restore.  Sequences that do not need it
  // take part with empty tables.
  int ransac_phases(std::vector<int>& full) {
    cudaStream_t st = st2;
    HostScope hs("ransac_phases");
    std::vector<int> act;
    for (int b : full)
      if (est[b]->ransac.active) act.push_back(b);
    if (!dP0.p && !dP0.alloc((size_t)B * N * N)) return fail(XIVO_ERR_CUDA, "1-point RANSAC: covariance backup allocation failed");
    for (int b : act)  // BackupState
      XB_CUDA(cudaMemcpyAsync(dP0.p + (size_t)b * N * N, dP.p + (size_t)b * N * N, sizeof(double) * N * N, cudaMemcpyDeviceToDevice, st));
    // ---- phase 1: the low-innovation update
    for (int b = 0; b < B; ++b) { nsel.h[b] = 0; nopsU.h[b] = 0; firstU.h[b] = 0; }
    int nops_total = 0;
    for (int b : act) {
      Estimator& e = *est[b];
      firstU.h[b] = nops_total;
      nopsU.h[b] = (int)e.ransac.zero_edits.size();
      if (nops_total + nopsU.h[b] > (int)opsU.n) return fail(XIVO_ERR_STATE, "covariance edit list overflow (1-point RANSAC)");
      for (const EditOp& op : e.ransac.zero_edits) opsU.h[nops_total++] = op;
      int k = 0;
      for (size_t i = 0; i < e.ransac.mh_inliers.size(); ++i) {
        if (!e.ransac.low[i]) continue;
        const auto it = std::find(table_order[b].begin(), table_order[b].end(), e.ransac.mh_inliers[i]);
        sel.h[(size_t)b * lay.F + k++] = (int)(it - table_order[b].begin());
      }
      nsel.h[b] = k;
    }
    XB_CUDA(up_blob(blobU, blobU_fixed + (size_t)nops_total * sizeof(EditOp), st));
    if (int rc = launch_ekf_update(st, lay, dJac.p, sel.d, nsel.d, R.d, dP.p, dErr.p, dHP.p, dKt.p, nullptr, B, 0, opsU.d, firstU.d, nopsU.d, nullptr, 1)) return rc;
    if (int rc = launch_pack_state(st, N, dP.p, dErr.p, pack.d, B)) return rc;
    g_launches += 3;
    XB_CUDA(pack.down(st));
    if (int rc = wait(st)) return rc;
    for (int b : act) {
      Estimator& e = *est[b];
      const double* pk = pack.h + (size_t)b * (2 * N + 529);
      if (nsel.h[b] && !(pk[0] == pk[0])) { e.error = XIVO_ERR_STATE; e.error_msg = "innovation covariance not positive definite (1-point RANSAC)"; continue; }
      e.ransac_after_temp_update(pk);
      double* Xh = X.h + (size_t)b * kPoseDoubles;
      memcpy(Xh, e.X.Rsb.m, 72); memcpy(Xh + 9, e.X.Tsb.v, 24); memcpy(Xh + 12, e.X.Rbc.m, 72); memcpy(Xh + 21, e.X.Tbc.v, 24);
    }
    if (int rc = settle(full)) return rc;
    prune(act);
    // ---- phase 2: Jacobians and r' (J P J' + R)^-1 r at the temporary state (features and groups did not move: their tables are still on the device)
    std::vector<int> nfeat_saved(B);
    for (int b = 0; b < B; ++b) { nfeat_saved[b] = nfeat.h[b]; nfeat.h[b] = 0; nopsJ.h[b] = 0; firstJ.h[b] = 0; }
    for (int b : act) nfeat.h[b] = nfeat_saved[b];
    XB_CUDA(up_blob(blobS, blobS_fixed, st));
    XB_CUDA(up_blob(blobJ, blobJ_fixed, st));
    if (int rc = launch_jacobian_gate(st, lay, cam.d, X.d, groups.d, fx.d, fxp.d, fref.d, fsind.d, nfeat.d, dP.p, R.d, dJac.p, nullptr, mh.d, B, opsJ.d, firstJ.d, nopsJ.d,
                                      nullptr))
      return rc;
    g_launches += 1;
    XB_CUDA(mh.down(st, (size_t)B * lay.F));
    for (int b : act)  // RestoreState (stream order: after the kernel above)
      XB_CUDA(cudaMemcpyAsync(dP.p + (size_t)b * N * N, dP0.p + (size_t)b * N * N, sizeof(double) * N * N, cudaMemcpyDeviceToDevice, st));
    if (int rc = wait(st)) return rc;
    for (int b : act) est[b]->ransac_finish(mh.h + (size_t)b * lay.F, table_order[b]);
    if (int rc = settle(full)) return rc;
    prune(act);
    // ---- phase 3: the survivors' Jacobians at the restored state (update.cpp:381-385), from their CURRENT owner and local state
    for (int b : act) {
      Estimator& e = *est[b];
      for (size_t k = 0; k < e.ransac.jalive.size() && (int)k < lay.F; ++k) {
        if (!e.ransac.jalive[k]) continue;
        const size_t fi = (size_t)b * lay.F + k;
        memcpy(fx.h + 3 * fi, &e.ransac.jx[3 * k], 24);
        fref.h[fi] = e.ransac.jref[k];
        fsind.h[fi] = e.ransac.jsind[k];
      }
      double* Xh = X.h + (size_t)b * kPoseDoubles;
      memcpy(Xh, e.X.Rsb.m, 72); memcpy(Xh + 9, e.X.Tsb.v, 24); memcpy(Xh + 12, e.X.Rbc.m, 72); memcpy(Xh + 21, e.X.Tbc.v, 24);
    }
    XB_CUDA(up_blob(blobS, blobS_fixed, st));
    XB_CUDA(up_blob(blobJ, blobJ_fixed, st));  // (nfeat still selects the active sequences only)
    if (int rc = launch_jacobian_gate(st, lay, cam.d, X.d, groups.d, fx.d, fxp.d, fref.d, fsind.d, nfeat.d, dP.p, R.d, dJac.p, nullptr, mh.d, B, opsJ.d, firstJ.d, nopsJ.d,
                                      nullptr))
      return rc;
    g_launches += 1;
    for (int b = 0; b < B; ++b) nfeat.h[b] = seq_failed(b) ? 0 : nfeat_saved[b];
    return 0;
  }

  // ---- one visual message per active sequence ----------------------------------------------
  int process_visual(const std::vector<int>& act_in, std::vector<Msg>& msgs) {
    cudaStream_t st = st2;  // covariance-side stream; the image tracker uses ctx->stream
    std::vector<int> act, full, lk_act, lk_slots;
    std::vector<char> proceed(act_in.size(), 0);
    {
      HostScope hs("visual_begin");
      std::vector<int> ord(act_in.size());
      for (size_t i = 0; i < ord.size(); ++i) ord[i] = (int)i;
      pfor(ord, [&](int i, int) {
        Estimator& e = *est[act_in[i]];
        Msg& m = msgs[i];
        if (!e.visual_begin(m.ts, m.type) || e.error) return;
        proceed[i] = 1;
      }, [&](int i) { return act_in[i]; });
    }
    // isolating: a sequence that failed here has proceed = 0 already
    if (int rc = isolate ? pool_error() : first_error(act_in)) return rc;
    {
      // predict / point-cloud bookkeeping on the host (the nominal state is already propagated)
      HostScope hs("predict");
      std::vector<int> ord(act_in.size());
      for (size_t i = 0; i < ord.size(); ++i) ord[i] = (int)i;
      pfor(ord, [&](int i, int) {
        if (!proceed[i]) return;
        Estimator& e = *est[act_in[i]];
        Msg& m = msgs[i];
        if (m.type == 1 || m.type == 3) e.predict_features();
        if (m.type == 3)
          for (size_t k = 0; k < m.ids.size(); ++k) e.ids_to_depths.insert({m.ids[k], m.xp_depth[3 * k + 2]});
        if (m.type == 3 || m.type == 4) {
          e.tracker_update_pointcloud(m.ids, m.xp_depth);
          if (m.type == 4 && !e.error) e.tracker_only_finish();
        }
      }, [&](int i) { return act_in[i]; });
    }
    if (isolate) {
      if (int rc = pool_error()) return rc;
      for (size_t i = 0; i < act_in.size(); ++i) proceed[i] = proceed[i] && !est[act_in[i]]->error;
    } else if (int rc = first_error(act_in)) return rc;
    for (size_t i = 0; i < act_in.size(); ++i) {
      if (!proceed[i]) continue;
      const int b = act_in[i];
      act.push_back(b);
      if (msgs[i].type == 1 || msgs[i].type == 2) { lk_act.push_back(b); lk_slots.push_back(msgs[i].img_slot); }
      if (msgs[i].type == 1 || msgs[i].type == 3) full.push_back(b);
    }
    // covariance side of Propagate: enqueued now, overlaps the tracker (nothing below touches P before phase J)
    if (int rc = integrate(full)) return rc;
    if (!lk_act.empty()) {
      if (int rc = est[0]->tc.match_tracker ? tracker_update_match(lk_act, lk_slots) : tracker_update_lk(lk_act, lk_slots)) return rc;
      if (int rc = settle(lk_act)) return rc;
      prune(full);
      for (size_t i = 0; i < act_in.size(); ++i)
        if (proceed[i] && msgs[i].type == 2 && !seq_failed(act_in[i])) est[act_in[i]]->tracker_only_finish();
    }
    if (full.empty()) return 0;

    // ---- ProcessTracks + depth sub-filter (device) ----
    std::vector<int> sub_off(B + 1, 0);
    {
      HostScope hs("process_tracks");
      pfor(full, [&](int b, int) { est[b]->update_step_pre(); });
      if (isolate) {  // one sequence's sub-filter list over its share of the packed table
        for (int b : full)
          if ((int)est[b]->subfilter_list.size() > max_sub) fail_sequence(b, XIVO_ERR_STATE, "sub-filter list exceeds capacity");
        if (int rc = settle(full)) return rc;
        if (full.empty()) return 0;
      }
      int nsub = 0;
      for (int b : full) {
        if ((int)est[b]->subfilter_list.size() > max_sub) return fail(XIVO_ERR_STATE, "sub-filter list exceeds capacity");
        sub_off[b] = nsub;
        nsub += (int)est[b]->subfilter_list.size();
      }
      sub_off[B] = nsub;
      pfor(full, [&](int b, int) {
        HostScope hx("x_sub_stage");
        Estimator& e = *est[b];
        int o = sub_off[b];
        for (size_t i = 0; i < e.subfilter_list.size(); ++i) {
          Feature* f = e.subfilter_list[i];
          prefetch_ahead(e.subfilter_list, i, 4);
          SubfilterIn& s = sub_in.h[o++];
          memcpy(s.x, f->x, sizeof(s.x));
          memcpy(s.P, f->P, sizeof(s.P));
          s.xp[0] = f->xp()[0]; s.xp[1] = f->xp()[1];
          memcpy(s.ref, f->ref->Rsb.m, 72);
          memcpy(s.ref + 9, f->ref->Tsb.v, 24);
          s.outlier_counter = f->outlier_counter;
          s.filter = b;
          s.pad = 0;
        }
        double* Xh = X.h + (size_t)b * kPoseDoubles;
        memcpy(Xh, e.X.Rsb.m, 72); memcpy(Xh + 9, e.X.Tsb.v, 24); memcpy(Xh + 12, e.X.Rbc.m, 72); memcpy(Xh + 21, e.X.Tbc.v, 24);
      });
    }
    const int nsub = sub_off[B];
    {
      HostScope hsi("issue_subfilter");
      XB_CUDA(up_blob(blobS, blobS_fixed + (size_t)nsub * sizeof(SubfilterIn), st));  // [X | sub_in[0 .. nsub)]
      if (nsub) {
        if (int rc = launch_subfilter(st, cam.d, X.d, sub_in.d, sub_out.d, nsub, est[0]->c.sub_Rtri, est[0]->c.sub_mh)) return rc;
        g_launches += 1;
        XB_CUDA(sub_out.down(st, nsub));
      }
    }
    if (nsub) { HostScope hw("wait_subfilter"); if (int rc = wait(st)) return rc; }
    // ---- select/add features, fill the device tables ----
    std::atomic<int> bad_slot{0};
    int nops_total = 0;
    {
      HostScope hs("select_and_tables");
      for (int b = 0; b < B; ++b) nfeat.h[b] = 0;
      pfor(full, [&](int b, int) {
        HostScope hx("x_select_tables");
        Estimator& e = *est[b];
        e.update_step_after_subfilter(sub_out.h + sub_off[b]);
        if (e.error) return;
        const int n = (int)e.instate_features.size();
        nfeat.h[b] = n;
        for (int s2 = 0; s2 < lay.G; ++s2) {  // the groups in the state, by slot
          Group* g = e.gslot[s2];
          if (!g) continue;
          double* gh = groups.h + ((size_t)b * lay.G + g->sind) * kGroupDoubles;
          memcpy(gh, g->Rsb.m, 72);
          memcpy(gh + 9, g->Tsb.v, 24);
        }
        for (int i = 0; i < n; ++i) {
          Feature* f = e.instate_features[i];
          const size_t fi = (size_t)b * lay.F + i;
          memcpy(fx.h + 3 * fi, f->x, 24);
          fxp.h[2 * fi] = f->xp()[0]; fxp.h[2 * fi + 1] = f->xp()[1];
          if (f->ref->sind < 0 || f->sind < 0) {
            if (isolate) fail_sequence(b, XIVO_ERR_STATE, "in-state feature without state slot");
            else bad_slot = 1;
            return;
          }
          fref.h[fi] = f->ref->sind;
          fsind.h[fi] = f->sind;
        }
      });
      if (int rc = settle(full)) return rc;
      if (bad_slot) return fail(XIVO_ERR_STATE, "in-state feature without state slot");
      if (int rc = stage_edits(full, opsJ, firstJ, nopsJ, &nops_total)) return rc;
      prune(full);
      if (isolate && full.empty()) return 0;
    }
    std::unique_ptr<HostScope> hs_issue(new HostScope("issue_jacobian"));
    // one copy: [nfeat | nops | first | fref | fsind | fxp | fx | groups | packed edit list]; the kernel applies the edits, then the features
    XB_CUDA(up_blob(blobJ, blobJ_fixed + (size_t)nops_total * sizeof(EditOp), st));
    if (int rc = launch_jacobian_gate(st, lay, cam.d, X.d, groups.d, fx.d, fxp.d, fref.d, fsind.d, nfeat.d, dP.p, R.d, dJac.p, nullptr, mh.d, B, opsJ.d,
                                      firstJ.d, nopsJ.d, use_1pt ? mh.d + (size_t)B * lay.F : nullptr))
      return rc;
    g_launches += 1;
    {
      double nf = 0;
      for (int b : full) nf += nfeat.h[b];
      Prof::get().add_work("jacobian_gate", nf * 2.0 * N * 8.0);  // §8d: M N 8 bytes of H written
    }
    XB_CUDA(mh.down(st, use_1pt ? 0 : (size_t)B * lay.F));  // [Mahalanobis distances | with the 1-point RANSAC: diag(P) after the edits]
    hs_issue.reset();
    { HostScope hw("wait_jacobian"); if (int rc = wait(st)) return rc; }
    // ---- gating decisions (host), post-gate edits, update (device) ----
    {
      HostScope hs("gating");
      for (int b = 0; b < B; ++b) nsel.h[b] = 0;
      pfor(full, [&](int b, int) {
        Estimator& e = *est[b];
        table_order[b] = e.instate_features;  // index space of mh / the device feature table
        e.update_step_after_gate(mh.h + (size_t)b * lay.F, use_1pt ? mh.h + (size_t)B * lay.F + (size_t)b * N : nullptr);
      });
      if (int rc = settle(full)) return rc;
    }
    if (use_1pt) {  // Estimator::OnePointRANSAC's two device phases for the sequences whose gate asked for them (ransac.active)
      bool any = false;
      for (int b : full) any = any || est[b]->ransac.active;
      if (any) {
        hs_issue.reset();
        if (int rc = ransac_phases(full)) return rc;
      }
    }
    {
      HostScope hs("gating");
      pfor(full, [&](int b, int) {
        Estimator& e = *est[b];
        if (e.error) return;
        const std::vector<Feature*>& order = table_order[b];
        int k = 0;
        for (Feature* f : e.in_update) {
          const auto it = std::find(order.begin(), order.end(), f);
          sel.h[(size_t)b * lay.F + k++] = (int)(it - order.begin());
        }
        nsel.h[b] = k;
      });
      if (int rc = settle(full)) return rc;
      if (int rc = stage_edits(full, opsU, firstU, nopsU, &nops_total)) return rc;
      prune(full);
      if (isolate && full.empty()) return 0;
    }
    hs_issue.reset(new HostScope("issue_update"));
    XB_CUDA(up_blob(blobU, blobU_fixed + (size_t)nops_total * sizeof(EditOp), st));  // [nsel | nops | first | sel | packed post-gate edit list]
    if (int rc = launch_ekf_update(st, lay, dJac.p, sel.d, nsel.d, R.d, dP.p, dErr.p, dHP.p, dKt.p, nullptr, B, cov_tc, opsU.d, firstU.d, nopsU.d, dKt32.p ? &tcops : nullptr)) return rc;
    if (int rc = launch_pack_state(st, N, dP.p, dErr.p, pack.d, B)) return rc;
    g_launches += 3;
    for (int b : full) {
      const double M = 2.0 * nsel.h[b], Nn = N;
      if (M > 0) Prof::get().add_work("ekf_update", 4 * Nn * Nn * Nn + 6 * M * Nn * Nn + 4 * M * M * Nn + M * M * M / 3.0);  // §8d Joseph flop count
    }
    XB_CUDA(pack.down(st));
    hs_issue.reset();
    { HostScope hw("wait_update"); if (int rc = wait(st)) return rc; }
    Prof::get().collect();
    {
      HostScope hs("absorb_and_manage");
      pfor(full, [&](int b, int) {
        Estimator& e = *est[b];
        const double* pk = pack.h + (size_t)b * (2 * N + 529);
        bool notpd = false;
        for (int i = 0; i < N && !notpd; ++i) notpd = nsel.h[b] && !(pk[i] == pk[i]);
        // Innovation covariance not positive definite (the reference's LDLT would return garbage silently): the gain kernel zeroed its
        // gain, so the device covariance is the prior; the frame's bookkeeping is finished without the correction and the sequence
        // carries a sticky error, like the reference's LOG(FATAL) paths.
        e.update_step_after_update(pk, pk + N, pk + N + 529, nsel.h[b] > 0 && !notpd);
        if (notpd && !e.error) { e.error = XIVO_ERR_STATE; e.error_msg = "innovation covariance not positive definite"; }
      });
    }
    return settle(full);
  }

  // Several messages per sequence in one call (same semantics as pushing them one by one): every
  // sequence runs ahead through its IMU messages until its heap releases a visual message; those are
  // then processed together, and the loop continues with the remaining messages.
  // A sequence with no message (xivo_batch_feed) is not touched, nor is a failed sequence of an isolating handle: the rest of its
  // messages are dropped from the moment it fails.
  int ingest_many(std::vector<std::vector<Msg>>& in) {
    WorkPool::get().pin_driver();
    std::vector<int> all(B), fed, vis;
    std::vector<size_t> pos(B, 0);
    std::vector<Msg> popped(B), vmsgs;
    std::vector<char> has(B, 0);
    for (int b = 0; b < B; ++b) {
      all[b] = b;
      if (!in[b].empty() && !seq_failed(b)) fed.push_back(b);
    }
    for (;;) {
      if (isolate) {
        size_t k = 0;
        for (int b : fed) {
          if (est[b]->error) has[b] = 0;
          else fed[k++] = b;
        }
        fed.resize(k);
      }
      {
        HostScope hs("ingest_imu");
        pfor(fed, [&](int b, int) {
          HostScope hx("x_ingest_imu");
          has[b] = 0;
          while (pos[b] < in[b].size()) {
            est[b]->push(std::move(in[b][pos[b]++]));
            Msg m;
            if (!est[b]->pop_ready(&m)) continue;
            if (m.type == 0) {
              est[b]->inertial_internal(m.ts, m.gyro, m.accel);
              if (isolate && est[b]->error) return;
              if (est[b]->needs_state_now()) { has[b] = 2; return; }  // integrate on the device before going on
            } else { popped[b] = std::move(m); has[b] = 1; return; }
          }
        });
      }
      if (isolate) {
        if (int rc = pool_error()) return rc;
        for (int b : fed)
          if (est[b]->error) has[b] = 0;
      } else if (int rc = first_error(all)) return rc;
      vis.clear();
      vmsgs.clear();
      std::vector<int> need_int;
      bool more = false;
      for (int b = 0; b < B; ++b) {
        if (has[b] == 1) { vis.push_back(b); vmsgs.push_back(std::move(popped[b])); }
        if (has[b] == 2) need_int.push_back(b);
      }
      for (int b : fed)
        if (!seq_failed(b)) more = more || pos[b] < in[b].size();
      if (!need_int.empty())
        if (int rc = integrate(need_int)) return rc;
      if (vis.empty()) {
        if (!more) return 0;
        continue;
      }
      if (int rc = process_visual(vis, vmsgs)) return rc;
    }
  }

  // Push one message per sequence, then execute whatever each heap releases (MaintainBuffer).  The message of a failed sequence of an
  // isolating handle is dropped.
  int ingest(std::vector<Msg>& in) {
    WorkPool::get().pin_driver();
    std::vector<int> all = live_sequences(), vis;
    std::vector<Msg> popped(B), vmsgs;
    std::vector<char> has(B, 0);
    {
      HostScope hs("ingest_imu");
      pfor(all, [&](int b, int) {
        est[b]->push(std::move(in[b]));
        Msg m;
        if (!est[b]->pop_ready(&m)) return;
        if (m.type == 0) { est[b]->inertial_internal(m.ts, m.gyro, m.accel); if (est[b]->needs_state_now()) has[b] = 2; }
        else { popped[b] = std::move(m); has[b] = 1; }
      });
    }
    if (isolate) {
      if (int rc = pool_error()) return rc;
      for (int b : all)
        if (est[b]->error) has[b] = 0;
    } else if (int rc = first_error(all)) return rc;
    std::vector<int> need_int;
    for (int b = 0; b < B; ++b) {
      if (has[b] == 1) { vis.push_back(b); vmsgs.push_back(std::move(popped[b])); }
      if (has[b] == 2) need_int.push_back(b);
    }
    if (!need_int.empty())
      if (int rc = integrate(need_int)) return rc;
    if (vis.empty()) return 0;
    return process_visual(vis, vmsgs);
  }

 private:
  // tracker_cfg.normalize (tracker.cpp:343-344, :465-467): cv::normalize NORM_MINMAX of every new frame in its ring slot before its first
  // pyramid pass; norm_part holds the per-CTA partial min / max of launch_normalize_minmax.  Declared after every other member, so that
  // the members the per-frame host phases touch keep the layout they have without the option.
  bool norm_on = false;
  DevBuf<unsigned> norm_part;
};

}  // namespace xb

using namespace xb;
// A batch handle is one lock-step Batch, driven by the thread that calls the C ABI; its per-sequence host code runs on the shared worker
// pool.  Parallelism across sequences beyond one batch comes from several handles per GPU, each driven by its own caller.
struct xivo_batch : Batch {
  using Batch::Batch;
};

#define BATCH_BEGIN                \
  if (!b) {                        \
    set_error("null batch");       \
    return XIVO_ERR_ARG;           \
  }                                \
  Batch& B_ = *b;                  \
  XB_CUDA(cudaSetDevice(B_.ctx->device));
#define SEQ_CHECK                                     \
  if (seq < 0 || seq >= B_.B) {                       \
    set_error("sequence index %d out of range", seq); \
    return XIVO_ERR_ARG;                              \
  }
// the state getters of a failed sequence of an isolating handle refuse with its message
#define SEQ_LIVE                                                                                           \
  if (B_.seq_failed(seq)) {                                                                                \
    set_error("sequence %d has failed (%s); reset it to use it again", seq, B_.est[seq]->error_msg.c_str()); \
    return XIVO_ERR_STATE;                                                                                 \
  }

extern "C" {

int xivo_batch_create(xivo_ctx* ctx, const char* cfg_json, int n_seq, int max_groups, int max_features, int tracker_only,
                      xivo_batch** out) {
  if (!ctx || !cfg_json || !out || n_seq <= 0 || max_groups <= 0 || max_features <= 0) {
    set_error("batch_create: bad arguments");
    return XIVO_ERR_ARG;
  }
  XB_CUDA(cudaSetDevice(ctx->device));
  try {
    Json cfg = Json::parse(cfg_json);
    if (cfg.get("lanes", 0) > 1) {
      set_error("batch_create: \"lanes\" > 1 is not supported; for more parallelism create several batch handles, each driven by its own thread");
      return XIVO_ERR_ARG;
    }
    *out = new xivo_batch(ctx, cfg, n_seq, EkfLayout{max_groups, max_features}, tracker_only != 0);
  } catch (const std::exception& e) {
    set_error("batch_create: %s", e.what());
    return XIVO_ERR_ARG;
  }
  return XIVO_OK;
}

void xivo_batch_destroy(xivo_batch* b) {
  if (!b) return;
  if (b->ctx) cudaSetDevice(b->ctx->device);
  delete b;
}
int xivo_batch_size(const xivo_batch* b) { return b ? b->B : 0; }
int xivo_batch_state_dim(const xivo_batch* b) { return b ? b->N : 0; }
int xivo_batch_lanes(const xivo_batch* b) { return b ? 1 : 0; }

int xivo_batch_inertial_meas(xivo_batch* b, const uint64_t* ts_ns, const double* gyro, const double* accel) {
  BATCH_BEGIN;
  XB_REQUIRE(ts_ns && gyro && accel, "inertial_meas: null argument");
  if (int rc = B_.begin_call("inertial_meas")) return rc;
  const int failed0 = B_.n_failed();
  std::vector<Msg> in(B_.B);
  for (int s = 0; s < B_.B; ++s) {
    in[s].ts = ts_ns[s];
    in[s].type = 0;
    memcpy(in[s].gyro, gyro + 3 * (size_t)s, 24);
    memcpy(in[s].accel, accel + 3 * (size_t)s, 24);
  }
  return B_.end_call(B_.ingest(in), failed0);
}

static int visual_meas_impl(xivo_batch* b, const uint64_t* ts_ns, const uint8_t* const* imgs, int rows, int cols, int channels,
                            int tracker_only, bool on_device) {
  BATCH_BEGIN;
  XB_REQUIRE(ts_ns && imgs && rows > 0 && cols > 0, "visual_meas: bad arguments");
  for (int s = 0; s < B_.B; ++s) XB_REQUIRE(imgs[s], "visual_meas: null image");
  if (int rc = B_.begin_call("visual_meas")) return rc;
  if (int rc = B_.ensure_images(rows, cols, channels)) return rc;
  const int failed0 = B_.n_failed();
  const size_t ib = (size_t)rows * cols * channels;
  std::vector<Msg> in(B_.B);
  std::vector<int> slot_of(B_.B);
  bool uploaded = false;
  const std::vector<int> all = B_.live_sequences();
  B_.take_slots(imgs, on_device, all, slot_of, &uploaded);
  for (int s = 0; s < B_.B; ++s) {
    in[s].ts = ts_ns[s];
    in[s].type = tracker_only ? 2 : 1;
    in[s].img_slot = slot_of[s];
  }
  if (!uploaded)
    if (int rc = B_.upload_frames(imgs, all, slot_of, on_device, ib)) return B_.end_call(rc, failed0);
  const int rc = B_.ingest(in);
  const int rc2 = B_.ingest_done(all, slot_of);
  return B_.end_call(rc ? rc : rc2, failed0);
}

int xivo_batch_visual_meas(xivo_batch* b, const uint64_t* ts_ns, const uint8_t* const* imgs, int rows, int cols, int channels,
                           int tracker_only) {
  return visual_meas_impl(b, ts_ns, imgs, rows, cols, channels, tracker_only, false);
}
int xivo_batch_visual_meas_device(xivo_batch* b, const uint64_t* ts_ns, const uint8_t* const* imgs_dev, int rows, int cols,
                                  int channels, int tracker_only) {
  return visual_meas_impl(b, ts_ns, imgs_dev, rows, cols, channels, tracker_only, true);
}
int xivo_batch_visual_meas_png(xivo_batch* b, const uint64_t* ts_ns, const uint8_t* const* png, const size_t* png_bytes, int channels,
                               int tracker_only) {
  BATCH_BEGIN;
  XB_REQUIRE(ts_ns && png && png_bytes, "visual_meas_png: bad arguments");
  for (int s = 0; s < B_.B; ++s) XB_REQUIRE(png[s], "visual_meas_png: null data");
  if (channels != 1 && channels != 3) return B_.fail(XIVO_ERR_ARG, "visual_meas_png: channels must be 1 or 3, got " + std::to_string(channels));
  if (int rc = B_.begin_call("visual_meas_png")) return rc;
  HostScope ht("visual_meas_png_total");
  const int failed0 = B_.n_failed();
  std::vector<int> slot_of(B_.B);
  if (int rc = B_.decode_png_frames(B_.live_sequences(), png, png_bytes, channels, slot_of)) return rc;
  std::vector<Msg> in(B_.B);
  for (int s = 0; s < B_.B; ++s) {
    in[s].ts = ts_ns[s];
    in[s].type = tracker_only ? 2 : 1;
    in[s].img_slot = slot_of[s];
  }
  return B_.end_call(B_.ingest(in), failed0);
}
int xivo_batch_step(xivo_batch* b, int n_imu, const uint64_t* imu_ts, const double* gyro, const double* accel, const uint64_t* frame_ts,
                    const uint8_t* const* imgs, int rows, int cols, int channels, int on_device) {
  BATCH_BEGIN;
  XB_REQUIRE(n_imu >= 0 && frame_ts && imgs && (n_imu == 0 || (imu_ts && gyro && accel)), "batch_step: bad arguments");
  const int nb = B_.B;  // the IMU arrays are (n_imu, nb[, 3])
  for (int s = 0; s < nb; ++s) XB_REQUIRE(imgs[s], "batch_step: null image");
  if (int rc = B_.begin_call("batch_step")) return rc;
  HostScope hst("ingest_many_total");
  if (int rc = B_.ensure_images(rows, cols, channels)) return rc;
  const int failed0 = B_.n_failed();
  const size_t ib = (size_t)rows * cols * channels;
  std::vector<std::vector<Msg>> in(nb);
  std::vector<int> slot_of(nb);
  bool uploaded = false;
  const std::vector<int> all = B_.live_sequences();
  B_.take_slots(imgs, on_device != 0, all, slot_of, &uploaded);
  {
    HostScope hm("marshal");
    for (int s = 0; s < nb; ++s) {
      in[s].resize(n_imu + 1);
      for (int k = 0; k < n_imu; ++k) {
        Msg& m = in[s][k];
        const size_t o = (size_t)k * nb + s;
        m.ts = imu_ts[o];
        m.type = 0;
        memcpy(m.gyro, gyro + o * 3, 24);
        memcpy(m.accel, accel + o * 3, 24);
      }
      Msg& v = in[s][n_imu];
      v.ts = frame_ts[s];
      v.type = 1;
      v.img_slot = slot_of[s];
    }
  }
  if (!uploaded)
    if (int rc = B_.upload_frames(imgs, all, slot_of, on_device != 0, ib)) return B_.end_call(rc, failed0);
  const int rc = B_.ingest_many(in);
  const int rc2 = B_.ingest_done(all, slot_of);
  return B_.end_call(rc ? rc : rc2, failed0);
}

// xivo_batch_feed[_png]: what is refused is refused here, before a ring slot is taken or a message pushed.
static int feed_check(Batch& B_, const char* what, const int* n_imu, const uint64_t* imu_ts, const double* gyro, const double* accel,
                      const uint64_t* frame_ts, bool any_frame) {
  if (int rc = B_.refuse_if_failed(what)) return rc;
  if (!n_imu) return B_.fail(XIVO_ERR_ARG, std::string(what) + ": null n_imu");
  for (int s = 0; s < B_.B; ++s) {
    if (n_imu[s] < 0) return B_.fail(XIVO_ERR_ARG, std::string(what) + ": sequence " + std::to_string(s) + ": negative n_imu (" + std::to_string(n_imu[s]) + ")");
    if (n_imu[s] > 0 && !(imu_ts && gyro && accel))
      return B_.fail(XIVO_ERR_ARG, std::string(what) + ": sequence " + std::to_string(s) + " has " + std::to_string(n_imu[s]) + " IMU samples but the IMU arrays are null");
  }
  if (any_frame && !frame_ts) return B_.fail(XIVO_ERR_ARG, std::string(what) + ": null frame_ts");
  return 0;
}
// Sequence s: its n_imu[s] IMU rows (from offset sum(n_imu[0..s-1])), then its frame in ring slot slot_of[s] if it has one.
static void feed_messages(const Batch& B_, const int* n_imu, const uint64_t* imu_ts, const double* gyro, const double* accel, const uint64_t* frame_ts,
                          const std::vector<int>& present, const std::vector<int>& slot_of, int tracker_only, std::vector<std::vector<Msg>>& in) {
  HostScope hm("marshal");
  std::vector<char> has_frame(B_.B, 0);
  for (int s : present) has_frame[s] = 1;
  size_t o = 0;
  for (int s = 0; s < B_.B; ++s) {
    in[s].resize((size_t)n_imu[s] + has_frame[s]);
    for (int k = 0; k < n_imu[s]; ++k, ++o) {
      Msg& m = in[s][k];
      m.ts = imu_ts[o];
      m.type = 0;
      memcpy(m.gyro, gyro + o * 3, 24);
      memcpy(m.accel, accel + o * 3, 24);
    }
    if (has_frame[s]) {
      Msg& v = in[s][n_imu[s]];
      v.ts = frame_ts[s];
      v.type = tracker_only ? 2 : 1;
      v.img_slot = slot_of[s];
    }
  }
}

int xivo_batch_feed(xivo_batch* b, const int* n_imu, const uint64_t* imu_ts, const double* gyro, const double* accel, const uint64_t* frame_ts,
                    const uint8_t* const* imgs, int rows, int cols, int channels, int on_device, int tracker_only) {
  BATCH_BEGIN;
  HostScope hst("feed_total");
  std::vector<int> present;  // the sequences that get a frame (a failed sequence of an isolating handle gets none)
  if (imgs)
    for (int s = 0; s < B_.B; ++s)
      if (imgs[s] && !B_.seq_failed(s)) present.push_back(s);
  if (int rc = feed_check(B_, "feed", n_imu, imu_ts, gyro, accel, frame_ts, !present.empty())) return rc;
  const int failed0 = B_.n_failed();
  std::vector<int> slot_of(B_.B, -1);
  const size_t ib = (size_t)rows * cols * channels;
  if (!present.empty()) {
    const std::string first = std::to_string(present[0]);
    if (rows <= 0 || cols <= 0) return B_.fail(XIVO_ERR_ARG, "feed: sequence " + first + ": bad frame geometry");
    if (B_.img_ready && (rows != B_.rows || cols != B_.cols || channels != B_.cn))
      return B_.fail(XIVO_ERR_ARG, "feed: sequence " + first + ": frame is " + std::to_string(rows) + " x " + std::to_string(cols) + " x " + std::to_string(channels) +
                                       ", the handle's frames are " + std::to_string(B_.rows) + " x " + std::to_string(B_.cols) + " x " + std::to_string(B_.cn));
    if (int rc = B_.ensure_images(rows, cols, channels)) return rc;
    B_.drop_prefetches();
    B_.fresh_slots(present, slot_of);
    if (int rc = B_.upload_frames(imgs, present, slot_of, on_device != 0, ib)) return B_.end_call(rc, failed0);
  }
  std::vector<std::vector<Msg>> in(B_.B);
  feed_messages(B_, n_imu, imu_ts, gyro, accel, frame_ts, present, slot_of, tracker_only, in);
  const int rc = B_.ingest_many(in);
  const int rc2 = present.empty() ? 0 : B_.ingest_done(present, slot_of);
  return B_.end_call(rc ? rc : rc2, failed0);
}

int xivo_batch_feed_png(xivo_batch* b, const int* n_imu, const uint64_t* imu_ts, const double* gyro, const double* accel, const uint64_t* frame_ts,
                        const uint8_t* const* png, const size_t* png_bytes, int channels, int tracker_only) {
  BATCH_BEGIN;
  HostScope hst("feed_png_total");
  std::vector<int> present;
  if (png)
    for (int s = 0; s < B_.B; ++s)
      if (png[s] && !B_.seq_failed(s)) present.push_back(s);
  if (int rc = feed_check(B_, "feed_png", n_imu, imu_ts, gyro, accel, frame_ts, !present.empty())) return rc;
  const int failed0 = B_.n_failed();
  std::vector<int> slot_of(B_.B, -1);
  if (!present.empty()) {
    if (!png_bytes) return B_.fail(XIVO_ERR_ARG, "feed_png: null png_bytes");
    if (channels != 1 && channels != 3) return B_.fail(XIVO_ERR_ARG, "feed_png: channels must be 1 or 3, got " + std::to_string(channels));
    if (int rc = B_.decode_png_frames(present, png, png_bytes, channels, slot_of)) return rc;
  }
  std::vector<std::vector<Msg>> in(B_.B);
  feed_messages(B_, n_imu, imu_ts, gyro, accel, frame_ts, present, slot_of, tracker_only, in);
  return B_.end_call(B_.ingest_many(in), failed0);
}

int xivo_batch_prefetch_frames(xivo_batch* b, const uint8_t* const* imgs, int rows, int cols, int channels) {
  BATCH_BEGIN;
  XB_REQUIRE(imgs && rows > 0 && cols > 0, "prefetch_frames: bad arguments");
  for (int s = 0; s < B_.B; ++s) XB_REQUIRE(imgs[s], "prefetch_frames: null image");
  if (int rc = B_.ensure_images(rows, cols, channels)) return rc;
  return B_.prefetch_frames(imgs, (size_t)rows * cols * channels);
}

int xivo_set_frame_ingest(int mode) {
  if (mode != XIVO_INGEST_ZERO_COPY && mode != XIVO_INGEST_COPY_ENGINE) return g_frame_ingest.load();
  return g_frame_ingest.exchange(mode);
}

void xivo_profile_enable(int on) {  // 0 off, 1 kernels + batch-level host phases, 2 + per-sequence host scopes, 3 host scopes only (no kernel events)
  Prof::get().enabled = on != 0;
  Prof::get().fine = on >= 2;
  Prof::get().kernels = on != 3;
}
void xivo_profile_reset(void) { Prof::get().reset(); }
int xivo_profile_report(char* buf, int n) {
  const std::string s = Prof::get().json();
  if ((int)s.size() + 1 > n) return XIVO_ERR_ARG;
  memcpy(buf, s.c_str(), s.size() + 1);
  return 0;
}

int xivo_batch_visual_meas_pointcloud(xivo_batch* b, const uint64_t* ts_ns, const int* n_pts, const int* const* ids,
                                      const double* const* xp_depth, int tracker_only) {
  BATCH_BEGIN;
  XB_REQUIRE(ts_ns && n_pts && ids && xp_depth, "visual_meas_pointcloud: null argument");
  if (int rc = B_.begin_call("visual_meas_pointcloud")) return rc;
  const int failed0 = B_.n_failed();
  std::vector<Msg> in(B_.B);
  for (int s = 0; s < B_.B; ++s) {
    if (B_.seq_failed(s)) continue;
    in[s].ts = ts_ns[s];
    in[s].type = tracker_only ? 4 : 3;
    in[s].ids.assign(ids[s], ids[s] + n_pts[s]);
    in[s].xp_depth.assign(xp_depth[s], xp_depth[s] + 3 * (size_t)n_pts[s]);
  }
  return B_.end_call(B_.ingest(in), failed0);
}

static void put34(const SE3h& g, double* out) {
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) out[4 * i + j] = g.R.m[3 * i + j];
    out[4 * i + 3] = g.T.v[i];
  }
}
int xivo_get_gsb(xivo_batch* b, int seq, double* out) {
  BATCH_BEGIN; SEQ_CHECK; SEQ_LIVE;
  put34(B_.est[seq]->gsb(), out);
  return 0;
}
int xivo_get_gbc(xivo_batch* b, int seq, double* out) { BATCH_BEGIN; SEQ_CHECK; SEQ_LIVE; put34(B_.est[seq]->gbc(), out); return 0; }
int xivo_get_gsc(xivo_batch* b, int seq, double* out) {
  BATCH_BEGIN; SEQ_CHECK; SEQ_LIVE;
  put34(se3_mul(B_.est[seq]->gsb(), B_.est[seq]->gbc()), out);
  return 0;
}
int xivo_get_motion(xivo_batch* b, int seq, double* Vsb, double* bg, double* ba, double* Rsg) {
  BATCH_BEGIN; SEQ_CHECK; SEQ_LIVE;
  const MotionX& X = B_.est[seq]->X;
  if (Vsb) memcpy(Vsb, X.Vsb.v, 24);
  if (bg) memcpy(bg, X.bg.v, 24);
  if (ba) memcpy(ba, X.ba.v, 24);
  if (Rsg) memcpy(Rsg, X.Rsg.m, 72);
  return 0;
}
int xivo_get_P(xivo_batch* b, int seq, double* out) {
  BATCH_BEGIN; SEQ_CHECK; SEQ_LIVE;
  XB_REQUIRE(out, "get_P: null output");
  if (int rc = B_.flush({seq})) return rc;
  SEQ_LIVE;  // its share of the edit list may have overflowed
  XB_CUDA(cudaMemcpy(out, B_.dP.p + (size_t)seq * B_.N * B_.N, sizeof(double) * B_.N * B_.N, cudaMemcpyDeviceToHost));
  return 0;
}
int xivo_get_Pstate(xivo_batch* b, int seq, double* out81) {
  BATCH_BEGIN; SEQ_CHECK; SEQ_LIVE;
  if (int rc = B_.flush({seq})) return rc;
  SEQ_LIVE;  // its share of the edit list may have overflowed
  for (int i = 0; i < 9; ++i)
    XB_CUDA(cudaMemcpy(out81 + 9 * i, B_.dP.p + (size_t)seq * B_.N * B_.N + (size_t)i * B_.N, sizeof(double) * 9, cudaMemcpyDeviceToHost));
  return 0;
}
int xivo_get_counters(xivo_batch* b, int seq, int* out) {
  BATCH_BEGIN; SEQ_CHECK; SEQ_LIVE;
  Estimator& e = *B_.est[seq];
  int ng = 0;
  for (auto& kv : e.graph.groups) ng += kv.second->instate();
  out[0] = (int)e.instate_features.size();
  out[1] = ng;
  out[2] = e.gauge_group;
  out[3] = e.num_mh_rejected;
  out[4] = e.num_failed_to_track;
  out[5] = e.num_new_detections;
  out[6] = e.vision_counter;
  out[7] = e.imu_counter;
  out[8] = e.meas_update_initialized;
  out[9] = e.vision_initialized;
  out[10] = (int)e.tracks.size();
  out[11] = e.error;
  return 0;
}
int xivo_get_time_ns(xivo_batch* b, int seq, uint64_t* ts) { BATCH_BEGIN; SEQ_CHECK; SEQ_LIVE; *ts = B_.est[seq]->curr_time; return 0; }
int xivo_get_tracked_features(xivo_batch* b, int seq, int* ids, double* xy, int* status, int max_n, int* n) {
  BATCH_BEGIN; SEQ_CHECK; SEQ_LIVE;
  int k = 0;
  for (Feature* f : B_.est[seq]->tracks) {
    if (k < max_n) {
      if (ids) ids[k] = f->id;
      if (xy) { xy[2 * k] = f->xp()[0]; xy[2 * k + 1] = f->xp()[1]; }
      if (status) status[k] = (int)f->tstatus;
    }
    ++k;
  }
  *n = k;
  return 0;
}
int xivo_get_tracked_descriptors(xivo_batch* b, int seq, uint8_t* desc, uint8_t* has, int max_n, int* n) {
  BATCH_BEGIN; SEQ_CHECK; SEQ_LIVE;
  XB_REQUIRE(n, "get_tracked_descriptors: null count");
  int k = 0;
  for (Feature* f : B_.est[seq]->tracks) {
    if (k < max_n) {
      if (desc) memcpy(desc + 32 * (size_t)k, f->descriptor, 32);
      if (has) has[k] = f->has_descriptor ? 1 : 0;
    }
    ++k;
  }
  *n = k;
  return 0;
}
int xivo_get_instate_features(xivo_batch* b, int seq, int* ids, int* sinds, int* refs, double* Xs3, double* x3, int max_n, int* n) {
  BATCH_BEGIN; SEQ_CHECK; SEQ_LIVE;
  Estimator& e = *B_.est[seq];
  int k = 0;
  for (Feature* f : e.instate_features) {
    if (k < max_n) {
      if (ids) ids[k] = f->id;
      if (sinds) sinds[k] = f->sind;
      if (refs) refs[k] = f->ref ? f->ref->id : -1;
      if (x3) memcpy(x3 + 3 * k, f->x, 24);
      if (Xs3 && f->ref) {
        const SE3h gsc = se3_mul(f->ref->gsb(), e.gbc());
        const double z = std::exp(f->x[2]);
        const V3 Xs = se3_apply(gsc, V3{{f->x[0] * z, f->x[1] * z, z}});
        memcpy(Xs3 + 3 * k, Xs.v, 24);
      }
    }
    ++k;
  }
  *n = k;
  return 0;
}
int xivo_get_instate_groups(xivo_batch* b, int seq, int* ids, int* sinds, double* gsb12, int max_n, int* n) {
  BATCH_BEGIN; SEQ_CHECK; SEQ_LIVE;
  int k = 0;
  for (auto& kv : B_.est[seq]->graph.groups) {
    Group* g = kv.second;
    if (!g->instate()) continue;
    if (k < max_n) {
      if (ids) ids[k] = g->id;
      if (sinds) sinds[k] = g->sind;
      if (gsb12) put34(g->gsb(), gsb12 + 12 * k);
    }
    ++k;
  }
  *n = k;
  return 0;
}
// ---- the rest of the reference's read-back surface (estimator.h:153-231, estimator_accessors.cpp) -------------------------
static int fetch_P(Batch& B_, int seq, std::vector<double>* P) {
  P->resize((size_t)B_.N * B_.N);
  if (int rc = B_.flush({seq})) return rc;
  SEQ_LIVE;  // its share of the edit list may have overflowed
  XB_CUDA(cudaMemcpy(P->data(), B_.dP.p + (size_t)seq * B_.N * B_.N, sizeof(double) * B_.N * B_.N, cudaMemcpyDeviceToHost));
  return 0;
}
int xivo_get_instate_feature_table(xivo_batch* b, int seq, int n_output, int* ids, int* sinds, int* ref_group_ids, double* Xs3, double* Xc3,
                                   double* xc3, double* pred2, double* meas2, double* cov6, int max_n, int* n) {
  BATCH_BEGIN; SEQ_CHECK; SEQ_LIVE;
  XB_REQUIRE(n, "get_instate_feature_table: null count");
  std::vector<double> P;
  if (int rc = fetch_P(B_, seq, &P)) return rc;
  const std::vector<FeatureRow> rows = B_.est[seq]->instate_feature_rows(P.data(), n_output);
  for (size_t i = 0; i < rows.size() && (int)i < max_n; ++i) {
    const FeatureRow& r = rows[i];
    if (ids) ids[i] = r.id;
    if (sinds) sinds[i] = r.sind;
    if (ref_group_ids) ref_group_ids[i] = r.ref_group_id;
    if (Xs3) memcpy(Xs3 + 3 * i, r.Xs, 24);
    if (Xc3) memcpy(Xc3 + 3 * i, r.Xc, 24);
    if (xc3) memcpy(xc3 + 3 * i, r.xc, 24);
    if (pred2) memcpy(pred2 + 2 * i, r.pred, 16);
    if (meas2) memcpy(meas2 + 2 * i, r.meas, 16);
    if (cov6) memcpy(cov6 + 6 * i, r.cov, 48);
  }
  *n = (int)rows.size();
  return 0;
}
int xivo_get_instate_group_table(xivo_batch* b, int seq, int* ids, int* sinds, double* pose7, double* cov36, int max_n, int* n) {
  BATCH_BEGIN; SEQ_CHECK; SEQ_LIVE;
  XB_REQUIRE(n, "get_instate_group_table: null count");
  std::vector<double> P;
  if (int rc = fetch_P(B_, seq, &P)) return rc;
  const std::vector<GroupRow> rows = B_.est[seq]->instate_group_rows(P.data());
  for (size_t i = 0; i < rows.size() && (int)i < max_n; ++i) {
    if (ids) ids[i] = rows[i].id;
    if (sinds) sinds[i] = rows[i].sind;
    if (pose7) memcpy(pose7 + 7 * i, rows[i].pose, 56);
    if (cov36) memcpy(cov36 + 36 * i, rows[i].cov, 288);
  }
  *n = (int)rows.size();
  return 0;
}
int xivo_get_calibration(xivo_batch* b, int seq, double* Ca9, double* Cg9, double* td, double* intrinsics9, int* distortion_type) {
  BATCH_BEGIN; SEQ_CHECK; SEQ_LIVE;
  const Estimator& e = *B_.est[seq];
  if (Ca9) memcpy(Ca9, e.c.Ca.m, 72);
  if (Cg9) memcpy(Cg9, e.c.Cg.m, 72);
  if (td) *td = e.X.td;
  if (intrinsics9) {  // BaseCamera::GetIntrinsics (camera_base.h:65-69), EquidistantCamera::GetIntrinsics (camera_equidist.h:169-173)
    const CameraParams& k = e.cam;
    const double v[9] = {k.fx, k.fy, k.cx, k.cy, k.model == 3 ? k.k0 : 0, k.model == 3 ? k.k1 : 0, k.model == 3 ? k.k2 : 0, k.model == 3 ? k.k3 : 0, 0};
    memcpy(intrinsics9, v, sizeof(v));
  }
  if (distortion_type) *distortion_type = e.cam.model;  // DistortionType (camera_base.h:12-17): PINHOLE 0, EQUI 3
  return 0;
}
int xivo_get_just_dropped(xivo_batch* b, int seq, int* ids, int max_n, int* n) {
  BATCH_BEGIN; SEQ_CHECK; SEQ_LIVE;
  XB_REQUIRE(n, "get_just_dropped: null count");
  const std::vector<int>& v = B_.est[seq]->just_dropped_ids;
  for (size_t i = 0; i < v.size() && (int)i < max_n; ++i)
    if (ids) ids[i] = v[i];
  *n = (int)v.size();
  return 0;
}
int xivo_get_tracker_counters(xivo_batch* b, int seq, int out[4]) {
  BATCH_BEGIN; SEQ_CHECK; SEQ_LIVE;
  const Estimator& e = *B_.est[seq];
  out[0] = e.num_outliers_rejected;  // Tracker::num_rejected_outliers()
  out[1] = e.num_failed_to_track;
  out[2] = e.num_new_detections;
  out[3] = e.num_oneptransac_rejected;
  return 0;
}
int xivo_scale_init_velocity(xivo_batch* b, int seq, double scale) {  // Estimator::ScaleInitVelocity: X_.Vsb /= scale
  BATCH_BEGIN; SEQ_CHECK; SEQ_LIVE;
  Estimator& e = *B_.est[seq];
  for (int k = 0; k < 3; ++k) e.X.Vsb.v[k] /= scale;
  return 0;
}

int xivo_init_with_sim_depths(xivo_batch* b) {
  BATCH_BEGIN;
  for (auto& e : B_.est) e->sim_initialize_depths = true;
  B_.sim_depths = true;
  return 0;
}
int xivo_batch_reset_sequence(xivo_batch* b, int seq, const char* cfg_json) {
  BATCH_BEGIN; SEQ_CHECK;
  if (!cfg_json) return B_.reset_sequence(seq, nullptr);
  Json cfg;
  try {
    cfg = Json::parse(cfg_json);
  } catch (const std::exception& e) {
    set_error("reset_sequence: config does not parse: %s", e.what());
    return XIVO_ERR_ARG;
  }
  return B_.reset_sequence(seq, &cfg);
}
int xivo_batch_isolate_failures(xivo_batch* b, int on) {
  if (!b) {
    set_error("null batch");
    return XIVO_ERR_ARG;
  }
  return b->set_isolation(on != 0);
}
int xivo_batch_sequence_status(const xivo_batch* b, int seq, int* code, char* msg, int msg_cap) {
  if (!b || !code) {
    set_error("sequence_status: null argument");
    return XIVO_ERR_ARG;
  }
  if (seq < 0 || seq >= b->B) {
    set_error("sequence index %d out of range", seq);
    return XIVO_ERR_ARG;
  }
  const Estimator& e = *b->est[seq];
  *code = e.error;
  if (msg && msg_cap > 0) {
    const size_t n = std::min(e.error ? e.error_msg.size() : 0, (size_t)msg_cap - 1);
    memcpy(msg, e.error_msg.data(), n);
    msg[n] = 0;
  }
  return XIVO_OK;
}
const char* xivo_batch_error(xivo_batch* b, int seq) {
  if (!b || seq < 0 || seq >= b->B) return "";
  return b->est[seq]->error_msg.c_str();
}

}  // extern "C"
