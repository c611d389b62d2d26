// nvb_api.cu -- the C-ABI (include/nvblox_b200.h) and the host-side orchestration.
//
// Host responsibilities are reduced to what the reference also does on the host
// for this path and cannot be avoided: the view AABB from the camera pose
// (Camera::getViewAABB, nvblox/src/sensors/camera.cpp:31-83; ViewCalculator setup,
// view_calculator_impl.cuh:137-156), T_C_L = T_L_C^-1
// (projective_integrator_impl.cuh:268), and capacity bookkeeping. Block lists,
// allocation, the update tracker and the ESDF wavefront stay on the device.
#include <algorithm>
#include <array>
#include <cfloat>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <functional>
#include <set>
#include <string>
#include <vector>

#include "nvb_esdf_block.cuh"

using namespace nvb;

namespace {

thread_local std::string g_last_error;

int fail(int code, const std::string& msg) {
  g_last_error = msg;
  return code;
}

#define NVB_CUDA(expr)                                                                               \
  do {                                                                                               \
    cudaError_t e_ = (expr);                                                                         \
    if (e_ != cudaSuccess)                                                                           \
      return fail(NVB_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(e_));                 \
  } while (0)

constexpr int kDefaultCapacity = 1 << 18;
constexpr int kStagingBuffers = 3;
constexpr int kCountRing = 8;
constexpr int kNumStages = 6;

struct StageEvent {
  cudaEvent_t start, stop;
  int stage;
};

constexpr int kNoFill = -1;
constexpr bool kKeepContents = true;

// One device allocation of size() elements, freed by the destructor. The mapper's buffers and the temporaries of a single
// call both use it, so that no return path leaks and no failed allocation leaves a pointer to freed memory behind.
template <typename T>
class DeviceArray {
 public:
  DeviceArray() = default;
  DeviceArray(const DeviceArray&) = delete;
  DeviceArray& operator=(const DeviceArray&) = delete;
  DeviceArray(DeviceArray&& o) noexcept : p_(o.p_), n_(o.n_) {
    o.p_ = nullptr;
    o.n_ = 0;
  }
  DeviceArray& operator=(DeviceArray&& o) noexcept {
    std::swap(p_, o.p_);
    std::swap(n_, o.n_);
    return *this;
  }
  ~DeviceArray() { cudaFree(p_); }

  T* get() const { return p_; }
  size_t size() const { return n_; }

  // Makes room for `need` elements by allocating `count` of them (at least `need`); nothing happens when need <= size().
  // The new allocation is filled with the byte `fill` unless that is kNoFill, and `keep` copies the old elements to its
  // front. An existing allocation is replaced only once both of the mapper's streams are idle, and freed once the fill
  // and the copy are done; the new pointer is published last, so after a failure the array still owns the old one.
  cudaError_t grow(NvbMapper* m, size_t need, size_t count, int fill = kNoFill, bool keep = false);
  // Doubling growth: room for `need` elements in an allocation of max(need, 2 x size()), unfilled, keeping nothing.
  cudaError_t growDoubling(NvbMapper* m, size_t need) { return grow(m, need, 2 * n_); }

 private:
  T* p_ = nullptr;
  size_t n_ = 0;
};

// One layer's slab, owned: the blocks, the block-index array, the free-slot stack, its two counters and the hash. Kernels
// get them as the DevLayer that dev() returns, which is rebuilt whenever the arrays change. The layer exists once create()
// has allocated and initialised all of them. No operation counts launches in m->launches: that stays with each caller.
class LayerSlab {
 public:
  bool exists() const { return d_.blocks != nullptr; }
  int capacity() const { return d_.capacity; }
  const DevLayer& dev() const { return d_; }

  // `capacity` zeroed slots, none handed out, and an empty hash. Replaces the layer only once every array is allocated.
  cudaError_t create(NvbMapper* m, int capacity, int block_bytes);
  // Doubling growth of the slab (BlockMemoryPool expansion, map/internal/impl/block_memory_pool_impl.h:54-73) to
  // `capacity` slots; nothing happens when it has that many. Synchronising and rare. The used slots, the free stack and
  // the counters are copied and the hash is rebuilt. The new arrays replace the old ones last, so after a failure the
  // layer is as it was.
  cudaError_t grow(NvbMapper* m, int capacity);

  // The high-water mark (slots handed out so far; above the capacity after a slab overflow), read on `st` and waited for.
  // On the legacy default stream this is a blocking copy. 0 for a layer that does not exist.
  cudaError_t highWaterMark(int* n, cudaStream_t st = nullptr) const {
    *n = 0;
    if (!exists()) return cudaSuccess;
    const cudaError_t e = cudaMemcpyAsync(n, d_.count, sizeof(int), cudaMemcpyDeviceToHost, st);
    return e == cudaSuccess ? cudaStreamSynchronize(st) : e;
  }
  // The fill level: the high-water mark clamped to the capacity.
  cudaError_t fillLevel(int* n, cudaStream_t st = nullptr) const {
    const cudaError_t e = highWaterMark(n, st);
    *n = std::min(*n, d_.capacity);
    return e;
  }

  // No blocks: the slots below the fill level (a blocking read) are zeroed, since free slots are zero, both counters are
  // reset and the hash is emptied.
  cudaError_t empty(cudaStream_t st) {
    int n = 0;
    cudaError_t e = fillLevel(&n);
    if (e == cudaSuccess) e = cudaMemsetAsync(blocks_.get(), 0, (size_t)n * d_.block_bytes, st);
    if (e == cudaSuccess) e = cudaMemsetAsync(count_.get(), 0, sizeof(int), st);
    if (e == cudaSuccess) e = cudaMemsetAsync(free_count_.get(), 0, sizeof(int), st);
    if (e == cudaSuccess) rehash(0, st);
    return e;
  }
  // Empties the hash and reinserts the live slots of [0, n).
  void rehash(int n, cudaStream_t st) {
    launchFillU64(d_.hash.keys, kEmptyKey, (size_t)d_.hash.mask + 1, st);
    launchRehash(d_, n, st);
  }

 private:
  DeviceArray<unsigned char> blocks_;
  DeviceArray<int> block_index_;
  DeviceArray<int> free_slots_;
  DeviceArray<int> count_;
  DeviceArray<int> free_count_;
  DeviceArray<unsigned long long> keys_;
  DeviceArray<int> vals_;
  DevLayer d_{};
};

// Upper bounds of the slabs' fill levels, kept on the host so that the frame path never waits for a count (DESIGN.md §5).
// The projective bound is the last count seen plus the cells added since; each frame reads the count back into a ring of
// pinned slots, and the newest read-back that has landed tightens the bound. The blocks the ESDF slab and the slabs that
// follow the projective slab (colour, mesh, freespace) may hold beyond the projective fill level are counted apart.
class SlabBounds {
 public:
  ~SlabBounds() {
    for (cudaEvent_t e : count_events_)
      if (e) cudaEventDestroy(e);
  }
  int create();  // the read-back ring

  // The projective bound for a launch over the projective slab's blocks: tightened, at most the slab's capacity.
  int projectiveUpper(int capacity) {
    for (int k = 0; k < kCountRing; k++) {
      if (count_pending_[k] && cudaEventQuery(count_events_[k]) == cudaSuccess) {
        count_pending_[k] = false;
        if (count_cum_at_[k] > confirmed_cum_) {
          confirmed_cum_ = count_cum_at_[k];
          tsdf_count_confirmed_ = h_count_ring_[k];
        }
      }
    }
    tsdf_count_ub_ = clampToInt(tsdf_count_confirmed_ + (cells_cum_ - confirmed_cum_));
    return std::min(tsdf_count_ub_, capacity);
  }
  // The slots the projective slab needs to take `cells` more blocks, and those the ESDF slab needs.
  long long projectiveNeed(long long cells) { return (long long)projectiveUpper(0x7fffffff) + derived_extra_ub_ + cells; }
  long long esdfNeed(int projective_capacity) const {
    return (long long)std::min(tsdf_count_ub_, projective_capacity) + esdf_extra_ub_;
  }
  void add(long long projective, int esdf_extra, int derived_extra) {
    cells_cum_ += projective;
    tsdf_count_ub_ = clampToInt(tsdf_count_ub_ + projective);
    esdf_extra_ub_ = clampToInt((long long)esdf_extra_ub_ + esdf_extra);
    derived_extra_ub_ = clampToInt((long long)derived_extra_ub_ + derived_extra);
  }
  // After a frame's kernels on `st`: its cells join the bound, and the projective `count` is read back behind them.
  int recordFrame(const int* count, long long cells, cudaStream_t st) {
    cells_cum_ += cells;
    const int k = count_ring_head_;
    if (!count_pending_[k]) {
      count_ring_head_ = (k + 1) % kCountRing;
      NVB_CUDA(cudaMemcpyAsync(&h_count_ring_[k], count, sizeof(int), cudaMemcpyDeviceToHost, st));
      NVB_CUDA(cudaEventRecord(count_events_[k], st));
      count_pending_[k] = true;
      count_cum_at_[k] = cells_cum_;
    }
    tsdf_count_ub_ = clampToInt(tsdf_count_ub_ + cells);
    return NVB_OK;
  }
  // A projective count read with nothing in flight, and the ESDF's and derived slabs' blocks beyond it.
  void reset(int projective, int esdf_extra, int derived_extra) {
    for (bool& p : count_pending_) p = false;
    tsdf_count_confirmed_ = tsdf_count_ub_ = projective;
    confirmed_cum_ = cells_cum_;
    esdf_extra_ub_ = esdf_extra, derived_extra_ub_ = derived_extra;
  }
  void confirm(int projective) { reset(projective, esdf_extra_ub_, derived_extra_ub_); }
  // The explicit-list entry points are synchronous: afterwards the real fill level of the ESDF slab is known and replaces
  // the running sum of list lengths (which would otherwise grow the slab without need in a long session).
  int tightenEsdfBound(const LayerSlab& esdf, int projective_capacity) {
    int count = 0;
    NVB_CUDA(esdf.fillLevel(&count));
    esdf_extra_ub_ = std::max(0, count - std::min(tsdf_count_ub_, projective_capacity));
    return NVB_OK;
  }

 private:
  static int clampToInt(long long v) { return (int)std::min<long long>(v, 0x7fffffff); }

  int tsdf_count_ub_ = 0;
  int esdf_extra_ub_ = 0;     // blocks submitted to the ESDF through explicit lists
  int derived_extra_ub_ = 0;  // written to a derived slab, or kept there when nvb_scene_to_mapper replaced the projective layer
  std::unique_ptr<int[], PinnedFree> h_count_ring_;
  cudaEvent_t count_events_[kCountRing] = {};
  bool count_pending_[kCountRing] = {};
  long long count_cum_at_[kCountRing] = {};  // cells_cum_ when the read-back was enqueued
  int count_ring_head_ = 0;
  int tsdf_count_confirmed_ = 0;  // last projective count seen by the host ...
  long long confirmed_cum_ = 0;   // ... and cells_cum_ at that moment
  long long cells_cum_ = 0;       // cells added to the bound so far
};

// A caller's buffers are host or device memory (NvbMemory); any other kind is rejected before anything is enqueued.
int checkMemoryKind(int32_t memory) {
  if (memory == NVB_MEM_HOST || memory == NVB_MEM_DEVICE) return NVB_OK;
  return fail(NVB_ERR_INVALID_ARGUMENT, "bad memory kind");
}

// What a call does with a caller's list of block indices, and so how much of it is checked.
enum class BlockList {
  kLookup,     // looked up only: the hash rejects an index it cannot hold
  kInsert,     // inserted in the caller's order: every index must be in range
  kInsertSet,  // inserted as a set, since find-or-insert needs unique keys per launch: in range, then sorted in (x, y, z)
               // order with repeats dropped
};

// Checks the caller's list `*xyz` of `*n` block indices (xyz triples in host memory) by `kind` before anything is enqueued:
// a negative count or a null list with a positive count is NVB_ERR_INVALID_ARGUMENT, an index outside +-2^20 is
// NVB_ERR_INDEX_RANGE. A set is built in `set`, and *xyz and *n then name it.
int takeBlockList(BlockList kind, const int32_t** xyz, int32_t* n, std::vector<std::array<int, 3>>* set = nullptr) {
  if (*n < 0 || (*n > 0 && !*xyz)) return fail(NVB_ERR_INVALID_ARGUMENT, "bad block list");
  if (kind == BlockList::kLookup) return NVB_OK;
  const int32_t* p = *xyz;
  for (int i = 0; i < *n; i++)
    if (!indexInRange(p[3 * i], p[3 * i + 1], p[3 * i + 2])) return fail(NVB_ERR_INDEX_RANGE, "block index outside +-2^20");
  if (kind == BlockList::kInsert) return NVB_OK;
  static_assert(sizeof(std::array<int, 3>) == 3 * sizeof(int32_t), "a set entry is one xyz triple");
  set->assign(reinterpret_cast<const std::array<int, 3>*>(p), reinterpret_cast<const std::array<int, 3>*>(p) + *n);
  std::sort(set->begin(), set->end());  // std::array compares lexicographically: (x, y, z) order
  set->erase(std::unique(set->begin(), set->end()), set->end());
  *xyz = set->data()->data(), *n = (int32_t)set->size();
  return NVB_OK;
}

// Where a block-list record keeps its block index.
enum class Record {
  kXyzFirst,  // {x, y, z, ·}: the frame, colour and mark-free lists
  kXyzLast,   // {slot, x, y, z}: the dead and shape-selection lists
};

// Returns a list of n block-index records to the caller: *out_count = n, and the first min(n, cap) indices as xyz triples
// to out_xyz. `sorted` puts all n records in (x, y, z) order before the cut; unsorted, only the first min(n, cap) are read.
void writeBlockList(int4* rec, int n, Record at, bool sorted, int32_t* out_xyz, int32_t cap, int32_t* out_count) {
  if (out_count) *out_count = n;
  if (!out_xyz || cap <= 0 || n <= 0) return;
  const auto xyz = [at](const int4& r) {
    return at == Record::kXyzFirst ? std::array<int, 3>{r.x, r.y, r.z} : std::array<int, 3>{r.y, r.z, r.w};
  };
  if (sorted) std::sort(rec, rec + n, [&](const int4& a, const int4& b) { return xyz(a) < xyz(b); });
  const int k = std::min(n, (int)cap);
  for (int i = 0; i < k; i++) {
    const std::array<int, 3> b = xyz(rec[i]);
    out_xyz[3 * i] = b[0], out_xyz[3 * i + 1] = b[1], out_xyz[3 * i + 2] = b[2];
  }
}

// The device side of one call's caller buffers, all of one memory kind, for work on `st`. Device buffers are used in place.
// Host buffers are staged in stream-ordered allocations on `st` from `pool` (the device's default pool when null): an input
// is copied down when it is staged, the outputs are copied back by finish(), and the destructor frees the staging on `st`
// behind everything enqueued so far, so an early return neither leaks it nor frees memory a kernel still reads, and the host
// never waits for the release. A null or empty host buffer stays null on the device.
class CallerBuffers {
 public:
  CallerBuffers(int32_t memory, cudaStream_t st, cudaMemPool_t pool) : host_(memory == NVB_MEM_HOST), st_(st), pool_(pool) {}
  CallerBuffers(const CallerBuffers&) = delete;
  CallerBuffers& operator=(const CallerBuffers&) = delete;
  ~CallerBuffers() {
    for (const Staged& s : staged_) cudaFreeAsync(s.dev, st_);
  }

  template <typename T>
  cudaError_t in(const T* p, size_t bytes, const T** dev) {
    void* d = nullptr;
    const cudaError_t e = stage(const_cast<T*>(p), bytes, false, true, &d);
    *dev = host_ ? static_cast<const T*>(d) : p;
    return e;
  }
  // `upload` also copies the caller's contents down, so that what the kernels do not write comes back unchanged.
  template <typename T>
  cudaError_t out(T* p, size_t bytes, T** dev, bool upload = false) {
    void* d = nullptr;
    const cudaError_t e = stage(p, bytes, true, upload, &d);
    *dev = host_ ? static_cast<T*>(d) : p;
    return e;
  }
  // Host memory: the outputs are copied back and `st` is synchronised. Device memory: nothing to do.
  cudaError_t finish() {
    if (!host_) return cudaSuccess;
    for (const Staged& s : staged_) {
      if (!s.copy_back) continue;
      const cudaError_t e = cudaMemcpyAsync(s.host, s.dev, s.bytes, cudaMemcpyDeviceToHost, st_);
      if (e != cudaSuccess) return e;
    }
    return cudaStreamSynchronize(st_);
  }

 private:
  struct Staged {
    void* dev;
    void* host;
    size_t bytes;
    bool copy_back;
  };
  cudaError_t stage(void* p, size_t bytes, bool copy_back, bool copy_down, void** dev) {
    if (!host_ || !p || bytes == 0) return cudaSuccess;
    cudaError_t e = pool_ ? cudaMallocFromPoolAsync(dev, bytes, pool_, st_) : cudaMallocAsync(dev, bytes, st_);
    if (e != cudaSuccess) return e;
    staged_.push_back({*dev, p, bytes, copy_back});
    return copy_down ? cudaMemcpyAsync(*dev, p, bytes, cudaMemcpyHostToDevice, st_) : cudaSuccess;
  }

  bool host_;
  cudaStream_t st_;
  cudaMemPool_t pool_;
  std::vector<Staged> staged_;
};

// One consumer of the block-update tracker: its dirty words and list, as large as the projective slab, and the list's
// count in DeviceCounters. Producers tell a consumer only once it is initialized, which its first all-blocks update does (the
// lazy initialisation of BlocksToUpdateTracker, map/blocks_to_update_tracker.h).
struct TrackedBlocks {
  DeviceArray<int> dirty;
  DeviceArray<int> slots;
  int* count = nullptr;
  bool initialized = false;

  TrackerList list() const { return {dirty.get(), slots.get(), count}; }
};

// The mapper's device counter words, one zeroed allocation. Most belong to the ESDF update; the frame count, the error
// word, the tracker consumers' list counts and the dead, colour and freespace work counts share the block.
struct DeviceCounters {
  int work_count;
  int upd_count;
  int clr_count;
  int clr_aabb[6];
  int cleared_count;
  int ring_count[3];  // [2]: the mark kernel's count of finished CTAs
  int unused_13;
  int ring_id;
  int todo_count;
  int frame_count;
  int error;
  int cleared_seq;
  int unused_19;
  int tail_state[2];
  int dead_count;
  int dead_cleared_count;
  int ges_counts[4];
  int todo_fs_count;
  int fs_work_count;
  int cols_count;
  int color_work_count;
  int xtail[4];
  int todo_mesh_count;
  int slice_box[4];  // nvb_esdf_slice_aabb's block-column box
};

// The mapper's pinned host words, one allocation: device words copied back behind a stream, read after it synchronises.
struct HostWords {
  int frame_count;  // FrameList::read
  int union_count;  // nvb_blocks_union
  int error_main;   // the error word behind `stream` ...
  int error_esdf;   // ... and behind `esdf_stream` (enqueueErrorCopies)
};

// The ESDF integrator's device state beside its layer slab (EsdfIntegrator's members, esdf_integrator.h): the per-slot
// arrays of an update, those that carry state from one update to the next, the wavefront driver's own arrays, the
// statistics and the switch of the clear pass's parent-box pruning. The per-slot arrays follow the ESDF slab's capacity.
// The driver (esdf_persistent) is 0 for the host loop, 1 for the persistent wavefront, 2 for the gather-replay wavefront
// and 3 for the exchange-slab wavefront; the shadow slab is driver 2's, the exchange slabs and records driver 3's.
class EsdfState {
 public:
  // Reads the driver's switches, allocates every array for `capacity` ESDF slots and sets the first ring id.
  int create(NvbMapper* m, int capacity, int driver);
  // The per-slot arrays at `capacity` slots; those that carry state from one update to the next keep their contents.
  int grow(NvbMapper* m, int capacity);
  // SMs the exchange-slab wavefront leaves to concurrently running kernels; its records follow the launch's grid.
  int setReservedSms(NvbMapper* m, int n);
  // An empty ESDF layer: no cleared list, no seeds, unlinked neighbour tables and exact parent boxes, so pruning is back.
  int reset(NvbMapper* m);
  // Voxels written from outside the update: the parent boxes are no longer bounds, and the new blocks are not linked, so
  // the face-neighbour table is forgotten (it is re-resolved lazily through the hash).
  int blocksWritten(NvbMapper* m);
  // Voxels of other blocks may keep parents inside deallocated blocks: the reference clears them when they happen to be
  // candidates of a later clear pass, which the per-block parent boxes cannot tell. No pruning from here on.
  void forgetParentBoxes() { prune_ok_ = false; }
  // The parent boxes of the ESDF slots [0, n), after blocks were loaded: pruning stays exact.
  void buildParentBoxes(const DevLayer& esdf, int n, cudaStream_t st) { launchEsdfParentBoxes(esdf, n, psum_.get(), st); }
  // The slice update's column set and column list for `columns` columns.
  int reserveSliceColumns(NvbMapper* m, size_t columns);
  // The list of deallocated blocks that were on the cleared list, 3 ints per ESDF slot.
  int reserveDeadCleared(NvbMapper* m);
  void beginUpdate() { update_seq_++; }
  // An EsdfCtx with the state pointers set, the counter words in `ctr`.
  EsdfCtx ctx(DeviceCounters* ctr) const;
  cudaError_t readStats(long long out[kNumEsdfStats]) const {
    return cudaMemcpy(out, stats_.get(), kNumEsdfStats * sizeof(long long), cudaMemcpyDeviceToHost);
  }
  cudaError_t readPhaseMax(int64_t* out, int n) const {
    return cudaMemcpy(out, phase_max_.get(), (size_t)n * sizeof(long long), cudaMemcpyDeviceToHost);
  }
  int driver() const { return driver_; }
  int reservedSms() const { return reserved_sms_; }

 private:
  static constexpr int kUnlinked = 0xFE;  // neighbour-table bytes: entries 0xFEFEFEFE, "unknown" (< -1), never linked
  template <typename F>
  cudaError_t eachSlotArray(F f);
  int allocRecords(NvbMapper* m, int capacity);

  int driver_ = 1;
  int reserved_sms_ = 2;
  int split_min_k_ = 0;   // exchange-slab wavefront: smallest grid ring that fetches its candidates' blocks split
  int ges_switch_ = 160;  // gather-replay wavefront: rings with more members run as four-phase rings
  bool prune_default_ = false;  // driver 3 and not switched off (NVB_CLEAR_PRUNE=0)
  bool prune_ok_ = false;       // the parent boxes are upper bounds for every block (only driver 3 keeps them)
  int update_seq_ = 0;
  // per ESDF slot (eachSlotArray)
  DeviceArray<int4> work_;
  DeviceArray<int> upd_list_, clr_list_, cleared_list_;
  DeviceArray<int> ring_a_, ring_b_, stamp_a_, stamp_b_;
  DeviceArray<int> seed_upd_, seed_clr_;
  DeviceArray<unsigned int> psum_;
  DeviceArray<int> nbr_, nbr27_;
  DeviceArray<int> cand_stamp_, cand_a_, cand_b_;
  // the drivers' own
  DeviceArray<unsigned char> shadow_;  // driver 2: a second ESDF slab (contents only live inside one launch)
  DeviceArray<unsigned char> xslab_;   // driver 3: two slabs by ring parity of six faces per slot (7.5 KiB) ...
  DeviceArray<int> xrec_;              // ... 2 x CTAs x xseg_ candidate records of 32 ints ...
  int xseg_ = 0;
  int xseg_grid_ = 0;                  // ... for a launch of this many CTAs ...
  DeviceArray<int> xcounts_;           // ... and the barrier flags
  // the rest
  DeviceArray<unsigned long long> colset_;  // the slice update's columns
  DeviceArray<int> cols_;
  DeviceArray<int> dead_cleared_xyz_;
  DeviceArray<unsigned int> clr_bits_;  // to-clear bitmap of the current update (2048 words)
  DeviceArray<long long> stats_;
  DeviceArray<unsigned int> barrier_;
  DeviceArray<unsigned long long> phase_max_;
};

// The view bitset (1 bit per cell of a ViewGrid) and its ordered compaction into a block list (nvb_view.cu): the chained
// scan's tile states, the device ticket counter and the host's ticket base and epoch. The view path and nvb_blocks_union
// both compact through compact(), so the ticket base follows every launch that draws tickets.
class ViewCompaction {
 public:
  int create(NvbMapper* m);  // the ticket counter
  // The bitset and the tile states for `g`: 1.5 x its words + 64 (kBufferExpansionFactor, view_calculator_impl.cuh:159),
  // 2 x its tiles, both zeroed when allocated.
  int reserve(NvbMapper* m, const ViewGrid& g);
  unsigned int* bits() const { return bits_.get(); }
  // Compacts the bitset of `g` into the records {x, y, z, slot} of `list` and their number in `*count`, in linear cell
  // order. With `allocate` each block is found or inserted in `layer` and `tracker` is told. The compaction leaves the
  // bitset set: `clear` zeroes it here, otherwise the TSDF / occupancy kernel's prologue does. One or two launches on `st`.
  void compact(const ViewGrid& g, int4* list, int* count, bool allocate, const DevLayer& layer, const TrackerLists& tracker,
               int* error, bool clear, cudaStream_t st);

 private:
  DeviceArray<unsigned int> bits_;
  DeviceArray<unsigned long long> tile_state_;
  DeviceArray<unsigned int> ticket_;  // monotonically increasing
  unsigned int ticket_base_ = 0;      // the tickets drawn so far
  unsigned int epoch_ = 0;
};

// ViewpointCache of the projective integrator's ViewCalculator (C/include/nvblox/integrators/view_calculator.h:196,211-244):
// up to two (pose, sensor) -> block-list entries, newest first. A list is kept as the view bitset it was compacted from (a
// few KB on the device): a hit skips the raycast and replays the compaction + allocation, which yields the same list in the
// same order and re-allocates blocks that were deallocated in between, like allocateBlocksWhereRequired does in the reference.
class ViewpointCache {
 public:
  struct Entry {
    float T_L_C[16];
    NvbCamera cam;
    ViewGrid grid;
    long long cells;
    DeviceArray<unsigned int> bits;
  };
  // ViewpointCache::getCachedResult (view_calculator_impl.h:120-155): keyed on the pose and the sensor only. Null on a miss.
  const Entry* find(const float* T_L_C, const NvbCamera& cam) const;
  // ViewpointCache::storeResultInCache (view_calculator_impl.h:157-174): newest first, the oldest of two is dropped. The
  // bitset is copied on m->stream, so this is enqueued after the raycast and before anything that clears `bits`.
  int store(NvbMapper* m, const float* T_L_C, const NvbCamera& cam, const ViewGrid& grid, long long cells,
            const unsigned int* bits);
  void clear() { n_ = 0; }

 private:
  Entry entries_[2];
  int n_ = 0;
};

// The ring of staging buffers for host depth images and masks: the upload of frame k+1 runs on copy_stream while the
// kernels of frame k read the slot before it. A slot's `copied` event hands its upload to `stream`, and its `consumed`
// event, recorded behind the frame's last reader, lets the next upload into it start.
class HostInputRing {
 public:
  ~HostInputRing() {
    for (int k = 0; k < kStagingBuffers; k++) {
      if (copied_[k]) cudaEventDestroy(copied_[k]);
      if (consumed_[k]) cudaEventDestroy(consumed_[k]);
    }
  }
  int create();  // the events
  // The frame's depth image and optional mask of `pixels` elements each, on the device, for kernels on m->stream. Device
  // inputs are used in place (*slot = -1). Host inputs are copied into the next slot, which grows first if it is too small.
  // Every frame advances the ring.
  int stage(NvbMapper* m, int32_t memory, const float* depth, const unsigned char* mask, size_t pixels,
            const float** depth_dev, const unsigned char** mask_dev, int* slot);
  // After the frame's last reader of `slot` on `st`; nothing for -1.
  int release(int slot, cudaStream_t st) {
    if (slot < 0) return NVB_OK;
    NVB_CUDA(cudaEventRecord(consumed_[slot], st));
    used_[slot] = true;
    return NVB_OK;
  }

 private:
  DeviceArray<float> depth_[kStagingBuffers];
  DeviceArray<unsigned char> mask_[kStagingBuffers];
  cudaEvent_t copied_[kStagingBuffers] = {};
  cudaEvent_t consumed_[kStagingBuffers] = {};
  bool used_[kStagingBuffers] = {};  // `consumed` has been recorded
  unsigned long long seq_ = 0;
};

// The last integrated view (Mapper::last_posed_depth_image_, mapper.h:830-833), kept when keep_last_view is set: the depth
// image the integrators saw, its pose and its camera. The decay's exclude-last-view path reads it.
struct LastView {
  DeviceArray<float> depth;
  int rows = 0, cols = 0;
  float T_L_C[16];
  NvbCamera cam;
  bool valid = false;

  // Keeps a copy of the device image `image` (h x w), made on m->stream.
  int keep(NvbMapper* m, const float* image, int h, int w, const float* T, const NvbCamera& camera);
  void forget() { valid = false; }
};

// The block list of the last frame: records {x, y, z, slot} on the device, their count in DeviceCounters, and the pinned
// buffer read() copies a prefix of the list into.
class FrameList {
 public:
  int create(NvbMapper* m);  // the count word and the pinned buffer
  // Room for a list of every cell of `g`: 1.5 x its cells + 64.
  int reserve(NvbMapper* m, const ViewGrid& g);
  bool exists() const { return blocks_.get() != nullptr; }
  int4* blocks() const { return blocks_.get(); }
  int* count() const { return count_; }
  // The count and the first min(count, cap) block indices (writeBlockList) with ONE synchronisation: the count, a
  // speculative prefix of the list (sized from the previous read's count) and the error words travel to pinned host memory
  // behind the frame's kernels.
  int read(NvbMapper* m, int32_t* out_xyz, int32_t cap, int32_t* out_count);

 private:
  DeviceArray<int4> blocks_;
  int* count_ = nullptr;
  std::unique_ptr<int4[], PinnedFree> host_;
  int last_n_ = 0;  // the count of the last read
};

// The mesh layer's arena (nvb_mesh.cu): the segments of every mesh block's vertices, normals, triangle indices and colours
// in one set of four arrays, and a spare set that a repack moves the live segments into before the two swap. Beside them
// the kArena* state words, an update's per-entry counts and offsets, and the device copy of an explicit block list.
class MeshArena {
 public:
  // The state words, zeroed; nothing happens once they exist.
  int create(NvbMapper* m);
  size_t capacity() const { return live_.t.size(); }  // entries
  bool hasGeometry() const { return live_.v.get() != nullptr; }
  // The arrays, the state words, the counts and the offsets into `c`.
  void fill(MeshCtx* c) const;
  // The counts and offsets of an update over `list` entries.
  int reserveList(NvbMapper* m, size_t list);
  // After an update's count pass on m->stream (one synchronisation): when the update does not fit behind the fill level,
  // the arena is repacked with room for it, `c` is pointed at the new arrays and the offsets are scanned again.
  int fitUpdate(NvbMapper* m, MeshCtx* c);
  // The n block indices `xyz` (host) copied to the device on m->stream and waited for; valid until the next upload.
  int upload(NvbMapper* m, const int32_t* xyz, int n, const int** dev);
  // No segments: the state words are zeroed on `st`.
  cudaError_t empty(cudaStream_t st) { return cudaMemsetAsync(state_.get(), 0, kArenaInts * sizeof(int), st); }
  // The state words, a blocking copy.
  cudaError_t readState(int out[kArenaInts]) const {
    return cudaMemcpy(out, state_.get(), kArenaInts * sizeof(int), cudaMemcpyDeviceToHost);
  }

 private:
  // One arena of `entries` entries: 3 floats per entry in v and n, 1 int in t and 4 bytes in c.
  struct Geometry {
    DeviceArray<float> v, n;
    DeviceArray<int> t;
    DeviceArray<unsigned char> c;
    cudaError_t grow(NvbMapper* m, size_t entries) {
      cudaError_t e = v.grow(m, 3 * entries, 3 * entries);
      if (e == cudaSuccess) e = n.grow(m, 3 * entries, 3 * entries);
      if (e == cudaSuccess) e = t.grow(m, entries, entries);
      if (e == cudaSuccess) e = c.grow(m, 4 * entries, 4 * entries);
      return e;
    }
  };
  // Moves the live segments into the spare arrays with at least `need` free entries behind them, then swaps the two.
  int repack(NvbMapper* m, long long need, const MeshCtx& c);

  Geometry live_, spare_;
  DeviceArray<int> state_;
  DeviceArray<int> counts_, offsets_;
  DeviceArray<int> xyz_;
};

// The slots [0, hw) of a layer in (x, y, z) block-index order, sorted on the device: their packIndex keys and the slots,
// each followed by its sorted copy, and the radix sort's scratch. Free slots sort last.
class SlotOrder {
 public:
  // Sorts the slots of [0, hw) of `layer` on m->stream (two launches); *sorted is the list of hw sorted slots.
  int sort(NvbMapper* m, const DevLayer& layer, int hw, const int** sorted);

 private:
  DeviceArray<unsigned long long> keys_;  // 2 x hw
  DeviceArray<int> slots_;                // 2 x hw
  DeviceArray<unsigned char> temp_;
};

// The ground-plane estimator (GroundPlaneEstimator, experimental/ground_plane/): the TSDF slots' order, the zero crossings'
// counts and totals, the crossings and candidates of the last computation (its optionals), the RANSAC fit's generator
// states, costs, planes and result word, nvb_ransac_fit_plane's copy of its points, and the last plane.
class GroundPlaneEstimator {
 public:
  // GroundPlaneEstimator::computeGroundPlane on the TSDF layer with m->gp. The state is reset first, and again when the
  // fit fails or returns an error.
  int compute(NvbMapper* m, float plane[4], int32_t* found);
  void lastPlane(float plane[4], int32_t* found) const {
    *found = found_ ? 1 : 0;
    if (found_ && plane) std::memcpy(plane, plane_, sizeof(plane_));
  }
  // The first min(n, cap) crossings or candidates of the last computation, as xyz triples.
  int points(NvbMapper* m, int32_t which, float* xyz, int32_t cap, int32_t* n, int32_t* valid) const;
  // RansacPlaneFitter::fit on n >= 3 points (xyz triples in `memory`).
  int fitPoints(NvbMapper* m, const float* xyz, int32_t memory, int n, int iterations, float threshold, float plane[4],
                int32_t* found);

 private:
  int ransacFit(NvbMapper* m, const float4* pts, int n, int iterations, float threshold, float plane[4], int* found);
  void reset() {  // GroundPlaneEstimator::resetInternal
    valid_ = found_ = false;
    num_crossings_ = num_candidates_ = 0;
  }

  SlotOrder order_;
  DeviceArray<int2> counts_;
  DeviceArray<int> totals_;
  DeviceArray<float3> crossings_;
  DeviceArray<float4> candidates_;
  DeviceArray<float4> fit_points_;
  DeviceArray<unsigned char> states_;  // curand_init(1234, i, 0) for each state of ransacStateBytes() bytes
  DeviceArray<float> costs_;           // per iteration
  DeviceArray<float4> planes_;
  DeviceArray<float> result_;  // {nx, ny, nz, d, found}
  bool valid_ = false;         // crossings and candidates of the last computation are kept
  int num_crossings_ = 0, num_candidates_ = 0;
  bool found_ = false;
  float plane_[4] = {0, 0, 0, 0};
};

// A published output's device buffer and its size in bytes.
struct DeviceBytes {
  const void* p;
  size_t bytes;
};

// Dynamics detection's outputs of the last frame (DynamicsDetection, dynamics/dynamics_detection.h), sized by pixels: the
// staged depth, the mask, the filtered mask, the overlay and the points, with the tile counts, the point total and the
// published rows and cols. Also the scratch of the connected-component filter (MaskPreprocessor).
class DynamicsOutputs {
 public:
  // DynamicsDetection::computeDynamics on m->stream: the caller's depth image of a.rows x a.cols pixels (in `memory`) is
  // staged, `a` gets the output buffers and the size is published. The other fields of `a` are the caller's.
  int compute(NvbMapper* m, const float* depth, int32_t memory, DynamicsArgs a);
  // The filter's labels and sizes for a->drows x a->dcols pixels (at least one), into `a`.
  int reserveComponents(NvbMapper* m, CcArgs* a);
  int rows() const { return rows_; }
  int cols() const { return cols_; }
  DeviceBytes mask() const { return {mask_.get(), (size_t)rows_ * cols_}; }
  DeviceBytes overlay() const { return {overlay_.get(), (size_t)rows_ * cols_ * 3}; }
  DeviceBytes points(int k) const { return {points_.get(), (size_t)k * 3 * sizeof(float)}; }
  // The number of points of the last detection, read on `st` and waited for; 0 before the first.
  int pointCount(int* n, cudaStream_t st) const;
  void deviceBuffers(NvbDynamicsBuffers* out) const {
    out->depth = depth_.get(), out->mask = mask_.get(), out->cleaned_mask = clean_.get(), out->overlay = overlay_.get();
    out->points = points_.get(), out->num_points = totals_.get();
    out->rows = rows_, out->cols = cols_;
  }

 private:
  // Grows the per-pixel buffers (nothing is kept: the next call rewrites them). Growing synchronises first, so that no
  // pending kernel, and no consumer ordered behind this mapper's streams, still reads the old buffers.
  int reserve(NvbMapper* m, int pixels);

  DeviceArray<float> depth_;
  DeviceArray<unsigned char> mask_, clean_, overlay_;
  DeviceArray<float> points_;
  DeviceArray<int2> counts_;
  DeviceArray<int> totals_;  // {points, 0}
  int rows_ = 0, cols_ = 0;
  DeviceArray<int> cc_labels_, cc_sizes_;
};

// The image masker's outputs of the last split (ImageMasker, semantics/image_masker.h): background, foreground and overlay,
// sized by depth pixels, the min-depth scratch, sized by mask pixels, and the published rows, cols and overlay flag.
class MaskerOutputs {
 public:
  // ImageMasker::splitImageOnGPU on m->stream, without a synchronisation: the caller's depth image and mask (sizes in `a`,
  // in `memory`) are staged, `a` gets the outputs (the overlay only `with_overlay`) and the sizes are published. The other
  // fields of `a` are the caller's.
  int split(NvbMapper* m, const float* depth, const uint8_t* mask, int32_t memory, MaskerArgs a, bool with_overlay);
  // The buffer and byte count that `which` (NvbSplitOutput) names, and its size; an overlay that was not made has none.
  int output(int32_t which, DeviceBytes* out, int32_t* rows, int32_t* cols) const;
  void deviceBuffers(NvbSplitBuffers* out) const {
    out->background = background_.get(), out->foreground = foreground_.get();
    out->overlay = has_overlay_ ? overlay_.get() : nullptr;
    out->rows = rows_, out->cols = cols_;
  }

 private:
  DeviceArray<float> min_depth_;
  DeviceArray<float> background_, foreground_;
  DeviceArray<unsigned char> overlay_;
  int rows_ = 0, cols_ = 0;
  bool has_overlay_ = false;
};

// Unions of block lists: nvb_blocks_union's own list and count (so the last frame's block list survives a union), and
// the bitset and state words of the device-resident merge of segments, usable on any stream.
class BlockUnion {
 public:
  // The n device block indices `xyz` marked in the view bitset of the AABB grid `g` and compacted into the own list in
  // linear cell order; the first cap go to `out_xyz`, the count to `out_count` (one synchronisation). Four launches.
  int merge(NvbMapper* m, const int32_t* xyz, int n, const ViewGrid& g, int32_t* out_xyz, int32_t cap, int32_t* out_count);
  // The union of `num` segments (launchUnionSegments) on `st`, without a synchronisation. Five launches.
  int mergeSegments(NvbMapper* m, const int32_t* segments, int32_t num, int32_t stride, int32_t cap_entries,
                    int32_t* out_xyz, int32_t out_cap, int32_t* out_count, cudaStream_t st);
  // The error word of the last merge of segments, once the device is idle; 0 before the first.
  int readError(int32_t* error) const;

 private:
  DeviceArray<int4> list_;
  DeviceArray<int> count_;
  DeviceArray<unsigned int> bits_;
  DeviceArray<UnionState> state_;  // one
};

}  // namespace

struct NvbMapper {
  int device = 0;
  int num_sms = 132;
  cudaStream_t stream = nullptr;
  cudaStream_t copy_stream = nullptr;
  // The ESDF wavefront only touches the ESDF layer: it runs on its own stream so that the next
  // frame's raycast / compaction / TSDF update overlaps it.
  cudaStream_t esdf_stream = nullptr;
  cudaEvent_t esdf_ready = nullptr;  // TSDF chain of the update done on `stream`
  cudaEvent_t mark_done = nullptr;   // allocate + mark done on `esdf_stream`
  cudaEvent_t esdf_done = nullptr;   // wavefront done on `esdf_stream`
  bool esdf_in_flight = false;
  float voxel_size = 0.05f, block_size = 0.4f;
  NvbTsdfParams tp;
  NvbEsdfParams ep;
  NvbOccupancyParams op;
  // NVB_PROJECTIVE_TSDF or NVB_PROJECTIVE_OCCUPANCY: which voxel type the projective layer (`tsdf` below) holds
  // (ProjectiveLayerType, mapper/mapper.h:52-53).
  int projective_layer_type = 0;

  LayerSlab tsdf, esdf;
  EsdfState esdf_state;  // the ESDF integrator's state beside its slab
  LayerSlab freespace;  // FreespaceLayer of a NVB_PROJECTIVE_TSDF_WITH_FREESPACE mapper
  LayerSlab color;      // ColorLayer, created by the first nvb_mapper_integrate_color
  NvbColorParams cp{};
  DeviceArray<int4> color_work;  // blocks of the last colour frame {x, y, z, colour slot}
  DeviceArray<float> color_synth;  // sphere-traced synthetic depth
  NvbFreespaceParams fp;
  NvbEsdfSliceParams sp;
  int esdf_mode = 0;                // EsdfMode: 0 unset, 1 3-D, 2 2-D slice (mapper.h:61, src/mapper/mapper.cpp:408-470)
  long long fs_last_update_ms = 0;  // FreespaceIntegrator::last_update_time_ms_ (freespace_integrator.h:171)
  DeviceArray<int4> fs_work;
  SlabBounds bounds;

  BlockUnion block_union;

  // Mesh layer (nvb_mesh.cu): the header slab and the arena its headers point into
  LayerSlab mesh;
  // every layer of the mapper, the absent ones included
  std::array<LayerSlab*, 5> layers() { return {&tsdf, &esdf, &freespace, &color, &mesh}; }
  MeshArena mesh_arena;
  NvbMeshParams mp{1e-4f, 1, 5.0f};
  int cache_last_viewpoint = 1;
  // Mapper::do_depth_preprocessing / depth_preprocessing_num_dilations (mapper_params.h:33-42; mapper.cpp:335-352)
  int do_depth_preprocessing = 0;
  int depth_preprocessing_num_dilations = 4;
  DeviceArray<float> pre_depth;
  ViewpointCache viewpoints;
  ViewCompaction view;
  FrameList frame_list;
  HostInputRing inputs;
  int* error_dev = nullptr;  // in counters

  TrackedBlocks tracker[kNumBlocksToUpdateTypes];  // by BlocksToUpdateType

  DeviceArray<DeviceCounters> counters;  // one element
  // decay integrators
  NvbTsdfDecayParams tdp;
  NvbOccupancyDecayParams odp;
  DeviceArray<int4> dead;        // deallocated projective blocks of the last decay call
  DeviceArray<int> skip_stamp;   // per projective slot: == skip_seq -> block excluded from this decay call
  int skip_seq = 0;
  // map clearing: Mapper::cleared_blocks_ (every clearBlocksInLayers adds to it), ShapeClearer's scratch
  std::set<std::array<int, 3>> cleared_blocks;
  DeviceArray<int4> shape_sel;
  DeviceArray<NvbBoundingShape> shapes_dev;
  // ground-plane estimator (nvb_ground.cu)
  NvbGroundPlaneParams gp{};
  GroundPlaneEstimator ground;
  DynamicsOutputs dynamics;  // nvb_dynamics.cu
  MaskerOutputs masker;      // nvb_masker.cu
  cudaEvent_t dyn_event = nullptr;    // nvb_mapper_wait_for: recorded on this mapper's stream
  // CallerBuffers' staging of host buffers. Unlike the device's default pool, it keeps freed memory across synchronisations,
  // so a call does not map its staging anew each time.
  cudaMemPool_t stage_pool = nullptr;
  cudaEvent_t query_event = nullptr;  // point queries (nvb_query_*): the hand-over between this mapper and the query's stream
  int keep_last_view = 0;
  LastView last_view;
  DeviceArray<int> xyz_upload;

  std::unique_ptr<HostWords, PinnedFree> host_words;

  long long launches = 0;
  bool profiling = false;
  std::vector<StageEvent> stage_events;
  double stage_ms[kNumStages] = {0, 0, 0, 0, 0, 0};
  long long stage_calls[kNumStages] = {0, 0, 0, 0, 0, 0};
};

namespace {

cudaError_t syncAll(NvbMapper* m) {
  cudaError_t e = cudaStreamSynchronize(m->stream);
  if (e != cudaSuccess) return e;
  if (m->esdf_stream) e = cudaStreamSynchronize(m->esdf_stream);
  m->esdf_in_flight = false;
  return e;
}

template <typename T>
cudaError_t DeviceArray<T>::grow(NvbMapper* m, size_t need, size_t count, int fill, bool keep) {
  if (need <= n_) return cudaSuccess;
  count = std::max(count, need);
  if (p_) {
    const cudaError_t e = syncAll(m);
    if (e != cudaSuccess) return e;
  }
  T* q = nullptr;
  cudaError_t e = cudaMalloc(&q, count * sizeof(T));
  if (e == cudaSuccess && fill != kNoFill) e = cudaMemsetAsync(q, fill, count * sizeof(T), m->stream);
  if (e == cudaSuccess && keep && n_ > 0) e = cudaMemcpyAsync(q, p_, n_ * sizeof(T), cudaMemcpyDeviceToDevice, m->stream);
  if (e == cudaSuccess && (fill != kNoFill || keep)) e = cudaStreamSynchronize(m->stream);
  if (e != cudaSuccess) {
    cudaFree(q);
    return e;
  }
  cudaFree(p_);
  p_ = q;
  n_ = count;
  return cudaSuccess;
}

// Device-side join: later work on `stream` waits for the wavefront on `esdf_stream`.
cudaError_t joinEsdf(NvbMapper* m) {
  if (!m->esdf_in_flight) return cudaSuccess;
  m->esdf_in_flight = false;
  return cudaStreamWaitEvent(m->stream, m->esdf_done, 0);
}

int nextPow2(long long v) {
  long long p = 1;
  while (p < v) p <<= 1;
  return (int)p;
}

cudaError_t LayerSlab::create(NvbMapper* m, int capacity, int block_bytes) {
  const size_t n = capacity, bytes = n * block_bytes, hcap = nextPow2(2ll * capacity);
  LayerSlab s;
  cudaError_t e = s.blocks_.grow(m, bytes, bytes);
  if (e == cudaSuccess) e = s.block_index_.grow(m, 3 * n, 3 * n);
  if (e == cudaSuccess) e = s.free_slots_.grow(m, n, n);
  if (e == cudaSuccess) e = s.count_.grow(m, 1, 1);
  if (e == cudaSuccess) e = s.free_count_.grow(m, 1, 1);
  if (e == cudaSuccess) e = s.keys_.grow(m, hcap, hcap);
  if (e == cudaSuccess) e = s.vals_.grow(m, hcap, hcap);
  if (e == cudaSuccess) e = cudaMemsetAsync(s.blocks_.get(), 0, bytes, m->stream);
  if (e == cudaSuccess) e = cudaMemsetAsync(s.count_.get(), 0, sizeof(int), m->stream);
  if (e == cudaSuccess) e = cudaMemsetAsync(s.free_count_.get(), 0, sizeof(int), m->stream);
  if (e != cudaSuccess) return e;
  s.d_ = {s.blocks_.get(), s.block_index_.get(), s.count_.get(), s.free_slots_.get(), s.free_count_.get(), capacity,
          block_bytes, {s.keys_.get(), s.vals_.get(), (unsigned int)hcap - 1}};
  s.rehash(0, m->stream);
  *this = std::move(s);
  return cudaSuccess;
}

cudaError_t LayerSlab::grow(NvbMapper* m, int capacity) {
  if (capacity <= d_.capacity) return cudaSuccess;
  int n = 0;
  cudaError_t e = syncAll(m);
  if (e == cudaSuccess) e = fillLevel(&n);
  LayerSlab s;
  if (e == cudaSuccess) e = s.create(m, capacity, d_.block_bytes);
  const auto copy = [&](void* to, const void* from, size_t bytes) {
    if (e == cudaSuccess) e = cudaMemcpyAsync(to, from, bytes, cudaMemcpyDeviceToDevice, m->stream);
  };
  copy(s.count_.get(), count_.get(), sizeof(int));
  copy(s.free_count_.get(), free_count_.get(), sizeof(int));
  copy(s.free_slots_.get(), free_slots_.get(), (size_t)d_.capacity * sizeof(int));
  copy(s.blocks_.get(), blocks_.get(), (size_t)n * d_.block_bytes);
  copy(s.block_index_.get(), block_index_.get(), (size_t)n * 3 * sizeof(int));
  if (e != cudaSuccess) return e;
  s.rehash(n, m->stream);
  e = syncAll(m);
  if (e == cudaSuccess) *this = std::move(s);  // the old arrays leave with s
  return e;
}

// The colour, mesh and freespace slabs follow the projective slab's capacity, on their next use: L is created at that
// capacity, or grown to it.
cudaError_t followProjectiveSlab(NvbMapper* m, LayerSlab* L, int block_bytes) {
  return L->exists() ? L->grow(m, m->tsdf.capacity()) : L->create(m, m->tsdf.capacity(), block_bytes);
}

// Pinned host memory for n elements (one for a single object), owned by *out.
template <typename T>
cudaError_t allocPinned(std::unique_ptr<T, PinnedFree>* out, size_t n) {
  using E = typename std::unique_ptr<T, PinnedFree>::element_type;
  void* p = nullptr;
  const cudaError_t e = cudaMallocHost(&p, n * sizeof(E));
  if (e == cudaSuccess) out->reset(static_cast<E*>(p));
  return e;
}

int SlabBounds::create() {
  NVB_CUDA(allocPinned(&h_count_ring_, kCountRing));
  for (cudaEvent_t& e : count_events_) NVB_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  return NVB_OK;
}

int ViewCompaction::create(NvbMapper* m) {
  NVB_CUDA(ticket_.grow(m, 16, 16, 0));  // 64 bytes
  return NVB_OK;
}

int ViewCompaction::reserve(NvbMapper* m, const ViewGrid& g) {
  const size_t words = g.num_words, tiles = compactNumTiles(g);
  NVB_CUDA(bits_.grow(m, words, (size_t)(1.5 * words) + 64, 0));
  NVB_CUDA(tile_state_.grow(m, tiles, 2 * tiles, 0));
  return NVB_OK;
}

void ViewCompaction::compact(const ViewGrid& g, int4* list, int* count, bool allocate, const DevLayer& layer,
                             const TrackerLists& tracker, int* error, bool clear, cudaStream_t st) {
  CompactArgs a{};
  a.bits = bits_.get(), a.grid = g, a.frame_blocks = list, a.frame_count = count;
  a.tile_state = tile_state_.get(), a.ticket = ticket_.get(), a.ticket_base = ticket_base_, a.epoch = ++epoch_;
  a.allocate = allocate ? 1 : 0, a.layer = layer, a.error = error, a.tracker = tracker;
  launchCompactAllocate(a, st);
  if (compactUsesTickets(g)) ticket_base_ += (unsigned int)compactNumTiles(g);
  if (clear) launchClearBits(bits_.get(), g.num_words, st);
}

int HostInputRing::create() {
  for (int k = 0; k < kStagingBuffers; k++) {
    NVB_CUDA(cudaEventCreateWithFlags(&copied_[k], cudaEventDisableTiming));
    NVB_CUDA(cudaEventCreateWithFlags(&consumed_[k], cudaEventDisableTiming));
  }
  return NVB_OK;
}

int HostInputRing::stage(NvbMapper* m, int32_t memory, const float* depth, const unsigned char* mask, size_t pixels,
                         const float** depth_dev, const unsigned char** mask_dev, int* slot) {
  const int k = (int)(seq_ % kStagingBuffers);
  *depth_dev = depth, *mask_dev = mask, *slot = -1;
  if (memory == NVB_MEM_HOST) {
    if (pixels > mask_[kStagingBuffers - 1].size()) {  // the last buffer a growth replaces
      NVB_CUDA(cudaStreamSynchronize(m->copy_stream));
      for (int j = 0; j < kStagingBuffers; j++) {
        NVB_CUDA(depth_[j].grow(m, pixels, pixels));
        NVB_CUDA(mask_[j].grow(m, pixels, pixels));
        used_[j] = false;
      }
    }
    if (used_[k]) NVB_CUDA(cudaStreamWaitEvent(m->copy_stream, consumed_[k], 0));
    NVB_CUDA(cudaMemcpyAsync(depth_[k].get(), depth, pixels * sizeof(float), cudaMemcpyHostToDevice, m->copy_stream));
    if (mask) NVB_CUDA(cudaMemcpyAsync(mask_[k].get(), mask, pixels, cudaMemcpyHostToDevice, m->copy_stream));
    NVB_CUDA(cudaEventRecord(copied_[k], m->copy_stream));
    NVB_CUDA(cudaStreamWaitEvent(m->stream, copied_[k], 0));
    *depth_dev = depth_[k].get();
    *mask_dev = mask ? mask_[k].get() : nullptr;
    *slot = k;
  }
  seq_++;
  return NVB_OK;
}

int LastView::keep(NvbMapper* m, const float* image, int h, int w, const float* T, const NvbCamera& camera) {
  const size_t pixels = (size_t)h * w;
  NVB_CUDA(depth.grow(m, pixels, pixels));
  NVB_CUDA(cudaMemcpyAsync(depth.get(), image, pixels * sizeof(float), cudaMemcpyDeviceToDevice, m->stream));
  rows = h, cols = w, cam = camera, valid = true;
  memcpy(T_L_C, T, sizeof(T_L_C));
  return NVB_OK;
}

// Every per-slot array once, for f(array, elements per slot, fill byte of a new allocation, whether growth keeps the
// contents, whether reset() refills it). The kept ones carry state from one update to the next.
template <typename F>
cudaError_t EsdfState::eachSlotArray(F f) {
  cudaError_t e = cudaSuccess;
  const auto a = [&](auto& array, size_t per_slot, int fill, bool keep, bool reset) {
    if (e == cudaSuccess) e = f(array, per_slot, fill, keep, reset);
  };
  constexpr bool kReset = true;
  a(work_, 1, kNoFill, false, false);
  a(upd_list_, 1, kNoFill, false, false);
  a(clr_list_, 1, kNoFill, false, false);
  a(cleared_list_, 1, 0, kKeepContents, false);
  a(ring_a_, 1, kNoFill, false, false);
  a(ring_b_, 1, kNoFill, false, false);
  a(stamp_a_, 1, 0, kKeepContents, false);
  a(stamp_b_, 1, 0, kKeepContents, false);
  a(seed_upd_, 1, 0, kKeepContents, kReset);
  a(seed_clr_, 1, 0, kKeepContents, kReset);
  a(psum_, 2, 0, kKeepContents, kReset);
  a(nbr_, 6, kUnlinked, kKeepContents, kReset);
  a(nbr27_, 27, kUnlinked, kKeepContents, kReset);
  a(cand_stamp_, 1, 0, kKeepContents, false);
  a(cand_a_, 1, kNoFill, false, false);
  a(cand_b_, 1, kNoFill, false, false);
  return e;
}

int EsdfState::create(NvbMapper* m, int capacity, int driver) {
  driver_ = driver;
  split_min_k_ = esdfWaveXSplitMinK();
  if (const char* e = getenv("NVB_GES_SWITCH")) ges_switch_ = atoi(e);
  const char* e = getenv("NVB_CLEAR_PRUNE");
  prune_default_ = prune_ok_ = driver == 3 && !(e && atoi(e) == 0);
  if (int rc = grow(m, capacity)) return rc;
  const int one = 1;
  NVB_CUDA(cudaMemcpyAsync(&m->counters.get()->ring_id, &one, sizeof(int), cudaMemcpyHostToDevice, m->stream));
  NVB_CUDA(clr_bits_.grow(m, 2048, 2048));
  NVB_CUDA(stats_.grow(m, kNumEsdfStats, kNumEsdfStats, 0));
  NVB_CUDA(phase_max_.grow(m, kPhaseMaxEntries, kPhaseMaxEntries, 0));
  NVB_CUDA(barrier_.grow(m, 16, 16, 0));  // 64 bytes
  return NVB_OK;
}

int EsdfState::grow(NvbMapper* m, int capacity) {
  const size_t n = capacity;
  const auto grow_slots = [&](auto& a, size_t per_slot, int fill, bool keep, bool) {
    return a.grow(m, per_slot * n, per_slot * n, fill, keep);
  };
  NVB_CUDA(eachSlotArray(grow_slots));
  if (driver_ == 2) NVB_CUDA(shadow_.grow(m, n * kEsdfBlockBytes, n * kEsdfBlockBytes));
  if (driver_ == 3) {
    NVB_CUDA(xslab_.grow(m, esdfWaveXSlabBytes(capacity), esdfWaveXSlabBytes(capacity)));
    if (int rc = allocRecords(m, capacity)) return rc;
    const size_t flags = esdfWaveXFlagBytes() / sizeof(int);
    NVB_CUDA(xcounts_.grow(m, flags, flags, 0));
  }
  return NVB_OK;
}

// Candidate records of the exchange-slab wavefront: one segment per CTA of the launch, by ring parity. In a ring a CTA
// processes at most ceil(capacity / CTAs) members (seeds or candidates, dealt round-robin) and registers at most 6 face
// neighbours for each; the single-CTA tail registers at most 6 per group. So the segment is sized for the grid the launch
// really uses, which shrinks as SMs are reserved.
int EsdfState::allocRecords(NvbMapper* m, int capacity) {
  const int grid = esdfWaveXGrid(m->num_sms, reserved_sms_);
  NVB_CUDA(syncAll(m));
  xrec_ = DeviceArray<int>();  // released first: the exact size follows the grid down as well as up
  xseg_ = 6 * ((capacity + grid - 1) / grid) + 64;
  xseg_grid_ = grid;
  const size_t n = 2 * (size_t)grid * xseg_ * 32;
  NVB_CUDA(xrec_.grow(m, n, n));
  return NVB_OK;
}

int EsdfState::setReservedSms(NvbMapper* m, int n) {
  reserved_sms_ = n;
  if (xrec_.get() && esdfWaveXGrid(m->num_sms, n) != xseg_grid_) return allocRecords(m, m->esdf.capacity());
  return NVB_OK;
}

int EsdfState::reset(NvbMapper* m) {
  DeviceCounters* ctr = m->counters.get();
  NVB_CUDA(cudaMemsetAsync(&ctr->cleared_count, 0, sizeof(int), m->stream));
  NVB_CUDA(cudaMemsetAsync(&ctr->cleared_seq, 0, sizeof(int), m->stream));
  NVB_CUDA(cudaMemsetAsync(&ctr->dead_cleared_count, 0, sizeof(int), m->stream));
  const auto refill = [&](auto& a, size_t, int fill, bool, bool reset) {
    return reset ? cudaMemsetAsync(a.get(), fill, a.size() * sizeof(*a.get()), m->stream) : cudaSuccess;
  };
  NVB_CUDA(eachSlotArray(refill));
  prune_ok_ = prune_default_;
  return NVB_OK;
}

int EsdfState::blocksWritten(NvbMapper* m) {
  prune_ok_ = false;
  NVB_CUDA(cudaMemsetAsync(nbr_.get(), kUnlinked, nbr_.size() * sizeof(int), m->stream));
  NVB_CUDA(cudaStreamSynchronize(m->stream));
  return NVB_OK;
}

int EsdfState::reserveSliceColumns(NvbMapper* m, size_t columns) {
  const size_t keys = (size_t)nextPow2(2ll * columns);
  NVB_CUDA(colset_.grow(m, keys, keys));
  NVB_CUDA(cols_.grow(m, 2 * columns, 2 * columns));
  return NVB_OK;
}

int EsdfState::reserveDeadCleared(NvbMapper* m) {
  const size_t n = 3 * (size_t)m->esdf.capacity();
  NVB_CUDA(dead_cleared_xyz_.grow(m, n, n, kNoFill, kKeepContents));
  return NVB_OK;
}

EsdfCtx EsdfState::ctx(DeviceCounters* ctr) const {
  EsdfCtx c{};
  c.work = work_.get(), c.work_count = &ctr->work_count;
  c.upd_list = upd_list_.get(), c.upd_count = &ctr->upd_count;
  c.clr_list = clr_list_.get(), c.clr_count = &ctr->clr_count;
  c.clr_aabb = ctr->clr_aabb;
  c.cleared_list = cleared_list_.get(), c.cleared_count = &ctr->cleared_count;
  c.ring_a = ring_a_.get(), c.ring_b = ring_b_.get();
  c.ring_count = ctr->ring_count;
  c.tail_state = ctr->tail_state;
  c.stamp_a = stamp_a_.get(), c.stamp_b = stamp_b_.get();
  c.ring_id = &ctr->ring_id;
  c.nbr = nbr_.get(), c.seed_upd = seed_upd_.get(), c.seed_clr = seed_clr_.get();
  c.clr_bits = clr_bits_.get();
  c.psum = psum_.get(), c.prune = (prune_ok_ && driver_ == 3) ? 1 : 0;
  c.nbr27 = nbr27_.get(), c.shadow = shadow_.get(), c.cand_stamp = cand_stamp_.get();
  c.xslab = xslab_.get(), c.xrec = xrec_.get(), c.xtail = ctr->xtail, c.xseg = xseg_, c.xcounts = xcounts_.get();
  c.xsplit_min_k = split_min_k_;
  c.ges_counts = ctr->ges_counts;
  c.cand_a = cand_a_.get(), c.cand_b = cand_b_.get(), c.ges_switch = ges_switch_;
  c.colset_keys = colset_.get(), c.colset_mask = colset_.size() ? (unsigned int)(colset_.size() - 1) : 0u;
  c.cols = cols_.get(), c.cols_count = &ctr->cols_count;
  c.dead_cleared_xyz = dead_cleared_xyz_.get();
  c.dead_cleared_count = dead_cleared_xyz_.get() ? &ctr->dead_cleared_count : nullptr;
  c.cleared_seq = &ctr->cleared_seq;
  c.update_seq = update_seq_;
  c.barrier = barrier_.get();
  c.phase_max = phase_max_.get();
  c.stats = stats_.get();
  return c;
}

constexpr int kHostListCap = 1 << 15;  // entries of the pinned frame-list buffer (512 KiB)

// ---- The block-update tracker: which consumers are told when a block changes, and how each one is refilled and reset.

// The consumers the mapper has: the ESDF always, the freespace layer on a TSDF-with-freespace mapper, the mesh once its
// layer exists. Their arrays follow the projective slab's capacity and keep their contents.
int growTracker(NvbMapper* m, int cap) {
  const bool has[kNumBlocksToUpdateTypes] = {true, m->freespace.exists(), m->mesh.exists()};
  DeviceCounters* ctr = m->counters.get();
  int* const count[kNumBlocksToUpdateTypes] = {&ctr->todo_count, &ctr->todo_fs_count, &ctr->todo_mesh_count};
  const size_t n = cap;
  for (int k = 0; k < kNumBlocksToUpdateTypes; k++) {
    if (!has[k]) continue;
    TrackedBlocks& t = m->tracker[k];
    NVB_CUDA(t.dirty.grow(m, n, n, 0, kKeepContents));
    NVB_CUDA(t.slots.grow(m, n, n, 0, kKeepContents));
    t.count = count[k];
  }
  return NVB_OK;
}

// The lists a producer appends to: those of the consumers whose tracking has started.
TrackerLists trackerListsToTell(const NvbMapper* m) {
  TrackerLists l{};
  for (int k = 0; k < kNumBlocksToUpdateTypes; k++)
    if (m->tracker[k].initialized) l.list[k] = m->tracker[k].list();
  return l;
}

// The list consumer k updates from: the blocks told since its last update or, on its first update, after a reset and
// with update_full_layer, every block (BlocksToUpdateState::setUpdateAllBlocks, map/blocks_to_update_tracker.cpp:107-124,
// src/mapper/mapper.cpp:523-537). Like setUpdateAllBlocks, the all-blocks list drops the pending entries, so no slot is
// listed twice.
int startTrackerUpdate(NvbMapper* m, int k, bool update_full_layer) {
  TrackedBlocks& t = m->tracker[k];
  if (t.initialized && !update_full_layer) return NVB_OK;
  NVB_CUDA(cudaMemsetAsync(t.count, 0, sizeof(int), m->stream));
  launchTodoAll(m->tsdf.dev(), t.list(), m->stream);
  m->launches++;
  t.initialized = true;
  return NVB_OK;
}

// BlocksToUpdateTracker::removeClearedBlocksFromTracking (src/map/blocks_to_update_tracker.cpp:75-90): the dead slots of
// m->dead (*dead_count <= n of them) lose their dirty words in every consumer and leave the started consumers' lists.
void forgetDeadSlots(NvbMapper* m, const int* dead_count, int n) {
  TrackerLists all{};
  for (int k = 0; k < kNumBlocksToUpdateTypes; k++) all.list[k] = m->tracker[k].list();
  launchTrackerDropDead(m->dead.get(), dead_count, n, all, m->stream);
  m->launches++;
  for (const TrackedBlocks& t : m->tracker)
    if (t.initialized) launchDropDeadSlots(m->tsdf.dev(), t.slots.get(), t.count, m->stream), m->launches++;
}

// Every consumer forgets its pending blocks, and its next update covers every block.
int resetTracker(NvbMapper* m) {
  for (TrackedBlocks& t : m->tracker) {
    t.initialized = false;
    if (!t.dirty.get()) continue;  // a consumer the mapper does not have (yet)
    NVB_CUDA(cudaMemsetAsync(t.dirty.get(), 0, t.dirty.size() * sizeof(int), m->stream));
    NVB_CUDA(cudaMemsetAsync(t.count, 0, sizeof(int), m->stream));
  }
  return NVB_OK;
}

float logOddsFromProbability(float p);

EsdfCtx makeEsdfCtx(NvbMapper* m) {
  EsdfCtx c = m->esdf_state.ctx(m->counters.get());
  c.tsdf = m->tsdf.dev(), c.esdf = m->esdf.dev();
  c.freespace = m->freespace.dev();
  c.use_freespace = m->projective_layer_type == NVB_PROJECTIVE_TSDF_WITH_FREESPACE ? 1 : 0;
  c.error = m->error_dev;
  // esdf_integrator.cu:693-696, 672-676
  const float max_esdf_distance_vox = m->ep.max_esdf_distance_m / m->voxel_size;
  c.max_sq = max_esdf_distance_vox * max_esdf_distance_vox;
  c.max_esdf_distance_m = m->ep.max_esdf_distance_m;
  c.max_site_distance_m = m->ep.max_site_distance_vox * m->voxel_size;
  c.min_weight = m->ep.min_weight;
  c.block_size = m->block_size;
  // OccupancySiteFunctor (esdf_integrator.cu:71-75, 140-170)
  c.from_occupancy = m->projective_layer_type == NVB_PROJECTIVE_OCCUPANCY ? 1 : 0;
  c.occupied_threshold_log_odds = logOddsFromProbability(m->ep.occupied_threshold);
  return c;
}

// logOddsFromProbability (core/log_odds.h:23-30): clamp to [1e-3, 1 - 1e-3], then log(p / (1 - p)). The reference
// evaluates it on the host too (integrator members and setters), so glibc's logf is the function to match.
float logOddsFromProbability(float p) {
  p = fmaxf(1e-3f, fminf(p, 1.0f - 1e-3f));
  return logf(p / (1.0f - p));
}

Rigid rigidFromColMajor(const float* T) {
  Rigid r;
  for (int i = 0; i < 3; i++) {
    for (int j = 0; j < 3; j++) r.r[i][j] = T[j * 4 + i];
    r.t[i] = T[12 + i];
  }
  return r;
}

// Transform::inverse() for an isometry: R' = R^T, t' = -(R^T t).
Rigid invertRigid(const Rigid& T) {
  Rigid o;
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) o.r[i][j] = T.r[j][i];
  for (int i = 0; i < 3; i++) o.t[i] = -sum3(o.r[i][0] * T.t[0], o.r[i][1] * T.t[1], o.r[i][2] * T.t[2]);
  return o;
}

// Camera::getViewAABB (src/sensors/camera.cpp:31-83) + applyWorkspaceBounds
// (src/geometry/workspace_bounds.cpp:20-61) + the block-index AABB of
// getBlocksInImageViewRaycast (view_calculator_impl.cuh:137-156).
// Returns false when the workspace-clipped AABB is empty.
bool computeViewGrid(const NvbCamera& cam, const Rigid& T_L_C, float block_size, float max_dist,
                     const NvbTsdfParams& P, ViewGrid* g, long long* cells) {
  const float w = (float)cam.width, h = (float)cam.height;
  const float ux[4] = {0.0f, w, w, 0.0f};
  const float vy[4] = {0.0f, 0.0f, h, h};
  Vec3 ray[4];
  for (int k = 0; k < 4; k++) {
    // Camera::vectorFromImagePlaneCoordinates (sensors/internal/impl/camera_impl.h:89-104)
    float nx = (ux[k] - cam.cu) / cam.fu, ny = (vy[k] - cam.cv) / cam.fv;
    if (cam.has_distortion) removeDistortion(cam, nx, ny);
    ray[k] = Vec3{nx, ny, 1.0f};
  }
  const int order[4] = {2, 1, 0, 3};
  float lo[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, hi[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
  for (int k = 0; k < 8; k++) {
    const float d = (k < 4) ? 0.0f : max_dist;
    const Vec3 r = ray[order[k & 3]];
    const Vec3 c = transformPoint(T_L_C, Vec3{d * r.x, d * r.y, d * r.z});
    const float cl[3] = {c.x, c.y, c.z};
    for (int i = 0; i < 3; i++) {
      lo[i] = std::min(lo[i], cl[i]);
      hi[i] = std::max(hi[i], cl[i]);
    }
  }
  if (P.workspace_bounds_type == NVB_WS_HEIGHT_BOUNDS) {
    lo[2] = std::max(lo[2], P.workspace_min[2]);
    hi[2] = std::min(hi[2], P.workspace_max[2]);
  } else if (P.workspace_bounds_type == NVB_WS_BOUNDING_BOX) {
    for (int i = 0; i < 3; i++) {
      lo[i] = std::max(P.workspace_min[i], lo[i]);
      hi[i] = std::min(P.workspace_max[i], hi[i]);
    }
  }
  if (lo[0] > hi[0] || lo[1] > hi[1] || lo[2] > hi[2]) return false;
  const int3 mn = blockIndexFromPosition(block_size, Vec3{lo[0], lo[1], lo[2]});
  const int3 mx = blockIndexFromPosition(block_size, Vec3{hi[0], hi[1], hi[2]});
  g->min_index = mn;
  g->size = make_int3(mx.x - mn.x + 1, mx.y - mn.y + 1, mx.z - mn.z + 1);
  *cells = (long long)g->size.x * g->size.y * g->size.z;
  if (*cells <= 0 || *cells > 0x7fffffffll) {
    *cells = -1;
    return false;
  }
  g->linear_size = (int)*cells;
  g->num_words = (g->linear_size + 31) / 32;
  return true;
}

void beginStageOn(NvbMapper* m, int stage, cudaStream_t st) {
  if (!m->profiling) return;
  StageEvent ev;
  ev.stage = stage;
  cudaEventCreate(&ev.start), cudaEventCreate(&ev.stop);
  cudaEventRecord(ev.start, st);
  m->stage_events.push_back(ev);
}
void endStageOn(NvbMapper* m, cudaStream_t st) {
  if (!m->profiling) return;
  cudaEventRecord(m->stage_events.back().stop, st);
}
void beginStage(NvbMapper* m, int stage) { beginStageOn(m, stage, m->stream); }
void endStage(NvbMapper* m) { endStageOn(m, m->stream); }
void collectStages(NvbMapper* m) {
  for (auto& ev : m->stage_events) {
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, ev.start, ev.stop) == cudaSuccess) {
      m->stage_ms[ev.stage] += ms;
      m->stage_calls[ev.stage]++;
    }
    cudaEventDestroy(ev.start), cudaEventDestroy(ev.stop);
  }
  m->stage_events.clear();
}

// The capacity a slab of `capacity` slots needs to hold `need` blocks: doubled until they fit, and at most 2^28. `what`
// names the slab in the error.
int grownCapacity(int capacity, long long need, const char* what, int* out) {
  long long cap = capacity;
  while (cap < need) cap *= 2;
  if (cap > (1ll << 28)) return fail(NVB_ERR_CAPACITY, std::string(what) + " would exceed 2^28 blocks");
  *out = (int)cap;
  return NVB_OK;
}

// Room in the projective slab for `cells` more blocks beyond its bound, without raising it. Growing to the capacity the slab
// already has changes nothing.
int ensureTsdfCapacity(NvbMapper* m, long long cells) {
  if (m->bounds.projectiveNeed(cells) <= m->tsdf.capacity()) return NVB_OK;
  // refine the bound with a synchronous read
  NVB_CUDA(syncAll(m));
  int count = 0, cap = 0, rc;
  NVB_CUDA(m->tsdf.highWaterMark(&count));
  m->bounds.confirm(count);
  if ((rc = grownCapacity(m->tsdf.capacity(), m->bounds.projectiveNeed(cells), "TSDF layer", &cap))) return rc;
  NVB_CUDA(m->tsdf.grow(m, cap));
  return growTracker(m, cap);
}

int ensureEsdfCapacity(NvbMapper* m, long long need) {
  int cap = 0, rc;
  if (need <= m->esdf.capacity()) return NVB_OK;
  if ((rc = grownCapacity(m->esdf.capacity(), need, "ESDF layer", &cap))) return rc;
  NVB_CUDA(m->esdf.grow(m, cap));
  return m->esdf_state.grow(m, cap);
}

// Every call that adds blocks reserves room through its slab's kind. The projective slab (TSDF or occupancy) counts them in
// its bound. ESDF blocks from explicit lists, and those of a slab that follows the projective slab (colour, mesh, freespace),
// count beyond it; such a slab then follows the projective slab's capacity.
int reserveProjective(NvbMapper* m, long long n) {
  const int rc = ensureTsdfCapacity(m, n);
  if (rc == NVB_OK) m->bounds.add(n, 0, 0);
  return rc;
}
int reserveEsdf(NvbMapper* m, int n) {
  m->bounds.add(0, n, 0);
  return ensureEsdfCapacity(m, m->bounds.esdfNeed(m->tsdf.capacity()));
}
int reserveDerived(NvbMapper* m, LayerSlab* L, int n) {
  m->bounds.add(0, 0, n);
  const int rc = ensureTsdfCapacity(m, 0);
  if (rc) return rc;
  NVB_CUDA(followProjectiveSlab(m, L, L->dev().block_bytes));
  return NVB_OK;
}

int checkDeviceError(NvbMapper* m) {
  int err = 0;
  NVB_CUDA(cudaMemcpy(&err, m->error_dev, sizeof(int), cudaMemcpyDeviceToHost));
  if (err) {
    cudaMemsetAsync(m->error_dev, 0, sizeof(int), m->stream);
    cudaStreamSynchronize(m->stream);
    if (err & 2) return fail(NVB_ERR_INDEX_RANGE, "a block index does not fit the 21-bit hash key");
    if (err & 4) return fail(NVB_ERR_CAPACITY, "a block-list segment of the multi-GPU merge overflowed (nvb_mapper_append_frame_blocks)");
    if (err & 8) return fail(NVB_ERR_CAPACITY, "a candidate-record segment of the exchange-slab ESDF wavefront overflowed");
    // Roll the overflow back: find-or-insert left the keys it could not serve in the hash (value -1) and the fill level
    // above the capacity. Clamp the level and rebuild the hashes from the live slots, so that the same indices can be
    // allocated again once the caller has made room (or after the next growth).
    syncAll(m);
    for (LayerSlab* L : m->layers()) {
      int count = 0;
      if (L->highWaterMark(&count) != cudaSuccess || count <= L->capacity()) continue;
      cudaMemcpyAsync(L->dev().count, &L->dev().capacity, sizeof(int), cudaMemcpyHostToDevice, m->stream);
      L->rehash(L->capacity(), m->stream);
      cudaStreamSynchronize(m->stream);
    }
    return fail(NVB_ERR_CAPACITY, "a layer slab overflowed on the device");
  }
  return NVB_OK;
}

int validateFrameArgs(const NvbMapper* m, const float* depth, int32_t memory, int rows, int cols, const float* T,
                      const NvbCamera* cam) {
  if (!m || !depth || !T || !cam) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  if (rows <= 0 || cols <= 0) return fail(NVB_ERR_INVALID_ARGUMENT, "image must have positive size");
  if (!(cam->fu != 0.0f) || !(cam->fv != 0.0f)) return fail(NVB_ERR_INVALID_ARGUMENT, "camera focal length is zero");
  return checkMemoryKind(memory);
}

// arePosesClose (C/src/geometry/transforms.cpp:20-36) in binary32, Eigen::AngleAxisf(R).angle() through the quaternion.
bool posesClose(const float* T1, const float* T2, float tol_m, float tol_deg) {
  auto R_ = [](const float* T, int i, int j) { return T[j * 4 + i]; };
  float inv[16] = {0};
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) inv[j * 4 + i] = R_(T1, j, i);
  for (int i = 0; i < 3; i++) inv[12 + i] = -(inv[0 * 4 + i] * T1[12] + (inv[1 * 4 + i] * T1[13] + inv[2 * 4 + i] * T1[14]));
  float R[3][3], t[3];
  for (int i = 0; i < 3; i++) {
    for (int j = 0; j < 3; j++) R[i][j] = (R_(inv, i, 0) * R_(T2, 0, j) + R_(inv, i, 1) * R_(T2, 1, j)) + R_(inv, i, 2) * R_(T2, 2, j);
    t[i] = ((R_(inv, i, 0) * T2[12] + R_(inv, i, 1) * T2[13]) + R_(inv, i, 2) * T2[14]) + inv[12 + i];
  }
  if (std::sqrt(t[0] * t[0] + (t[1] * t[1] + t[2] * t[2])) > tol_m) return false;
  float w, x, y, z;
  const float tr = R[0][0] + R[1][1] + R[2][2];
  if (tr > 0.0f) {
    float q = std::sqrt(tr + 1.0f);
    w = 0.5f * q;
    q = 0.5f / q;
    x = (R[2][1] - R[1][2]) * q, y = (R[0][2] - R[2][0]) * q, z = (R[1][0] - R[0][1]) * q;
  } else {
    int i = 0;
    if (R[1][1] > R[0][0]) i = 1;
    if (R[2][2] > R[i][i]) i = 2;
    const int j = (i + 1) % 3, k = (j + 1) % 3;
    float q = std::sqrt(R[i][i] - R[j][j] - R[k][k] + 1.0f);
    float v[3];
    v[i] = 0.5f * q;
    q = 0.5f / q;
    w = (R[k][j] - R[j][k]) * q;
    v[j] = (R[j][i] + R[i][j]) * q;
    v[k] = (R[k][i] + R[i][k]) * q;
    x = v[0], y = v[1], z = v[2];
  }
  const float n = std::sqrt(x * x + (y * y + z * z));
  const float angle = n != 0.0f ? 2.0f * std::atan2(n, std::fabs(w)) : 0.0f;
  const float deg = (float)((double)(angle * 180.0f) / 3.14159265358979323846);
  return !(std::fabs(deg) > tol_deg);
}
// operator==(Camera, Camera) (C/include/nvblox/sensors/internal/impl/camera_impl.h:134-156)
bool camerasEqual(const NvbCamera& a, const NvbCamera& b) {
  bool same = std::fabs((double)(a.fu - b.fu)) <= 0.1 && std::fabs((double)(a.fv - b.fv)) <= 0.1 &&
              std::fabs((double)(a.cu - b.cu)) <= 0.1 && std::fabs((double)(a.cv - b.cv)) <= 0.1 && a.width == b.width &&
              a.height == b.height && (a.has_distortion != 0) == (b.has_distortion != 0);
  if (same && a.has_distortion && b.has_distortion)
    same = a.k1 == b.k1 && a.k2 == b.k2 && a.k3 == b.k3 && a.k4 == b.k4 && a.k5 == b.k5 && a.k6 == b.k6 && a.p1 == b.p1 && a.p2 == b.p2;
  return same;
}

const ViewpointCache::Entry* ViewpointCache::find(const float* T_L_C, const NvbCamera& cam) const {
  for (int i = 0; i < n_; i++)
    if (posesClose(T_L_C, entries_[i].T_L_C, 0.001f, 0.1f) && camerasEqual(cam, entries_[i].cam)) return &entries_[i];
  return nullptr;
}

int ViewpointCache::store(NvbMapper* m, const float* T_L_C, const NvbCamera& cam, const ViewGrid& grid, long long cells,
                          const unsigned int* bits) {
  if (n_ == 2) n_ = 1;
  if (n_ == 1) std::swap(entries_[0], entries_[1]);  // the older entry's bitset is reused for the new one
  Entry& e = entries_[0];
  const size_t words = grid.num_words;
  NVB_CUDA(e.bits.grow(m, words, (size_t)(1.5 * words) + 64));
  NVB_CUDA(cudaMemcpyAsync(e.bits.get(), bits, words * sizeof(unsigned int), cudaMemcpyDeviceToDevice, m->stream));
  memcpy(e.T_L_C, T_L_C, sizeof(e.T_L_C));
  e.cam = cam, e.grid = grid, e.cells = cells;
  n_++;
  return NVB_OK;
}

// DepthPreprocessor's invalid_depth_threshold_ / invalid_depth_value_ (include/nvblox/sensors/depth_preprocessing.h)
constexpr float kInvalidDepthThreshold = 1e-2f;
constexpr float kInvalidDepthValue = 0.0f;
constexpr int kMaxDilations = 64;

// The depth-integration chain for one frame, enqueued on m->stream.
int enqueueFrame(NvbMapper* m, const float* depth, const unsigned char* mask, int mask_mode, int memory, int rows,
                 int cols, const float* T_L_C_cm, const NvbCamera* cam, float block_size, float trunc_m,
                 float max_dist, bool integrate) {
  const Rigid T_L_C = rigidFromColMajor(T_L_C_cm);
  const ViewpointCache::Entry* cached = integrate && m->cache_last_viewpoint ? m->viewpoints.find(T_L_C_cm, *cam) : nullptr;
  ViewGrid grid{};
  long long cells = 0;
  bool visible = true;
  if (cached)
    grid = cached->grid, cells = cached->cells;
  else
    visible = computeViewGrid(*cam, T_L_C, block_size, max_dist, m->tp, &grid, &cells);
  if (!visible) {
    if (cells < 0) return fail(NVB_ERR_CAPACITY, "view AABB has more than 2^31 blocks");
    NVB_CUDA(cudaMemsetAsync(m->frame_list.count(), 0, sizeof(int), m->stream));  // empty workspace -> empty list
    return NVB_OK;
  }
  int rc;
  if ((rc = m->view.reserve(m, grid)) || (rc = m->frame_list.reserve(m, grid))) return rc;
  if (integrate && (rc = ensureTsdfCapacity(m, cells))) return rc;

  const float* depth_dev;
  const unsigned char* mask_dev;
  int stage_slot;
  if ((rc = m->inputs.stage(m, memory, depth, mask, (size_t)rows * cols, &depth_dev, &mask_dev, &stage_slot))) return rc;
  if (integrate && m->do_depth_preprocessing) {
    // Mapper::preprocessDepthImageAsync (src/mapper/mapper.cpp:335-352): the integrators and the saved last view
    // both see the dilated copy (mapper_impl.h:38-76)
    // CHECK_GE(rows, 3), CHECK_GE(cols, 3) (src/sensors/depth_preprocessing.cpp:64-65)
    if (rows < 3 || cols < 3) return fail(NVB_ERR_INVALID_ARGUMENT, "depth preprocessing needs an image of at least 3x3");
    const size_t pixels = (size_t)rows * cols;
    NVB_CUDA(m->pre_depth.grow(m, pixels, pixels));
    launchDilateInvalid(depth_dev, m->pre_depth.get(), rows, cols, m->depth_preprocessing_num_dilations, kInvalidDepthThreshold,
                        kInvalidDepthValue, m->stream);
    m->launches++;
    depth_dev = m->pre_depth.get();
  }
  if (integrate && m->keep_last_view && (rc = m->last_view.keep(m, depth_dev, rows, cols, T_L_C_cm, *cam))) return rc;

  beginStage(m, 0);
  if (cached) {
    NVB_CUDA(cudaMemcpyAsync(m->view.bits(), cached->bits.get(), (size_t)grid.num_words * sizeof(unsigned int),
                             cudaMemcpyDeviceToDevice, m->stream));
  } else {
    launchViewRaycast(depth_dev, rows, cols, T_L_C, *cam, block_size, trunc_m, max_dist, m->tp.raycast_subsampling,
                      grid, m->view.bits(), m->stream);
    m->launches++;
    if (integrate && m->cache_last_viewpoint &&
        (rc = m->viewpoints.store(m, T_L_C_cm, *cam, grid, cells, m->view.bits())))
      return rc;
  }
  endStage(m);

  beginStage(m, 1);
  m->view.compact(grid, m->frame_list.blocks(), m->frame_list.count(), integrate, m->tsdf.dev(),
                  integrate ? trackerListsToTell(m) : TrackerLists{}, m->error_dev, !integrate, m->stream);
  endStage(m);
  m->launches += integrate ? 1 : 2;  // the view-only path clears the bitset itself

  if (integrate) {
    beginStage(m, 2);
    TsdfKernelParams p;
    p.block_size = block_size;
    p.voxel_size = block_size * (1.0f / kVps);       // blockSizeToVoxelSize, indexing_impl.h:26-29
    p.half_voxel_size = block_size * (0.5f / kVps);  // indexing_impl.h:75-77
    p.truncation_distance_m = trunc_m;
    p.max_integration_distance_m = max_dist;
    p.max_weight = m->tp.max_weight;
    p.invalid_depth_decay_factor = m->tp.invalid_depth_decay_factor;
    p.weighting_type = m->tp.weighting_type;
    const Rigid T_C_L = invertRigid(T_L_C);
    if (m->projective_layer_type == NVB_PROJECTIVE_OCCUPANCY) {
      // ProjectiveOccupancyIntegrator::setFunctorParameters (src/integrators/projective_occupancy_integrator.cu:41-49)
      OccKernelParams o;
      o.free_log_odds = logOddsFromProbability(m->op.free_region_occupancy_probability);
      o.occupied_log_odds = logOddsFromProbability(m->op.occupied_region_occupancy_probability);
      o.unobserved_log_odds = logOddsFromProbability(m->op.unobserved_region_occupancy_probability);
      o.occupied_half_width_m = m->op.occupied_region_half_width_m;
      o.min_log_odds = logOddsFromProbability(0.01f);
      o.max_log_odds = logOddsFromProbability(0.99f);
      launchOccupancyIntegrate(m->frame_list.blocks(), m->frame_list.count(), m->tsdf.dev().blocks, depth_dev, mask_dev,
                               mask_mode, rows, cols, T_C_L, *cam, p, o, m->num_sms, m->view.bits(), grid.num_words, m->stream);
    } else {
      launchTsdfIntegrate(m->frame_list.blocks(), m->frame_list.count(), m->tsdf.dev().blocks, depth_dev, mask_dev, mask_mode,
                          rows, cols, T_C_L, *cam, p, m->num_sms, m->view.bits(), grid.num_words, m->stream);
    }
    endStage(m);
    m->launches++;
    if ((rc = m->bounds.recordFrame(m->tsdf.dev().count, cells, m->stream))) return rc;
  }
  return m->inputs.release(stage_slot, m->stream);
}

// The error word, copied to pinned host memory behind everything that is enqueued so far on both streams: after the next
// syncAll the host knows whether any kernel raised an error without a blocking copy of its own (a 4-byte cudaMemcpy is a
// full host round trip, and the synchronous API paid two of them per frame).
int enqueueErrorCopies(NvbMapper* m) {
  HostWords* h = m->host_words.get();
  h->error_main = 0, h->error_esdf = 0;
  NVB_CUDA(cudaMemcpyAsync(&h->error_main, m->error_dev, sizeof(int), cudaMemcpyDeviceToHost, m->stream));
  if (m->esdf_stream)
    NVB_CUDA(cudaMemcpyAsync(&h->error_esdf, m->error_dev, sizeof(int), cudaMemcpyDeviceToHost, m->esdf_stream));
  return NVB_OK;
}
// After enqueueErrorCopies + syncAll.
int checkPrefetchedError(NvbMapper* m) {
  if ((m->host_words->error_main | m->host_words->error_esdf) == 0) return NVB_OK;
  return checkDeviceError(m);  // slow path: re-reads the word, rolls back, reports
}

int FrameList::create(NvbMapper* m) {
  count_ = &m->counters.get()->frame_count;
  NVB_CUDA(allocPinned(&host_, kHostListCap));
  return NVB_OK;
}

int FrameList::reserve(NvbMapper* m, const ViewGrid& g) {
  const size_t cells = g.linear_size;
  NVB_CUDA(blocks_.grow(m, cells, (size_t)std::min<long long>((long long)(1.5 * cells) + 64, 0x7fffffff)));
  return NVB_OK;
}

int FrameList::read(NvbMapper* m, int32_t* out_xyz, int32_t cap, int32_t* out_count) {
  int want = 0;
  if (out_xyz && cap > 0 && host_) {
    want = std::min<long long>(std::min<long long>(cap, kHostListCap), (long long)last_n_ * 3 / 2 + 512);
    want = (int)std::min<size_t>(want, blocks_.size());
  }
  NVB_CUDA(cudaMemcpyAsync(&m->host_words->frame_count, count_, sizeof(int), cudaMemcpyDeviceToHost, m->stream));
  if (want > 0)
    NVB_CUDA(cudaMemcpyAsync(host_.get(), blocks_.get(), (size_t)want * sizeof(int4), cudaMemcpyDeviceToHost, m->stream));
  int rc = enqueueErrorCopies(m);
  if (rc) return rc;
  NVB_CUDA(syncAll(m));
  const int n = m->host_words->frame_count;
  last_n_ = n;
  const int k = std::min(n, cap);
  int4* src = host_.get();
  std::vector<int4> tmp;
  if (out_xyz && cap > 0 && k > want) {  // the frame has more blocks than the speculative prefix: one more copy
    tmp.resize((size_t)k);
    NVB_CUDA(cudaMemcpy(tmp.data(), blocks_.get(), (size_t)k * sizeof(int4), cudaMemcpyDeviceToHost));
    src = tmp.data();
  }
  writeBlockList(src, n, Record::kXyzFirst, false, out_xyz, cap, out_count);
  return NVB_OK;
}

// writeBlockList for a list on the device, its count at `count_dev` and its records at `rec_dev`. The count is read first,
// then only the records the output needs.
int readBlockList(NvbMapper* m, const int* count_dev, const int4* rec_dev, Record at, bool sorted, int32_t* out_xyz,
                  int32_t cap, int32_t* out_count) {
  int n = 0;
  NVB_CUDA(cudaMemcpyAsync(&n, count_dev, sizeof(int), cudaMemcpyDeviceToHost, m->stream));
  NVB_CUDA(cudaStreamSynchronize(m->stream));
  std::vector<int4> rec;
  if (out_xyz && cap > 0 && n > 0) {
    rec.resize((size_t)(sorted ? n : std::min(n, (int)cap)));
    NVB_CUDA(cudaMemcpyAsync(rec.data(), rec_dev, rec.size() * sizeof(int4), cudaMemcpyDeviceToHost, m->stream));
    NVB_CUDA(cudaStreamSynchronize(m->stream));
  }
  writeBlockList(rec.data(), n, at, sorted, out_xyz, cap, out_count);
  return NVB_OK;
}

int enqueueEsdf(NvbMapper* m, const int* in_xyz_dev, int n_explicit, bool from_tracker, bool slice = false,
                const float* plane = nullptr) {
  int rc;
  // EsdfMode: a mapper's ESDF layer is 3-D or a 2-D slice, never both (src/mapper/mapper.cpp:410-415,436-441)
  const int want_mode = slice ? 2 : 1;
  if (m->esdf_mode != 0 && m->esdf_mode != want_mode)
    return fail(NVB_ERR_INVALID_ARGUMENT, "the ESDF layer of this mapper is already in the other mode (3-D vs 2-D slice)");
  m->esdf_mode = want_mode;
  const int upper = std::max(1, from_tracker ? m->bounds.projectiveUpper(m->tsdf.capacity()) : n_explicit);
  if ((rc = reserveEsdf(m, from_tracker ? 0 : n_explicit))) return rc;
  // the slice's columns: at most one per block of the projective layer
  if (slice && (rc = m->esdf_state.reserveSliceColumns(m, std::max(m->tsdf.capacity(), upper)))) return rc;
  m->esdf_state.beginUpdate();
  EsdfCtx c = makeEsdfCtx(m);
  const TrackerList todo = from_tracker ? m->tracker[kEsdfBlocks].list() : TrackerList{};
  c.tracker_dirty = todo.dirty;
  c.tracker_todo_count = todo.count;
  if (slice) {
    // getBlockAndVoxelIndexFrom1DPositionInLayer (core/internal/impl/indexing_impl.h:105-115), on the host like the
    // reference (ConstantZColumnBoundsGetter's constructor and markSitesInSlice, esdf_integrator.cu:959-962)
    auto split = [&](float p, int* b, int* v) {
      const float inv = (float)(1.0 / (double)(m->block_size * (1.0f / kVps)));
      *b = (int)std::floor(p / m->block_size);
      *v = std::min((int)((p - m->block_size * (float)*b) * inv), kVps - 1);
    };
    split(m->sp.slice_min_height_m, &c.slice_min_bz, &c.slice_min_vz);
    split(m->sp.slice_max_height_m, &c.slice_max_bz, &c.slice_max_vz);
    split(m->sp.slice_height_m, &c.slice_out_bz, &c.slice_out_vz);
    if (c.slice_max_bz < c.slice_min_bz) return fail(NVB_ERR_INVALID_ARGUMENT, "slice_max_height below slice_min_height");
    if (plane) {
      c.slice_planar = 1;
      c.plane_nx = plane[0], c.plane_ny = plane[1], c.plane_nz = plane[2], c.plane_d = plane[3];
      if (std::fabs(c.plane_nz) < 1e-4f) c.plane_nx = 0.0f, c.plane_ny = 0.0f, c.plane_nz = 1.0f, c.plane_d = 0.0f;  // checkForVerticalPlane
      c.slice_above_plane_m = m->sp.slice_height_above_plane_m;
      c.slice_thickness_m = m->sp.slice_height_thickness_m;
    }
  }
  int launches = 0;
  cudaError_t e;
  auto allocAndMark = [&](cudaStream_t st) {
    if (slice) {
      launchEsdfSliceAllocateAndMark(c, from_tracker ? nullptr : in_xyz_dev, todo.slots, todo.count,
                                     from_tracker ? upper : n_explicit, m->num_sms, st);
      m->launches += 3;
    } else {
      launchEsdfAllocate(c, from_tracker ? nullptr : in_xyz_dev, todo.slots, todo.count, from_tracker ? upper : n_explicit, st);
      launchEsdfMark(c, upper, m->num_sms, st);
      m->launches += 2;
    }
  };
  const int driver = m->esdf_state.driver();
  if (driver) {
    // The whole ESDF chain (allocate, mark, clear, wavefront) runs back to back on the side stream; the frame's
    // critical path has no cross-stream hand-over. `stream` only waits for the mark kernel: after it nothing on
    // the side stream reads the projective layer or the tracker, so the next frame's raycast / compaction /
    // TSDF update overlaps the clear pass and the wavefront. (The previous wavefront is ordered before this
    // chain by the side stream itself.)
    cudaStream_t es = m->esdf_stream;
    NVB_CUDA(cudaEventRecord(m->esdf_ready, m->stream));  // projective layer + tracker of this update are final
    NVB_CUDA(cudaStreamWaitEvent(es, m->esdf_ready, 0));
    beginStageOn(m, 3, es);
    allocAndMark(es);
    endStageOn(m, es);
    NVB_CUDA(cudaEventRecord(m->mark_done, es));
    NVB_CUDA(cudaStreamWaitEvent(m->stream, m->mark_done, 0));
    beginStageOn(m, 4, es);
    launchEsdfClear(c, m->esdf.capacity(), m->num_sms, es);
    m->launches++;
    endStageOn(m, es);
    beginStageOn(m, 5, es);
    e = driver == 3   ? launchEsdfComputeX(c, m->num_sms, m->esdf_state.reservedSms(), es, &launches)
        : driver == 2 ? launchEsdfComputeGes(c, m->num_sms, es, &launches)
                      : launchEsdfComputePersistent(c, m->num_sms, es, &launches);
    endStageOn(m, es);
    if (e == cudaSuccess) {
      NVB_CUDA(cudaEventRecord(m->esdf_done, es));
      m->esdf_in_flight = true;
    }
  } else {
    NVB_CUDA(joinEsdf(m));
    beginStage(m, 3);
    allocAndMark(m->stream);
    endStage(m);
    beginStage(m, 4);
    launchEsdfClear(c, m->esdf.capacity(), m->num_sms, m->stream);
    m->launches++;
    endStage(m);
    beginStage(m, 5);
    e = runEsdfComputeHostLoop(c, m->num_sms, m->stream, &launches);
    endStage(m);
  }
  m->launches += launches;
  if (e != cudaSuccess) return fail(NVB_ERR_CUDA, std::string("ESDF compute launch: ") + cudaGetErrorString(e));
  return NVB_OK;
}

}  // namespace

// ---------------------------------------------------------------------------
// C-ABI
// ---------------------------------------------------------------------------
extern "C" {

const char* nvb_last_error(void) { return g_last_error.c_str(); }
const char* nvb_version(void) { return "nvblox_b200 0.1 (sm_90a)"; }

int32_t nvb_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return n;
}

void nvb_default_mapper_options(NvbMapperOptions* o) {
  if (!o) return;
  o->voxel_size_m = 0.05f;
  o->device = 0;
  o->tsdf_capacity_blocks = kDefaultCapacity;
  o->esdf_capacity_blocks = kDefaultCapacity;
  o->esdf_persistent = 3;
  o->projective_layer_type = NVB_PROJECTIVE_TSDF;
  o->keep_last_view = 0;
}
void nvb_default_tsdf_params(NvbTsdfParams* p) {
  if (!p) return;
  memset(p, 0, sizeof(*p));
  p->truncation_distance_vox = 4.0f;
  p->max_integration_distance_m = 7.0f;
  p->max_weight = 5.0f;
  p->invalid_depth_decay_factor = -1.0f;
  p->weighting_type = NVB_WEIGHT_INVERSE_SQUARE;
  p->raycast_subsampling = 4;
  p->workspace_bounds_type = NVB_WS_UNBOUNDED;
}
void nvb_default_esdf_params(NvbEsdfParams* p) {
  if (!p) return;
  p->max_esdf_distance_m = 2.0f;
  p->max_site_distance_vox = 1.0f;
  p->min_weight = 1e-4f;
  p->occupied_threshold = 0.5f;
}
void nvb_default_occupancy_params(NvbOccupancyParams* p) {
  if (!p) return;
  // integrators/occupancy_integrator_params.h:21-40
  p->free_region_occupancy_probability = 0.3f;
  p->occupied_region_occupancy_probability = 0.7f;
  p->unobserved_region_occupancy_probability = 0.5f;
  p->occupied_region_half_width_m = 0.1f;
}

// Everything nvb_mapper_create allocates, on an already constructed object (so that a failure half way can be undone
// by nvb_mapper_destroy).
static int createMapperResources(const NvbMapperOptions* opts, NvbMapper* m) {
  m->device = opts->device;
  cudaDeviceProp prop;
  NVB_CUDA(cudaGetDeviceProperties(&prop, opts->device));
  m->num_sms = prop.multiProcessorCount;
  m->voxel_size = opts->voxel_size_m;
  m->block_size = opts->voxel_size_m * (float)kVps;  // voxelSizeToBlockSize (indexing_impl.h:22-24)
  nvb_default_tsdf_params(&m->tp);
  nvb_default_esdf_params(&m->ep);
  nvb_default_occupancy_params(&m->op);
  nvb_default_tsdf_decay_params(&m->tdp);
  nvb_default_occupancy_decay_params(&m->odp);
  nvb_default_freespace_params(&m->fp);
  nvb_default_esdf_slice_params(&m->sp);
  nvb_default_color_params(&m->cp);
  nvb_default_ground_plane_params(&m->gp);
  m->projective_layer_type = opts->projective_layer_type;
  m->keep_last_view = opts->keep_last_view ? 1 : 0;
  NVB_CUDA(cudaStreamCreateWithFlags(&m->stream, cudaStreamNonBlocking));
  NVB_CUDA(cudaStreamCreateWithFlags(&m->copy_stream, cudaStreamNonBlocking));
  {
    // The ESDF chain is the frame's critical path; the next frame's raycast / compaction / TSDF update only has to finish
    // before the next mark kernel, so the ESDF stream gets the highest priority.
    int lo = 0, hi = 0;
    cudaDeviceGetStreamPriorityRange(&lo, &hi);
    NVB_CUDA(cudaStreamCreateWithPriority(&m->esdf_stream, cudaStreamNonBlocking, hi));
  }
  NVB_CUDA(cudaEventCreateWithFlags(&m->esdf_ready, cudaEventDisableTiming));
  NVB_CUDA(cudaEventCreateWithFlags(&m->esdf_done, cudaEventDisableTiming));
  NVB_CUDA(cudaEventCreateWithFlags(&m->mark_done, cudaEventDisableTiming));
  {
    cudaMemPoolProps props{};
    props.allocType = cudaMemAllocationTypePinned;
    props.location.type = cudaMemLocationTypeDevice;
    props.location.id = m->device;
    NVB_CUDA(cudaMemPoolCreate(&m->stage_pool, &props));
    uint64_t keep = ~0ull;  // never release
    NVB_CUDA(cudaMemPoolSetAttribute(m->stage_pool, cudaMemPoolAttrReleaseThreshold, &keep));
  }
  const int tcap = opts->tsdf_capacity_blocks > 0 ? opts->tsdf_capacity_blocks : kDefaultCapacity;
  const int ecap = std::max(opts->esdf_capacity_blocks > 0 ? opts->esdf_capacity_blocks : kDefaultCapacity, tcap);
  int rc;
  NVB_CUDA(m->tsdf.create(m, tcap, m->projective_layer_type == NVB_PROJECTIVE_OCCUPANCY ? kOccBlockBytes : kTsdfBlockBytes));
  NVB_CUDA(m->esdf.create(m, ecap, kEsdfBlockBytes));
  if (m->projective_layer_type == NVB_PROJECTIVE_TSDF_WITH_FREESPACE)
    NVB_CUDA(m->freespace.create(m, tcap, kFreespaceBlockBytes));
  NVB_CUDA(m->counters.grow(m, 1, 1, 0));
  if ((rc = growTracker(m, tcap))) return rc;
  if ((rc = m->esdf_state.create(m, ecap, opts->esdf_persistent))) return rc;
  m->error_dev = &m->counters.get()->error;
  if ((rc = m->view.create(m))) return rc;
  NVB_CUDA(allocPinned(&m->host_words, 1));
  *m->host_words = {};
  if ((rc = m->frame_list.create(m))) return rc;
  if ((rc = m->bounds.create())) return rc;
  if ((rc = m->inputs.create())) return rc;
  NVB_CUDA(syncAll(m));
  return NVB_OK;
}

int32_t nvb_mapper_create(const NvbMapperOptions* opts, NvbMapper** out) {
  if (!opts || !out) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  if (!(opts->voxel_size_m > 0.0f)) return fail(NVB_ERR_INVALID_ARGUMENT, "voxel_size_m must be > 0");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    cudaGetLastError();
    return fail(NVB_ERR_NO_DEVICE, "no CUDA device: the depth-integration path has no CPU fallback");
  }
  if (opts->device < 0 || opts->device >= ndev) return fail(NVB_ERR_INVALID_ARGUMENT, "bad device ordinal");
  if (opts->projective_layer_type != NVB_PROJECTIVE_TSDF && opts->projective_layer_type != NVB_PROJECTIVE_OCCUPANCY &&
      opts->projective_layer_type != NVB_PROJECTIVE_TSDF_WITH_FREESPACE)
    return fail(NVB_ERR_INVALID_ARGUMENT, "unknown projective_layer_type");
  NVB_CUDA(cudaSetDevice(opts->device));
  NvbMapper* m = new NvbMapper();
  const int rc = createMapperResources(opts, m);
  if (rc != NVB_OK) {
    // no leak on a failed create: the partial object goes through the normal destructor (null handles are skipped by
    // the CUDA runtime with an error code that is cleared here; the message of the original failure is kept)
    const std::string why = g_last_error;
    nvb_mapper_destroy(m);
    cudaGetLastError();
    g_last_error = why;
    return rc;
  }
  *out = m;
  return NVB_OK;
}

void nvb_mapper_destroy(NvbMapper* m) {
  if (!m) return;
  cudaSetDevice(m->device);
  syncAll(m);
  cudaStreamSynchronize(m->copy_stream);
  collectStages(m);
  cudaEventDestroy(m->esdf_ready), cudaEventDestroy(m->esdf_done), cudaEventDestroy(m->mark_done);
  cudaStreamDestroy(m->esdf_stream);
  if (m->dyn_event) cudaEventDestroy(m->dyn_event);
  if (m->query_event) cudaEventDestroy(m->query_event);
  if (m->stage_pool) cudaMemPoolDestroy(m->stage_pool);  // a render's staging freed on a caller's stream is released once that free completes
  cudaStreamDestroy(m->stream), cudaStreamDestroy(m->copy_stream);
  delete m;  // the layers, device buffers, pinned buffers, the bounds' read-back ring and the input ring free themselves
}

// Empties the layers and the state derived from their blocks: the slabs and hashes, the tracker (every consumer's next
// update covers every block), the ESDF scratch, the neighbour tables, the mesh arena and the fill-level bounds.
// nvb_mapper_clear and nvb_mapper_load_map both start from here.
static int resetLayers(NvbMapper* m) {
  NVB_CUDA(syncAll(m));
  for (LayerSlab* L : m->layers())
    if (L->exists()) NVB_CUDA(L->empty(m->stream));
  int rc;
  if ((rc = resetTracker(m))) return rc;
  if ((rc = m->esdf_state.reset(m))) return rc;
  NVB_CUDA(cudaMemsetAsync(m->error_dev, 0, sizeof(int), m->stream));
  if (m->mesh.exists()) NVB_CUDA(m->mesh_arena.empty(m->stream));
  m->bounds.reset(0, 0, 0);
  NVB_CUDA(syncAll(m));
  return NVB_OK;
}

int32_t nvb_mapper_clear(NvbMapper* m) {
  if (!m) return fail(NVB_ERR_INVALID_ARGUMENT, "null mapper");
  NVB_CUDA(cudaSetDevice(m->device));
  const int rc = resetLayers(m);
  if (rc) return rc;
  m->esdf_mode = 0;
  m->fs_last_update_ms = 0;
  m->last_view.forget();
  return NVB_OK;
}

int32_t nvb_mapper_set_tsdf_params(NvbMapper* m, const NvbTsdfParams* p) {
  if (!m || !p) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  // CHECK_GT(max_weight, 0) etc. (src/integrators/projective_tsdf_integrator.cu:61-64)
  if (!(p->max_weight > 0.0f)) return fail(NVB_ERR_INVALID_ARGUMENT, "max_weight must be > 0");
  if (!(p->truncation_distance_vox > 0.0f)) return fail(NVB_ERR_INVALID_ARGUMENT, "truncation_distance_vox must be > 0");
  if (p->raycast_subsampling < 1) return fail(NVB_ERR_INVALID_ARGUMENT, "raycast_subsampling must be >= 1");
  if (p->weighting_type < 0 || p->weighting_type > NVB_WEIGHT_LINEAR_WITH_MAX)
    return fail(NVB_ERR_INVALID_ARGUMENT, "unknown weighting_type");
  if (p->workspace_bounds_type < 0 || p->workspace_bounds_type > NVB_WS_BOUNDING_BOX)
    return fail(NVB_ERR_INVALID_ARGUMENT, "unknown workspace_bounds_type");
  m->tp = *p;
  return NVB_OK;
}
int32_t nvb_mapper_get_tsdf_params(const NvbMapper* m, NvbTsdfParams* p) {
  if (!m || !p) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  *p = m->tp;
  return NVB_OK;
}
int32_t nvb_mapper_set_esdf_params(NvbMapper* m, const NvbEsdfParams* p) {
  if (!m || !p) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  // CHECK_GT in the setters (src/integrators/esdf_integrator.cu:55-68)
  if (!(p->max_esdf_distance_m > 0.0f) || !(p->max_site_distance_vox > 0.0f) || !(p->min_weight > 0.0f))
    return fail(NVB_ERR_INVALID_ARGUMENT, "ESDF parameters must be > 0");
  // occupied_threshold: CHECK_GE(0) / CHECK_LE(1) (esdf_integrator.cu:71-75)
  if (!(p->occupied_threshold >= 0.0f && p->occupied_threshold <= 1.0f))
    return fail(NVB_ERR_INVALID_ARGUMENT, "occupied_threshold must be a probability");
  m->ep = *p;
  return NVB_OK;
}
int32_t nvb_mapper_get_esdf_params(const NvbMapper* m, NvbEsdfParams* p) {
  if (!m || !p) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  *p = m->ep;
  return NVB_OK;
}
int32_t nvb_mapper_set_occupancy_params(NvbMapper* m, const NvbOccupancyParams* p) {
  if (!m || !p) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  // CHECK(value >= 0 && value <= 1) in the probability setters (src/integrators/projective_occupancy_integrator.cu:71-99);
  // the half width has no check there
  const float probs[3] = {p->free_region_occupancy_probability, p->occupied_region_occupancy_probability,
                          p->unobserved_region_occupancy_probability};
  for (float q : probs)
    if (!(q >= 0.0f && q <= 1.0f)) return fail(NVB_ERR_INVALID_ARGUMENT, "occupancy probabilities must be in [0, 1]");
  m->op = *p;
  return NVB_OK;
}
int32_t nvb_mapper_get_occupancy_params(const NvbMapper* m, NvbOccupancyParams* p) {
  if (!m || !p) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  *p = m->op;
  return NVB_OK;
}
void nvb_default_tsdf_decay_params(NvbTsdfDecayParams* p) {
  if (!p) return;
  // integrators/tsdf_decay_integrator_params.h:21-48, internal/decay_integrator_base_params.h:22-29
  p->decay_factor = 0.95f;
  p->decayed_weight_threshold = 1e-3f;
  p->set_free_distance_on_decayed = 0;
  p->free_distance_vox = 4.0f;
  p->deallocate_decayed_blocks = 1;
}
void nvb_default_occupancy_decay_params(NvbOccupancyDecayParams* p) {
  if (!p) return;
  // integrators/occupancy_decay_integrator_params.h:21-43
  p->free_region_decay_probability = 0.55f;
  p->occupied_region_decay_probability = 0.4f;
  p->decay_to_probability = 0.5f;
  p->deallocate_decayed_blocks = 1;
}
int32_t nvb_mapper_set_tsdf_decay_params(NvbMapper* m, const NvbTsdfDecayParams* p) {
  if (!m || !p) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  // CHECK_GT(decay_factor, 0) / CHECK_LT(decay_factor, 1) (src/integrators/tsdf_decay_integrator.cu:30-37)
  if (!(p->decay_factor > 0.0f && p->decay_factor < 1.0f)) return fail(NVB_ERR_INVALID_ARGUMENT, "decay_factor must be in (0, 1)");
  m->tdp = *p;
  return NVB_OK;
}
int32_t nvb_mapper_get_tsdf_decay_params(const NvbMapper* m, NvbTsdfDecayParams* p) {
  if (!m || !p) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  *p = m->tdp;
  return NVB_OK;
}
int32_t nvb_mapper_set_occupancy_decay_params(NvbMapper* m, const NvbOccupancyDecayParams* p) {
  if (!m || !p) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  // CHECKs of the setters (src/integrators/occupancy_decay_integrator.cu:24-57)
  if (!(p->free_region_decay_probability >= 0.5f && p->free_region_decay_probability <= 1.0f))
    return fail(NVB_ERR_INVALID_ARGUMENT, "free_region_decay_probability must be in [0.5, 1]");
  if (!(p->occupied_region_decay_probability >= 0.0f && p->occupied_region_decay_probability < 0.5f))
    return fail(NVB_ERR_INVALID_ARGUMENT, "occupied_region_decay_probability must be in [0, 0.5)");
  if (!(p->decay_to_probability >= 0.0f && p->decay_to_probability <= 1.0f))
    return fail(NVB_ERR_INVALID_ARGUMENT, "decay_to_probability must be a probability");
  m->odp = *p;
  return NVB_OK;
}
int32_t nvb_mapper_get_occupancy_decay_params(const NvbMapper* m, NvbOccupancyDecayParams* p) {
  if (!m || !p) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  *p = m->odp;
  return NVB_OK;
}

namespace {
// The dead list (projective capacity) and the ESDF side's dead-cleared list (ESDF capacity) of a deallocation.
int ensureRemovalScratch(NvbMapper* m) {
  const size_t dead = m->tsdf.capacity();
  NVB_CUDA(m->dead.grow(m, dead, dead));
  return m->esdf_state.reserveDeadCleared(m);
}

// Mapper::clearBlocksInLayers (src/mapper/mapper.cpp:546-634) for the n_dead {slot, x, y, z} of m->dead, whose projective
// slots the caller has freed already (the projective hash still lists them): the ESDF twins (3-D) or column blocks (2-D),
// the freespace, colour and mesh twins go, every touched hash is rebuilt without them, and the indices join
// cleared_blocks_. `removed` receives the dead list. The tracker is the caller's.
int removeDeadBlocks(NvbMapper* m, int n_dead, std::vector<int4>* removed) {
  const int* dead_count = &m->counters.get()->dead_count;
  EsdfCtx c = makeEsdfCtx(m);
  if (m->esdf_mode == 2) {
    c.slice_mode = 1;
    // getBlockIndexFromPositionInLayer of the slice heights (src/mapper/mapper.cpp:574-590)
    c.slice_min_bz = (int)std::floor(m->sp.slice_min_height_m / m->block_size);
    c.slice_max_bz = (int)std::floor(m->sp.slice_max_height_m / m->block_size);
    c.slice_out_bz = (int)std::floor(m->sp.slice_height_m / m->block_size);
  }
  launchEsdfRemoveBlocks(c, m->dead.get(), dead_count, n_dead, m->stream);
  m->esdf_state.forgetParentBoxes();
  std::vector<LayerSlab*> touched = {&m->tsdf, &m->esdf};
  if (m->freespace.exists()) {
    launchRemoveBlocks(m->freespace.dev(), m->dead.get(), dead_count, n_dead, m->stream);
    touched.push_back(&m->freespace);
  }
  if (m->color.exists()) {
    launchRemoveBlocks(m->color.dev(), m->dead.get(), dead_count, n_dead, m->stream);
    touched.push_back(&m->color);
  }
  // ColorMeshLayer::clearBlocksAsync (Mapper::clearBlocksInLayers, src/mapper/mapper.cpp:552-557): the arena segments
  // of the removed headers are no longer referenced and are dropped by the next arena repack
  if (m->mesh.exists()) {
    launchRemoveBlocks(m->mesh.dev(), m->dead.get(), dead_count, n_dead, m->stream);
    touched.push_back(&m->mesh);
  }
  for (LayerSlab* L : touched) {
    int hw = 0;
    NVB_CUDA(L->fillLevel(&hw, m->stream));
    L->rehash(hw, m->stream);
  }
  m->launches += 6;
  // cleared_blocks_.insert (mapper.cpp:631-633)
  removed->resize((size_t)n_dead);
  NVB_CUDA(cudaMemcpyAsync(removed->data(), m->dead.get(), (size_t)n_dead * sizeof(int4), cudaMemcpyDeviceToHost, m->stream));
  NVB_CUDA(cudaStreamSynchronize(m->stream));
  for (const int4& d : *removed) m->cleared_blocks.insert({d.y, d.z, d.w});
  return NVB_OK;
}
}  // namespace

int32_t nvb_mapper_decay(NvbMapper* m, const NvbDecayExclusion* exclusion, const float* depth, int32_t depth_memory,
                         int32_t rows, int32_t cols, const float* T_L_C, const NvbCamera* cam, int32_t* removed_xyz_host,
                         int32_t cap, int32_t* out_count) {
  if (!m) return fail(NVB_ERR_INVALID_ARGUMENT, "null mapper");
  if (out_count) *out_count = 0;
  if (depth) {
    int rc = validateFrameArgs(m, depth, depth_memory, rows, cols, T_L_C, cam);
    if (rc) return rc;
  }
  const int32_t* excl_xyz = exclusion ? exclusion->excluded_blocks_xyz_host : nullptr;
  int32_t ne = exclusion ? exclusion->num_excluded_blocks : 0;
  if (int rc = takeBlockList(BlockList::kLookup, &excl_xyz, &ne)) return rc;
  NVB_CUDA(cudaSetDevice(m->device));
  NVB_CUDA(syncAll(m));  // the decay touches both layers: nothing of the ESDF chain may be in flight
  const bool occupancy = m->projective_layer_type == NVB_PROJECTIVE_OCCUPANCY;
  const DevLayer& P = m->tsdf.dev();
  // scratch sized to the layer
  int rc = ensureRemovalScratch(m);
  if (rc) return rc;
  NVB_CUDA(m->skip_stamp.grow(m, P.capacity, P.capacity, 0));
  DecayArgs a{};
  a.layer = P;
  a.occupancy = occupancy ? 1 : 0;
  a.p.block_size = m->block_size;
  a.p.voxel_size = m->block_size * (1.0f / kVps);
  a.p.half_voxel_size = m->block_size * (0.5f / kVps);
  // DepthObservationSpace of Mapper::decay*ExcludeLastView (mapper_impl.h:190-203,227-243)
  a.p.max_integration_distance_m = m->tp.max_integration_distance_m;
  a.p.truncation_distance_m = m->tp.truncation_distance_vox * m->voxel_size;
  if (occupancy) {
    a.free_log_odds = logOddsFromProbability(m->odp.free_region_decay_probability);
    a.occupied_log_odds = logOddsFromProbability(m->odp.occupied_region_decay_probability);
    a.to_log_odds = logOddsFromProbability(m->odp.decay_to_probability);
    a.deallocate = m->odp.deallocate_decayed_blocks ? 1 : 0;
  } else {
    a.decay_factor = m->tdp.decay_factor;
    a.weight_threshold = m->tdp.decayed_weight_threshold;
    a.set_free_distance = m->tdp.set_free_distance_on_decayed ? 1 : 0;
    a.free_distance_m = m->tdp.free_distance_vox * m->voxel_size;  // tsdf_decay_integrator_impl.cuh:85
    a.deallocate = m->tdp.deallocate_decayed_blocks ? 1 : 0;
  }
  // block exclusion
  CallerBuffers host(NVB_MEM_HOST, m->stream, m->stage_pool);
  if (ne > 0) {
    const int* excl_dev;
    NVB_CUDA(host.in(excl_xyz, (size_t)ne * 3 * sizeof(int), &excl_dev));
    m->skip_seq++;
    launchMarkSkipped(P, excl_dev, ne, m->skip_stamp.get(), m->skip_seq, m->stream);
    a.skip_stamp = m->skip_stamp.get();
    a.skip_seq = m->skip_seq;
  }
  if (exclusion && exclusion->has_exclusion_sphere && exclusion->exclusion_radius_m * exclusion->exclusion_radius_m > 0.0f) {
    a.has_sphere = 1;
    a.cx = exclusion->exclusion_center[0], a.cy = exclusion->exclusion_center[1], a.cz = exclusion->exclusion_center[2];
    a.r2 = exclusion->exclusion_radius_m * exclusion->exclusion_radius_m;
  }
  // view exclusion
  CallerBuffers bufs(depth_memory, m->stream, m->stage_pool);
  if (depth) {
    NVB_CUDA(bufs.in(depth, (size_t)rows * cols * sizeof(float), &a.depth));
    a.rows = rows, a.cols = cols;
    a.T_C_L = invertRigid(rigidFromColMajor(T_L_C));
    a.cam = *cam;
  }
  a.dead = m->dead.get();
  a.dead_count = &m->counters.get()->dead_count;
  NVB_CUDA(cudaMemsetAsync(a.dead_count, 0, sizeof(int), m->stream));
  launchDecay(a, m->num_sms, m->stream);
  m->launches++;
  int n_dead = 0;
  NVB_CUDA(cudaMemcpyAsync(&n_dead, a.dead_count, sizeof(int), cudaMemcpyDeviceToHost, m->stream));
  NVB_CUDA(cudaStreamSynchronize(m->stream));
  if (n_dead > 0) {
    std::vector<int4> removed;
    if ((rc = removeDeadBlocks(m, n_dead, &removed))) return rc;
    writeBlockList(removed.data(), n_dead, Record::kXyzLast, false, removed_xyz_host, cap, out_count);
  }
  // BlocksToUpdateTracker::addAllBlocksToUpdate (mapper_impl.h:208-211): the next ESDF update covers every block. The
  // reset also zeroes the dirty words of the deallocated slots, so a block that gets one of them is told again.
  if ((rc = resetTracker(m))) return rc;
  NVB_CUDA(syncAll(m));
  return checkDeviceError(m);
}

void nvb_default_freespace_params(NvbFreespaceParams* p) {
  if (!p) return;
  // integrators/freespace_integrator_params.h:22-58
  p->max_tsdf_distance_for_occupancy_m = 0.15f;
  p->max_unobserved_to_keep_consecutive_occupancy_ms = 200;
  p->min_duration_since_occupied_for_freespace_ms = 1000;
  p->min_consecutive_occupancy_duration_for_reset_ms = 2000;
  p->check_neighborhood = 1;
  p->initialize_to_high_confidence_freespace = 0;
}
int32_t nvb_mapper_set_freespace_params(NvbMapper* m, const NvbFreespaceParams* p) {
  if (!m || !p) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  m->fp = *p;  // the reference's setters do not check (src/integrators/freespace_integrator.cu:35-83)
  return NVB_OK;
}
int32_t nvb_mapper_get_freespace_params(const NvbMapper* m, NvbFreespaceParams* p) {
  if (!m || !p) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  *p = m->fp;
  return NVB_OK;
}

namespace {
// FreespaceIntegrator::updateFreespaceLayer on the tracker's list (in_xyz_dev == nullptr) or on an explicit one.
int freespaceUpdateImpl(NvbMapper* m, const int* in_xyz_dev, int n_explicit, long long now_ms, const float* depth, int memory,
                        int rows, int cols, const float* T_L_C, const NvbCamera* cam, float max_view_distance_m,
                        float truncation_distance_m) {
  NVB_CUDA(followProjectiveSlab(m, &m->freespace, kFreespaceBlockBytes));
  const int upper = std::max(1, in_xyz_dev ? n_explicit : m->bounds.projectiveUpper(m->tsdf.capacity()));
  NVB_CUDA(m->fs_work.grow(m, upper, 2 * (size_t)upper));
  FreespaceArgs a{};
  a.tsdf = m->tsdf.dev(), a.fs = m->freespace.dev();
  if (in_xyz_dev) a.in_xyz = in_xyz_dev, a.n_explicit = n_explicit;
  else a.todo = m->tracker[kFreespaceBlocks].list();
  a.work = m->fs_work.get(), a.work_count = &m->counters.get()->fs_work_count, a.error = m->error_dev;
  a.max_tsdf_distance_for_occupancy_m = m->fp.max_tsdf_distance_for_occupancy_m;
  a.max_unobserved_ms = m->fp.max_unobserved_to_keep_consecutive_occupancy_ms;
  a.min_free_ms = m->fp.min_duration_since_occupied_for_freespace_ms;
  a.min_reset_ms = m->fp.min_consecutive_occupancy_duration_for_reset_ms;
  a.check_neighborhood = m->fp.check_neighborhood ? 1 : 0;
  a.init_high_confidence = m->fp.initialize_to_high_confidence_freespace ? 1 : 0;
  a.last_update_ms = m->fs_last_update_ms, a.now_ms = now_ms;
  a.p.block_size = m->block_size;
  a.p.voxel_size = m->block_size * (1.0f / kVps);
  a.p.half_voxel_size = m->block_size * (0.5f / kVps);
  a.p.max_integration_distance_m = max_view_distance_m > 0.0f ? max_view_distance_m : FLT_MAX;
  a.p.truncation_distance_m = truncation_distance_m > 0.0f ? truncation_distance_m : FLT_MAX;
  CallerBuffers bufs(memory, m->stream, m->stage_pool);
  if (depth) {
    NVB_CUDA(bufs.in(depth, (size_t)rows * cols * sizeof(float), &a.depth));
    a.rows = rows, a.cols = cols;
    a.T_C_L = invertRigid(rigidFromColMajor(T_L_C));
    a.cam = *cam;
  }
  launchFreespaceUpdate(a, upper, m->num_sms, m->stream);
  m->launches += 2;
  m->fs_last_update_ms = now_ms;
  NVB_CUDA(cudaStreamSynchronize(m->stream));
  return checkDeviceError(m);
}
}  // namespace

int32_t nvb_mapper_update_freespace(NvbMapper* m, int64_t update_time_ms, const float* depth, int32_t depth_memory,
                                    int32_t rows, int32_t cols, const float* T_L_C, const NvbCamera* cam,
                                    int32_t update_full_layer) {
  if (!m) return fail(NVB_ERR_INVALID_ARGUMENT, "null mapper");
  if (m->projective_layer_type != NVB_PROJECTIVE_TSDF_WITH_FREESPACE)
    return fail(NVB_ERR_INVALID_ARGUMENT, "the mapper has no freespace layer");  // CHECK(hasFreespaceLayer(...)), mapper_impl.h:180-181
  if (depth) {
    int rc = validateFrameArgs(m, depth, depth_memory, rows, cols, T_L_C, cam);
    if (rc) return rc;
  }
  NVB_CUDA(cudaSetDevice(m->device));
  int rc;
  if ((rc = startTrackerUpdate(m, kFreespaceBlocks, update_full_layer))) return rc;
  // kTruncationDistanceMultiplier = 2 (mapper_impl.h:157-172)
  return freespaceUpdateImpl(m, nullptr, 0, update_time_ms, depth, depth_memory, rows, cols, T_L_C, cam,
                             m->tp.max_integration_distance_m, 2.0f * (m->tp.truncation_distance_vox * m->voxel_size));
}

int32_t nvb_freespace_update_blocks(NvbMapper* m, const int32_t* blocks_xyz_host, int32_t num_blocks, int64_t update_time_ms,
                                    const float* depth, int32_t depth_memory, int32_t rows, int32_t cols, const float* T_L_C,
                                    const NvbCamera* cam, float max_view_distance_m, float truncation_distance_m) {
  if (!m) return fail(NVB_ERR_INVALID_ARGUMENT, "null mapper");
  if (m->projective_layer_type != NVB_PROJECTIVE_TSDF_WITH_FREESPACE)
    return fail(NVB_ERR_INVALID_ARGUMENT, "the mapper has no freespace layer");
  std::vector<std::array<int, 3>> set;  // a set, like every caller's list in the reference
  int rc = takeBlockList(BlockList::kInsertSet, &blocks_xyz_host, &num_blocks, &set);
  if (rc) return rc;
  if (num_blocks == 0) return NVB_OK;  // early return (:337-339)
  if (depth) {
    if ((rc = validateFrameArgs(m, depth, depth_memory, rows, cols, T_L_C, cam))) return rc;
  }
  NVB_CUDA(cudaSetDevice(m->device));
  CallerBuffers host(NVB_MEM_HOST, m->stream, m->stage_pool);
  const int* xyz_dev;
  NVB_CUDA(host.in(blocks_xyz_host, (size_t)num_blocks * 3 * sizeof(int), &xyz_dev));
  return freespaceUpdateImpl(m, xyz_dev, num_blocks, update_time_ms, depth, depth_memory, rows, cols, T_L_C, cam,
                             max_view_distance_m, truncation_distance_m);
}

int32_t nvb_mapper_decay_exclude_last_view(NvbMapper* m, const NvbDecayExclusion* exclusion, int32_t* removed_xyz_host,
                                           int32_t cap, int32_t* out_count) {
  if (!m) return fail(NVB_ERR_INVALID_ARGUMENT, "null mapper");
  if (!m->keep_last_view) return fail(NVB_ERR_INVALID_ARGUMENT, "the mapper was created without keep_last_view");
  const LastView& v = m->last_view;
  if (!v.valid)  // "Last view not set for sensor type. Decaying all voxels" (mapper_impl.h:200-203)
    return nvb_mapper_decay(m, exclusion, nullptr, 0, 0, 0, nullptr, nullptr, removed_xyz_host, cap, out_count);
  return nvb_mapper_decay(m, exclusion, v.depth.get(), NVB_MEM_DEVICE, v.rows, v.cols, v.T_L_C, &v.cam, removed_xyz_host, cap,
                          out_count);
}

int32_t nvb_mapper_clear_outside_radius(NvbMapper* m, const float center[3], float radius, int32_t* removed_xyz_host,
                                        int32_t cap, int32_t* out_count) {
  if (!m || !center) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  if (out_count) *out_count = 0;
  NVB_CUDA(cudaSetDevice(m->device));
  NVB_CUDA(syncAll(m));  // an update_esdf_async may still be reading the projective layer
  int rc = ensureRemovalScratch(m);
  if (rc) return rc;
  // getBlocksOutsideRadius over the projective layer's blocks (TSDF for kTsdf / kTsdfWithFreespace, occupancy for kOccupancy)
  int* dead_count = &m->counters.get()->dead_count;
  NVB_CUDA(cudaMemsetAsync(dead_count, 0, sizeof(int), m->stream));
  launchSelectOutsideRadius(m->tsdf.dev(), center, radius, m->block_size, m->dead.get(), dead_count, m->stream);
  m->launches++;
  int n = 0;
  NVB_CUDA(cudaMemcpyAsync(&n, dead_count, sizeof(int), cudaMemcpyDeviceToHost, m->stream));
  NVB_CUDA(cudaStreamSynchronize(m->stream));
  if (n == 0) return checkDeviceError(m);
  // {Tsdf,Occupancy}Layer::clearBlocksAsync
  launchRemoveBlocks(m->tsdf.dev(), m->dead.get(), dead_count, n, m->stream);
  m->launches++;
  forgetDeadSlots(m, dead_count, n);  // no switch to update-all (unlike the decay)
  std::vector<int4> removed;
  if ((rc = removeDeadBlocks(m, n, &removed))) return rc;
  writeBlockList(removed.data(), n, Record::kXyzLast, true, removed_xyz_host, cap, out_count);
  return checkDeviceError(m);
}

namespace {
// ShapeClearer<LayerType>::clear on `L`; `track`: the touched blocks join every initialised tracker consumer.
int clearShapesImpl(NvbMapper* m, const LayerSlab* L, int voxel_kind, bool track, const NvbBoundingShape* shapes, int32_t num_shapes,
                    int32_t* updated_xyz_host, int32_t cap, int32_t* out_count) {
  if (out_count) *out_count = 0;
  if (num_shapes < 0 || (num_shapes > 0 && !shapes)) return fail(NVB_ERR_INVALID_ARGUMENT, "bad shape list");
  for (int i = 0; i < num_shapes; i++)
    if (shapes[i].type != NVB_SHAPE_SPHERE && shapes[i].type != NVB_SHAPE_AABB)
      return fail(NVB_ERR_INVALID_ARGUMENT, "unknown shape type");  // LOG(FATAL) (bounding_shape.cpp:60-63)
  if (num_shapes == 0 || !L) return NVB_OK;
  NVB_CUDA(cudaSetDevice(m->device));
  NVB_CUDA(syncAll(m));  // an update_esdf_async may still be reading the layer
  const size_t sel = (size_t)L->capacity() + 1;  // the count, then the list
  NVB_CUDA(m->shape_sel.grow(m, sel, sel));
  NVB_CUDA(m->shapes_dev.grow(m, num_shapes, num_shapes));
  NVB_CUDA(cudaMemcpyAsync(m->shapes_dev.get(), shapes, (size_t)num_shapes * sizeof(NvbBoundingShape), cudaMemcpyHostToDevice,
                           m->stream));
  ShapeClearArgs a{};
  a.layer = L->dev();
  a.voxel_kind = voxel_kind;
  a.shapes = m->shapes_dev.get(), a.num_shapes = num_shapes;
  a.block_size = m->block_size;
  a.sel_count = reinterpret_cast<int*>(m->shape_sel.get());
  a.sel = m->shape_sel.get() + 1;
  if (track) a.tracker = trackerListsToTell(m);
  NVB_CUDA(cudaMemsetAsync(a.sel_count, 0, sizeof(int), m->stream));
  launchShapeSelect(a, m->stream);
  launchShapeClear(a, m->num_sms, m->stream);
  m->launches += 2;
  const int rc = readBlockList(m, a.sel_count, a.sel, Record::kXyzLast, true, updated_xyz_host, cap, out_count);
  return rc ? rc : checkDeviceError(m);
}
}  // namespace

int32_t nvb_mapper_clear_tsdf_inside_shapes(NvbMapper* m, const NvbBoundingShape* shapes, int32_t num_shapes,
                                            int32_t* updated_xyz_host, int32_t cap, int32_t* out_count) {
  if (!m) return fail(NVB_ERR_INVALID_ARGUMENT, "null mapper");
  // an occupancy mapper's TsdfLayer is empty: nothing is touched
  LayerSlab* L = m->projective_layer_type != NVB_PROJECTIVE_OCCUPANCY ? &m->tsdf : nullptr;
  return clearShapesImpl(m, L, 0, true, shapes, num_shapes, updated_xyz_host, cap, out_count);
}

static LayerSlab* layerOf(NvbMapper* m, int layer);
int32_t nvb_layer_clear_shapes(NvbMapper* m, int32_t layer, const NvbBoundingShape* shapes, int32_t num_shapes,
                               int32_t* updated_xyz_host, int32_t cap, int32_t* out_count) {
  if (!m) return fail(NVB_ERR_INVALID_ARGUMENT, "null mapper");
  // ShapeClearer is instantiated for the TSDF, occupancy and colour layers (src/integrators/shape_clearer.cu)
  const int kind = layer == NVB_LAYER_TSDF ? 0 : layer == NVB_LAYER_OCCUPANCY ? 1 : layer == NVB_LAYER_COLOR ? 2 : -1;
  if (kind < 0) return fail(NVB_ERR_INVALID_ARGUMENT, "shapes clear TSDF, occupancy or colour layers only");
  const LayerSlab* L = layerOf(m, layer);
  if (!L) return fail(NVB_ERR_INVALID_ARGUMENT, "the mapper has no such layer");
  return clearShapesImpl(m, L, kind, false, shapes, num_shapes, updated_xyz_host, cap, out_count);
}

int32_t nvb_mapper_get_cleared_blocks(NvbMapper* m, const int32_t* ignore_xyz, int32_t n_ignore, int32_t* out_xyz_host,
                                      int32_t cap, int32_t* out_count) {
  if (!m || !out_count) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  if (int rc = takeBlockList(BlockList::kLookup, &ignore_xyz, &n_ignore)) return rc;
  if (!out_xyz_host) {
    *out_count = (int32_t)m->cleared_blocks.size();
    return NVB_OK;
  }
  for (int i = 0; i < n_ignore; i++) m->cleared_blocks.erase({ignore_xyz[3 * i], ignore_xyz[3 * i + 1], ignore_xyz[3 * i + 2]});
  *out_count = (int32_t)m->cleared_blocks.size();
  if (*out_count > cap) return fail(NVB_ERR_CAPACITY, "more cleared blocks than the output holds");
  for (const auto& k : m->cleared_blocks) out_xyz_host = std::copy(k.begin(), k.end(), out_xyz_host);
  m->cleared_blocks.clear();
  return NVB_OK;
}

float nvb_mapper_voxel_size(const NvbMapper* m) { return m ? m->voxel_size : 0.0f; }
float nvb_mapper_block_size(const NvbMapper* m) { return m ? m->block_size : 0.0f; }

int32_t nvb_view_raycast(NvbMapper* m, const float* depth, int32_t depth_memory, int32_t rows, int32_t cols,
                         const float* T_L_C, const NvbCamera* cam, float block_size,
                         float max_integration_distance_behind_surface_m, float max_integration_distance_m,
                         int32_t* out_xyz_host, int32_t cap, int32_t* out_count) {
  int rc = validateFrameArgs(m, depth, depth_memory, rows, cols, T_L_C, cam);
  if (rc) return rc;
  if (!(block_size > 0.0f)) return fail(NVB_ERR_INVALID_ARGUMENT, "block_size must be > 0");
  NVB_CUDA(cudaSetDevice(m->device));
  if ((rc = enqueueFrame(m, depth, nullptr, 0, depth_memory, rows, cols, T_L_C, cam, block_size,
                         max_integration_distance_behind_surface_m, max_integration_distance_m, false)))
    return rc;
  return m->frame_list.read(m, out_xyz_host, cap, out_count);
}

int32_t nvb_mapper_integrate_depth_async(NvbMapper* m, const float* depth, const uint8_t* mask, int32_t mask_mode,
                                         int32_t memory, int32_t rows, int32_t cols, const float* T_L_C,
                                         const NvbCamera* cam) {
  int rc = validateFrameArgs(m, depth, memory, rows, cols, T_L_C, cam);
  if (rc) return rc;
  NVB_CUDA(cudaSetDevice(m->device));
  // max_integration_distance_behind_surface_m = truncation_distance_vox * voxel_size
  // (projective_integrator_impl.cuh:234-235)
  if (m->projective_layer_type == NVB_PROJECTIVE_OCCUPANCY &&
      m->tp.truncation_distance_vox * m->voxel_size < m->op.occupied_region_half_width_m) {
    // "truncation distance must be >= occupied region half width": the integrator raises it through its own
    // setter, so the new value persists (src/integrators/projective_occupancy_integrator.cu:51-64)
    m->tp.truncation_distance_vox = m->op.occupied_region_half_width_m / m->voxel_size;
  }
  const float trunc_m = m->tp.truncation_distance_vox * m->voxel_size;
  return enqueueFrame(m, depth, mask, mask_mode, memory, rows, cols, T_L_C, cam, m->block_size, trunc_m,
                      m->tp.max_integration_distance_m, true);
}

int32_t nvb_mapper_mark_unobserved_free_inside_radius(NvbMapper* m, const float center[3], float radius, int32_t* updated_xyz_host,
                                                      int32_t cap, int32_t* out_count) {
  if (!m || !center) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  if (!(radius > 0.0f)) return fail(NVB_ERR_INVALID_ARGUMENT, "radius must be positive");  // CHECK_GT(radius, 0.0f)
  if (out_count) *out_count = 0;
  NVB_CUDA(cudaSetDevice(m->device));
  MarkFreeArgs a{};
  const Vec3 mn{center[0] - radius, center[1] - radius, center[2] - radius};
  const Vec3 mx{center[0] + radius, center[1] + radius, center[2] + radius};
  a.lo = blockIndexFromPosition(m->block_size, mn);
  const int3 hi = blockIndexFromPosition(m->block_size, mx);
  a.size = make_int3(hi.x - a.lo.x + 1, hi.y - a.lo.y + 1, hi.z - a.lo.z + 1);
  const long long cells = (long long)a.size.x * a.size.y * a.size.z;
  if (cells <= 0 || cells > (1ll << 26)) return fail(NVB_ERR_CAPACITY, "the sphere covers more than 2^26 blocks");
  if (!indexInRange(a.lo.x, a.lo.y, a.lo.z) || !indexInRange(hi.x, hi.y, hi.z))
    return fail(NVB_ERR_INDEX_RANGE, "block index outside +-2^20");
  a.cells = (int)cells;
  int rc;
  if ((rc = reserveProjective(m, cells))) return rc;
  NVB_CUDA(syncAll(m));  // rare, synchronous call: the ESDF side stream may still be reading the projective layer
  a.layer = m->tsdf.dev();
  a.occupancy = m->projective_layer_type == NVB_PROJECTIVE_OCCUPANCY ? 1 : 0;
  a.cx = center[0], a.cy = center[1], a.cz = center[2];
  a.radius = radius;
  a.block_size = m->block_size;
  a.trunc_m = m->tp.truncation_distance_vox * m->voxel_size;  // get_truncation_distance_m(layer->voxel_size())
  a.error = m->error_dev;
  a.tracker = trackerListsToTell(m);
  DeviceArray<int4> out_dev;
  NVB_CUDA(out_dev.grow(m, (size_t)cells + 1, (size_t)cells + 1));
  a.out = out_dev.get() + 1;
  a.out_count = reinterpret_cast<int*>(out_dev.get());
  NVB_CUDA(cudaMemsetAsync(out_dev.get(), 0, sizeof(int4), m->stream));
  launchMarkFreeSphere(a, m->num_sms, m->stream);
  m->launches++;
  if ((rc = readBlockList(m, a.out_count, a.out, Record::kXyzFirst, false, updated_xyz_host, cap, out_count))) return rc;
  return checkDeviceError(m);
}

// ---------------------------------------------------------------------------
// Colour integration (nvb_color.cu)
// ---------------------------------------------------------------------------
void nvb_default_color_params(NvbColorParams* p) {
  if (!p) return;
  memset(p, 0, sizeof(*p));
  // integrators/projective_integrator_params.h:24-75, projective_appearance_integrator.h:164, rays/sphere_tracer.h:216-218
  p->max_integration_distance_m = 7.0f;
  p->truncation_distance_vox = 4.0f;
  p->max_weight = 5.0f;
  p->measurement_weight = 0.8f;
  p->sphere_tracing_ray_subsampling_factor = 4;
  p->sphere_tracer_maximum_steps = 100;
  p->sphere_tracer_maximum_ray_length_m = 7.0f;
  p->sphere_tracer_surface_distance_epsilon_vox = 0.1f;
  p->workspace_bounds_type = NVB_WS_UNBOUNDED;
}
int32_t nvb_mapper_set_color_params(NvbMapper* m, const NvbColorParams* p) {
  if (!m || !p) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  // the reference's setters CHECK these (projective_appearance_integrator.cu:168-208, projective_integrator.cpp setters)
  if (!(p->max_integration_distance_m > 0.0f) || !(p->truncation_distance_vox > 0.0f) || !(p->max_weight > 0.0f) ||
      !(p->measurement_weight > 0.0f) || !(p->measurement_weight <= 1.0f) || p->sphere_tracing_ray_subsampling_factor <= 0 ||
      p->sphere_tracer_maximum_steps <= 0 || !(p->sphere_tracer_maximum_ray_length_m > 0.0f) ||
      !(p->sphere_tracer_surface_distance_epsilon_vox > 0.0f))
    return fail(NVB_ERR_INVALID_ARGUMENT, "colour integrator parameter out of range");
  m->cp = *p;
  return NVB_OK;
}
int32_t nvb_mapper_get_color_params(const NvbMapper* m, NvbColorParams* p) {
  if (!m || !p) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  *p = m->cp;
  return NVB_OK;
}

namespace {
// binary32 -> binary16 -> binary32, round to nearest even (__float2half followed by the implicit __half -> float)
float roundThroughHalf(float f) {
  uint32_t x;
  memcpy(&x, &f, 4);
  const uint32_t sign = x & 0x80000000u, ax = x & 0x7fffffffu;
  uint32_t out;
  if (ax >= 0x7f800000u) {
    out = ax;
  } else if (ax >= 0x477ff000u) {
    out = 0x7f800000u;
  } else if (ax < 0x38800000u) {
    const float r = std::nearbyint(std::fabs(f) * 16777216.0f) * (1.0f / 16777216.0f);
    memcpy(&out, &r, 4);
  } else {
    out = (ax + 0x0fffu + ((ax >> 13) & 1u)) & 0xffffe000u;
  }
  out |= sign;
  float r;
  memcpy(&r, &out, 4);
  return r;
}

int ensureColorLayer(NvbMapper* m) {
  NVB_CUDA(followProjectiveSlab(m, &m->color, kColorBlockBytes));
  NVB_CUDA(m->color_work.grow(m, m->tsdf.capacity(), m->tsdf.capacity()));
  return NVB_OK;
}

// The tracer's half of ColorArgs + the launch. synth must hold (height / f) * (width / f) floats.
int fillTracerArgs(NvbMapper* m, ColorArgs* a, const float* T_L_C_cm, const NvbCamera* cam, float trunc_m, int f) {
  if (f <= 0 || cam->width % f != 0 || cam->height % f != 0)
    return fail(NVB_ERR_INVALID_ARGUMENT, "the ray subsampling factor must divide the image size");  // CHECK_EQ, sphere_tracer.cu:432-433
  a->tsdf = m->tsdf.dev();
  a->T_L_C = rigidFromColMajor(T_L_C_cm);
  a->T_C_L = invertRigid(a->T_L_C);
  a->cam = *cam;
  a->block_size = m->block_size;
  a->voxel_size = m->block_size * (1.0f / kVps);
  a->half_voxel_size = m->block_size * (0.5f / kVps);
  a->voxel_size_inv = (float)(1.0 / (double)(m->block_size * (1.0f / kVps)));  // indexing_impl.h:41
  a->trunc_m = trunc_m;
  a->subsample = f;
  a->drows = cam->height / f, a->dcols = cam->width / f;  // getSubsampledImageSize (sphere_tracer.cu:335-339)
  a->max_steps = m->cp.sphere_tracer_maximum_steps;
  a->max_ray_len = m->cp.sphere_tracer_maximum_ray_length_m;
  a->eps_m = m->cp.sphere_tracer_surface_distance_epsilon_vox * m->voxel_size;
  const size_t need = (size_t)a->drows * a->dcols;
  NVB_CUDA(m->color_synth.grow(m, need, need));
  a->synth = m->color_synth.get();
  return NVB_OK;
}

}  // namespace

int32_t nvb_sphere_tracer_render_depth(NvbMapper* m, const float* T_L_C, const NvbCamera* cam, float truncation_distance_m,
                                       int32_t ray_subsampling_factor, float* out_depth_host) {
  if (!m || !T_L_C || !cam || !out_depth_host) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  if (m->projective_layer_type == NVB_PROJECTIVE_OCCUPANCY)
    return fail(NVB_ERR_INVALID_ARGUMENT, "the sphere tracer needs a TSDF layer");
  NVB_CUDA(cudaSetDevice(m->device));
  ColorArgs a{};
  int rc = fillTracerArgs(m, &a, T_L_C, cam, truncation_distance_m, ray_subsampling_factor);
  if (rc) return rc;
  launchSphereTrace(a, m->stream);
  m->launches++;
  NVB_CUDA(cudaMemcpyAsync(out_depth_host, a.synth, (size_t)a.drows * a.dcols * sizeof(float), cudaMemcpyDeviceToHost, m->stream));
  NVB_CUDA(cudaStreamSynchronize(m->stream));
  return checkDeviceError(m);
}

int32_t nvb_mapper_integrate_color(NvbMapper* m, const uint8_t* color, const uint8_t* mask, int32_t mask_mode, int32_t memory,
                                   int32_t rows, int32_t cols, const float* T_L_C, const NvbCamera* cam,
                                   int32_t* updated_xyz_host, int32_t cap, int32_t* out_count) {
  if (!m || !color || !T_L_C || !cam) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  if (rows <= 0 || cols <= 0) return fail(NVB_ERR_INVALID_ARGUMENT, "image must have positive size");
  if (!(cam->fu != 0.0f) || !(cam->fv != 0.0f)) return fail(NVB_ERR_INVALID_ARGUMENT, "camera focal length is zero");
  int rc;
  if ((rc = checkMemoryKind(memory))) return rc;
  if (out_count) *out_count = 0;
  // "Color is only integrated for Tsdf layers (not for occupancy)" (mapper_impl.h:118-119)
  if (m->projective_layer_type == NVB_PROJECTIVE_OCCUPANCY) return NVB_OK;
  NVB_CUDA(cudaSetDevice(m->device));
  if ((rc = ensureColorLayer(m))) return rc;
  const float trunc_m = m->cp.truncation_distance_vox * m->voxel_size;
  ColorArgs a{};
  if ((rc = fillTracerArgs(m, &a, T_L_C, cam, trunc_m, m->cp.sphere_tracing_ray_subsampling_factor))) return rc;
  a.color = m->color.dev();
  // Camera::getViewAABB(T_L_C, 1e-6, max_integration_distance + truncation) + the integrator's own workspace bounds
  // (view_calculator_impl.h:47-58)
  {
    const float max_distance = m->cp.max_integration_distance_m + trunc_m;
    const float w = (float)cam->width, h = (float)cam->height;
    const float ux[4] = {0.0f, w, w, 0.0f}, vy[4] = {0.0f, 0.0f, h, h};
    Vec3 ray[4];
    for (int k = 0; k < 4; k++) {
      float nx = (ux[k] - cam->cu) / cam->fu, ny = (vy[k] - cam->cv) / cam->fv;
      if (cam->has_distortion) removeDistortion(*cam, nx, ny);
      ray[k] = Vec3{nx, ny, 1.0f};
    }
    const int order[4] = {2, 1, 0, 3};
    float lo[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, hi[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
    for (int k = 0; k < 8; k++) {
      const float d = (k < 4) ? 1e-6f : max_distance;
      const Vec3 r = ray[order[k & 3]];
      const Vec3 c = transformPoint(a.T_L_C, Vec3{d * r.x, d * r.y, d * r.z});
      const float cl[3] = {c.x, c.y, c.z};
      for (int i = 0; i < 3; i++) lo[i] = std::min(lo[i], cl[i]), hi[i] = std::max(hi[i], cl[i]);
    }
    if (m->cp.workspace_bounds_type == NVB_WS_HEIGHT_BOUNDS) {
      lo[2] = std::max(lo[2], m->cp.workspace_min[2]);
      hi[2] = std::min(hi[2], m->cp.workspace_max[2]);
    } else if (m->cp.workspace_bounds_type == NVB_WS_BOUNDING_BOX) {
      for (int i = 0; i < 3; i++) lo[i] = std::max(m->cp.workspace_min[i], lo[i]), hi[i] = std::min(hi[i], m->cp.workspace_max[i]);
    }
    if (lo[0] > hi[0] || lo[1] > hi[1] || lo[2] > hi[2]) return NVB_OK;  // empty workspace intersection: nothing in view
    a.aabb_lo = blockIndexFromPosition(m->block_size, Vec3{lo[0], lo[1], lo[2]});
    a.aabb_hi = blockIndexFromPosition(m->block_size, Vec3{hi[0], hi[1], hi[2]});
    // Camera::getNormalizedViewport(getViewportMargin(height)) (src/sensors/camera.cpp:85-96, view_calculator_impl.h:81-83)
    const float margin = (float)cam->height / 20.0f;
    float x0 = (-margin - cam->cu) / cam->fu, y0 = (-margin - cam->cv) / cam->fv;
    float x1 = (((float)cam->width + margin) - cam->cu) / cam->fu, y1 = (((float)cam->height + margin) - cam->cv) / cam->fv;
    if (cam->has_distortion) removeDistortion(*cam, x0, y0), removeDistortion(*cam, x1, y1);
    a.vmin_x = x0, a.vmin_y = y0, a.vmax_x = x1, a.vmax_y = y1;
  }
  a.max_integration_distance_m = m->cp.max_integration_distance_m;
  a.max_weight = m->cp.max_weight;
  a.measurement_weight = m->cp.measurement_weight;
  {  // blendTwoArrays (projective_appearance_integrator.cu:287-306)
    float w_old = 1.0f - m->cp.measurement_weight, w_new = m->cp.measurement_weight;
    const float total = w_old + w_new;
    w_old /= total, w_new /= total;
    a.w_old_h = roundThroughHalf(w_old), a.w_new_h = roundThroughHalf(w_new);
  }
  a.work = m->color_work.get();
  a.work_count = &m->counters.get()->color_work_count;
  a.error = m->error_dev;
  a.rows = rows, a.cols = cols;
  a.depth_subsample = rows / a.drows;  // projective_integrator_impl.cuh:320
  if (a.depth_subsample <= 0) return fail(NVB_ERR_INVALID_ARGUMENT, "the colour image is smaller than the synthetic depth image");
  a.mask_mode = mask_mode;
  CallerBuffers bufs(memory, m->stream, m->stage_pool);
  NVB_CUDA(bufs.in(color, (size_t)rows * cols * 3, &a.color_image));
  NVB_CUDA(bufs.in(mask, (size_t)rows * cols, &a.mask));
  NVB_CUDA(cudaMemsetAsync(a.work_count, 0, sizeof(int), m->stream));
  launchColorSelect(a, m->num_sms, m->stream);
  launchSphereTrace(a, m->stream);
  launchColorIntegrate(a, m->num_sms, m->stream);
  m->launches += 3;
  // Device-resident frames with no output requested stay asynchronous (read the list later with
  // nvb_mapper_last_color_blocks); host-memory frames and requested outputs return with the frame integrated.
  if (memory == NVB_MEM_DEVICE && !updated_xyz_host && !out_count) return NVB_OK;
  NVB_CUDA(cudaStreamSynchronize(m->stream));
  int rc2 = nvb_mapper_last_color_blocks(m, updated_xyz_host, cap, out_count);
  if (rc2) return rc2;
  return checkDeviceError(m);
}

int32_t nvb_mapper_last_color_blocks(NvbMapper* m, int32_t* out_xyz_host, int32_t cap, int32_t* out_count) {
  if (!m) return fail(NVB_ERR_INVALID_ARGUMENT, "null mapper");
  if (out_count) *out_count = 0;
  if (!m->color.exists() || !m->color_work.get()) return NVB_OK;
  NVB_CUDA(cudaSetDevice(m->device));
  return readBlockList(m, &m->counters.get()->color_work_count, m->color_work.get(), Record::kXyzFirst, false, out_xyz_host,
                       cap, out_count);
}

int32_t nvb_mapper_integrate_depth(NvbMapper* m, const float* depth, const uint8_t* mask, int32_t mask_mode,
                                   int32_t memory, int32_t rows, int32_t cols, const float* T_L_C,
                                   const NvbCamera* cam, int32_t* updated_xyz_host, int32_t cap, int32_t* out_count) {
  int rc = nvb_mapper_integrate_depth_async(m, depth, mask, mask_mode, memory, rows, cols, T_L_C, cam);
  if (rc) return rc;
  if ((rc = m->frame_list.read(m, updated_xyz_host, cap, out_count))) return rc;
  return checkPrefetchedError(m);
}

int32_t nvb_mapper_update_esdf_async(NvbMapper* m, int32_t update_full_layer) {
  if (!m) return fail(NVB_ERR_INVALID_ARGUMENT, "null mapper");
  NVB_CUDA(cudaSetDevice(m->device));
  const int rc = startTrackerUpdate(m, kEsdfBlocks, update_full_layer);
  return rc ? rc : enqueueEsdf(m, nullptr, 0, true);
}

int32_t nvb_mapper_update_esdf(NvbMapper* m, int32_t update_full_layer) {
  int rc = nvb_mapper_update_esdf_async(m, update_full_layer);
  if (rc) return rc;
  return nvb_mapper_synchronize(m);
}

int32_t nvb_esdf_integrate_blocks(NvbMapper* m, const int32_t* blocks_xyz_host, int32_t num_blocks) {
  if (!m) return fail(NVB_ERR_INVALID_ARGUMENT, "null mapper");
  // The list is a set for every caller of the reference (Mapper::getBlocksToUpdate); make it one.
  std::vector<std::array<int, 3>> set;
  int rc = takeBlockList(BlockList::kInsertSet, &blocks_xyz_host, &num_blocks, &set);
  if (rc) return rc;
  if (num_blocks == 0) return NVB_OK;  // early return, esdf_integrator.cu:226-228
  NVB_CUDA(cudaSetDevice(m->device));
  const int n = num_blocks;
  NVB_CUDA(m->xyz_upload.grow(m, 3 * (size_t)n, 6 * (size_t)n));
  // Stream-ordered upload: a blocking cudaMemcpy from pageable memory may return before the DMA has landed,
  // and the mapper's stream is non-blocking (not ordered against the legacy default stream).
  NVB_CUDA(cudaMemcpyAsync(m->xyz_upload.get(), blocks_xyz_host, (size_t)n * 3 * sizeof(int), cudaMemcpyHostToDevice, m->stream));
  NVB_CUDA(cudaStreamSynchronize(m->stream));  // the set is pageable and about to go out of scope
  if ((rc = enqueueEsdf(m, m->xyz_upload.get(), n, false))) return rc;
  if ((rc = nvb_mapper_synchronize(m))) return rc;
  return m->bounds.tightenEsdfBound(m->esdf, m->tsdf.capacity());
}

void nvb_default_esdf_slice_params(NvbEsdfSliceParams* p) {
  if (!p) return;
  // integrators/esdf_integrator_params.h:33-43
  p->slice_min_height_m = 0.0f;
  p->slice_max_height_m = 1.0f;
  p->slice_height_m = 1.0f;
  p->slice_height_above_plane_m = 0.0f;
  p->slice_height_thickness_m = 0.1f;
}
int32_t nvb_mapper_set_esdf_slice_params(NvbMapper* m, const NvbEsdfSliceParams* p) {
  if (!m || !p) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  if (!(p->slice_max_height_m >= p->slice_min_height_m)) return fail(NVB_ERR_INVALID_ARGUMENT, "slice_max_height below slice_min_height");
  // CHECK_GE(slice_height_above_plane_m, 0) / CHECK_GT(slice_height_thickness_m, 0) (esdf_integrator.cu:928-929)
  if (!(p->slice_height_above_plane_m >= 0.0f) || !(p->slice_height_thickness_m > 0.0f))
    return fail(NVB_ERR_INVALID_ARGUMENT, "planar slice: height above plane must be >= 0 and thickness > 0");
  m->sp = *p;
  return NVB_OK;
}
int32_t nvb_mapper_get_esdf_slice_params(const NvbMapper* m, NvbEsdfSliceParams* p) {
  if (!m || !p) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  *p = m->sp;
  return NVB_OK;
}

static int32_t updateEsdfSliceImpl(NvbMapper* m, const float* plane, int32_t update_full_layer);
int32_t nvb_mapper_update_esdf_slice(NvbMapper* m, int32_t update_full_layer) { return updateEsdfSliceImpl(m, nullptr, update_full_layer); }
int32_t nvb_mapper_update_esdf_slice_planar(NvbMapper* m, const float plane[4], int32_t update_full_layer) {
  if (!plane) return fail(NVB_ERR_INVALID_ARGUMENT, "null plane");
  return updateEsdfSliceImpl(m, plane, update_full_layer);
}
static int32_t updateEsdfSliceImpl(NvbMapper* m, const float* plane, int32_t update_full_layer) {
  if (!m) return fail(NVB_ERR_INVALID_ARGUMENT, "null mapper");
  NVB_CUDA(cudaSetDevice(m->device));
  int rc;
  if ((rc = startTrackerUpdate(m, kEsdfBlocks, update_full_layer))) return rc;
  if ((rc = enqueueEsdf(m, nullptr, 0, true, true, plane))) return rc;
  return nvb_mapper_synchronize(m);
}

static int32_t integrateSliceBlocksImpl(NvbMapper* m, const float* plane, const int32_t* blocks_xyz_host, int32_t num_blocks);
int32_t nvb_esdf_integrate_slice_blocks(NvbMapper* m, const int32_t* blocks_xyz_host, int32_t num_blocks) {
  return integrateSliceBlocksImpl(m, nullptr, blocks_xyz_host, num_blocks);
}
int32_t nvb_esdf_integrate_slice_planar_blocks(NvbMapper* m, const float plane[4], const int32_t* blocks_xyz_host,
                                               int32_t num_blocks) {
  if (!plane) return fail(NVB_ERR_INVALID_ARGUMENT, "null plane");
  return integrateSliceBlocksImpl(m, plane, blocks_xyz_host, num_blocks);
}
static int32_t integrateSliceBlocksImpl(NvbMapper* m, const float* plane, const int32_t* blocks_xyz_host, int32_t num_blocks) {
  if (!m) return fail(NVB_ERR_INVALID_ARGUMENT, "null mapper");
  int rc = takeBlockList(BlockList::kInsert, &blocks_xyz_host, &num_blocks);  // the column set dedupes on the device
  if (rc) return rc;
  if (num_blocks == 0) return NVB_OK;  // early return (:289-291)
  NVB_CUDA(cudaSetDevice(m->device));
  NVB_CUDA(m->xyz_upload.grow(m, 3 * (size_t)num_blocks, 6 * (size_t)num_blocks));
  NVB_CUDA(cudaMemcpyAsync(m->xyz_upload.get(), blocks_xyz_host, (size_t)num_blocks * 3 * sizeof(int), cudaMemcpyHostToDevice, m->stream));
  NVB_CUDA(cudaStreamSynchronize(m->stream));
  if ((rc = enqueueEsdf(m, m->xyz_upload.get(), num_blocks, false, true, plane))) return rc;
  if ((rc = nvb_mapper_synchronize(m))) return rc;
  return m->bounds.tightenEsdfBound(m->esdf, m->tsdf.capacity());
}

void nvb_default_ground_plane_params(NvbGroundPlaneParams* p) {
  if (!p) return;
  // ground_plane_estimator_params.h, ransac_plane_fitter_params.h, tsdf_zero_crossings_extractor.h
  p->ground_points_candidates_min_z_m = -0.1f;
  p->ground_points_candidates_max_z_m = 0.15f;
  p->ransac_distance_threshold_m = 0.2f;
  p->num_ransac_iterations = 1000;
  p->min_tsdf_weight = 0.1f;
  p->max_crossings = 360000;
}
int32_t nvb_mapper_set_ground_plane_params(NvbMapper* m, const NvbGroundPlaneParams* p) {
  if (!m || !p) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  if (p->num_ransac_iterations < 1) return fail(NVB_ERR_INVALID_ARGUMENT, "num_ransac_iterations must be >= 1");
  m->gp = *p;
  return NVB_OK;
}
int32_t nvb_mapper_get_ground_plane_params(const NvbMapper* m, NvbGroundPlaneParams* p) {
  if (!m || !p) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  *p = m->gp;
  return NVB_OK;
}
}  // extern "C"

namespace {
int SlotOrder::sort(NvbMapper* m, const DevLayer& layer, int hw, const int** sorted) {
  const size_t n = hw, temp_bytes = groundSortTempBytes(hw);
  NVB_CUDA(keys_.growDoubling(m, 2 * n));
  NVB_CUDA(slots_.growDoubling(m, 2 * n));
  NVB_CUDA(temp_.grow(m, std::max<size_t>(temp_bytes, 1), std::max<size_t>(temp_bytes, 1)));
  NVB_CUDA(launchGroundSortBlocks(layer, hw, keys_.get(), slots_.get(), temp_.get(), temp_bytes, m->stream));
  *sorted = slots_.get() + hw;
  return NVB_OK;
}

int GroundPlaneEstimator::compute(NvbMapper* m, float plane[4], int32_t* found) {
  *found = 0;
  reset();
  // an occupancy mapper's TsdfLayer is empty: no blocks, no plane
  if (m->projective_layer_type == NVB_PROJECTIVE_OCCUPANCY) return NVB_OK;
  NVB_CUDA(cudaSetDevice(m->device));
  // The TSDF layer is written on `stream` only; the ESDF stream does not touch it.
  int hw = 0;
  NVB_CUDA(m->tsdf.fillLevel(&hw, m->stream));
  if (hw == 0) return NVB_OK;  // "tsdf_layer.numBlocks() == 0"
  NVB_CUDA(counts_.growDoubling(m, hw));
  NVB_CUDA(totals_.grow(m, 2, 2));
  // The slots below the high-water mark in (x, y, z) block-index order; free slots sort last and count nothing (a layer
  // whose slots are all free gives no crossings, hence no plane, like an empty one).
  GroundExtractArgs a{};
  int rc;
  if ((rc = order_.sort(m, m->tsdf.dev(), hw, &a.slots))) return rc;
  m->launches += 2;
  a.tsdf = m->tsdf.dev();
  a.num_blocks = hw;
  a.counts = counts_.get(), a.totals = totals_.get();
  a.block_size = m->block_size, a.voxel_size = m->voxel_size;
  a.min_tsdf_weight = m->gp.min_tsdf_weight;
  a.min_z = m->gp.ground_points_candidates_min_z_m, a.max_z = m->gp.ground_points_candidates_max_z_m;
  launchGroundCount(a, m->stream);
  m->launches += 2;
  int totals[2];
  NVB_CUDA(cudaMemcpyAsync(totals, totals_.get(), sizeof(totals), cudaMemcpyDeviceToHost, m->stream));
  NVB_CUDA(cudaStreamSynchronize(m->stream));
  // "Maximum number of crossings reached." (tsdf_zero_crossings_extractor.cu:126-131)
  if (totals[0] >= m->gp.max_crossings) return checkDeviceError(m);
  NVB_CUDA(crossings_.growDoubling(m, std::max(totals[0], 1)));
  NVB_CUDA(candidates_.growDoubling(m, std::max(totals[1], 1)));
  a.crossings = crossings_.get(), a.candidates = candidates_.get();
  launchGroundEmit(a, m->stream);
  m->launches++;
  valid_ = true;
  num_crossings_ = totals[0], num_candidates_ = totals[1];
  int f = 0;
  float pl[4];
  if ((rc = ransacFit(m, candidates_.get(), totals[1], m->gp.num_ransac_iterations, m->gp.ransac_distance_threshold_m, pl, &f))) {
    reset();
    return rc;
  }
  if (!f) {
    reset();
    return checkDeviceError(m);
  }
  found_ = true;
  std::memcpy(plane_, pl, sizeof(pl));
  if (plane) std::memcpy(plane, pl, sizeof(pl));
  *found = 1;
  return checkDeviceError(m);
}

int GroundPlaneEstimator::points(NvbMapper* m, int32_t which, float* xyz, int32_t cap, int32_t* n, int32_t* valid) const {
  *valid = valid_ ? 1 : 0;
  *n = 0;
  if (!valid_) return NVB_OK;
  *n = which == NVB_GROUND_POINTS_CROSSINGS ? num_crossings_ : num_candidates_;
  const int k = std::min(*n, std::max(cap, 0));
  if (!xyz || k == 0) return NVB_OK;
  NVB_CUDA(cudaSetDevice(m->device));
  if (which == NVB_GROUND_POINTS_CROSSINGS) {
    NVB_CUDA(cudaMemcpyAsync(xyz, crossings_.get(), (size_t)k * sizeof(float3), cudaMemcpyDeviceToHost, m->stream));
    NVB_CUDA(cudaStreamSynchronize(m->stream));
  } else {
    std::vector<float4> c((size_t)k);
    NVB_CUDA(cudaMemcpyAsync(c.data(), candidates_.get(), (size_t)k * sizeof(float4), cudaMemcpyDeviceToHost, m->stream));
    NVB_CUDA(cudaStreamSynchronize(m->stream));
    for (int i = 0; i < k; i++) xyz[3 * i] = c[i].x, xyz[3 * i + 1] = c[i].y, xyz[3 * i + 2] = c[i].z;
  }
  return NVB_OK;
}

int GroundPlaneEstimator::fitPoints(NvbMapper* m, const float* xyz, int32_t memory, int n, int iterations, float threshold,
                                    float plane[4], int32_t* found) {
  NVB_CUDA(cudaSetDevice(m->device));
  const size_t points_n = n;
  NVB_CUDA(fit_points_.growDoubling(m, points_n));
  CallerBuffers bufs(memory, m->stream, m->stage_pool);
  const float* src;
  NVB_CUDA(bufs.in(xyz, points_n * 3 * sizeof(float), &src));
  launchPackPoints(src, n, fit_points_.get(), m->stream);
  m->launches++;
  int rc, f = 0;
  if ((rc = ransacFit(m, fit_points_.get(), n, iterations, threshold, plane, &f))) return rc;
  *found = f;
  return checkDeviceError(m);
}

// RansacPlaneFitter::fit on n points already on the device (float4); the generator states of new iterations are made
// once and kept.
int GroundPlaneEstimator::ransacFit(NvbMapper* m, const float4* pts, int n, int iterations, float threshold, float plane[4],
                                    int* found) {
  *found = 0;
  if (n < 3) return NVB_OK;  // "We need at least three points to form a plane"
  const size_t have = states_.size() / ransacStateBytes();
  if ((size_t)iterations > have) {
    const size_t bytes = (size_t)iterations * ransacStateBytes();
    NVB_CUDA(states_.grow(m, bytes, bytes, kNoFill, kKeepContents));
    launchRansacInit(states_.get(), (int)have, iterations, m->stream);
    m->launches++;
    NVB_CUDA(cudaStreamSynchronize(m->stream));
  }
  NVB_CUDA(costs_.growDoubling(m, iterations));
  NVB_CUDA(planes_.growDoubling(m, iterations));
  NVB_CUDA(result_.grow(m, 5, 5));
  launchRansacFit(pts, n, iterations, threshold, states_.get(), costs_.get(), planes_.get(), result_.get(), m->stream);
  m->launches += 2;
  float out[5];
  NVB_CUDA(cudaMemcpyAsync(out, result_.get(), sizeof(out), cudaMemcpyDeviceToHost, m->stream));
  NVB_CUDA(cudaStreamSynchronize(m->stream));
  int f = 0;
  std::memcpy(&f, &out[4], sizeof(int));
  if (f) {
    std::memcpy(plane, out, 4 * sizeof(float));
    *found = 1;
  }
  return NVB_OK;
}
}  // namespace

extern "C" {

int32_t nvb_mapper_compute_ground_plane(NvbMapper* m, float plane[4], int32_t* found) {
  if (!m || !found) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  return m->ground.compute(m, plane, found);
}

int32_t nvb_mapper_ground_plane(NvbMapper* m, float plane[4], int32_t* found) {
  if (!m || !found) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  m->ground.lastPlane(plane, found);
  return NVB_OK;
}

int32_t nvb_mapper_ground_plane_points(NvbMapper* m, int32_t which, float* xyz, int32_t cap, int32_t* n, int32_t* valid) {
  if (!m || !n || !valid) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  if (which != NVB_GROUND_POINTS_CROSSINGS && which != NVB_GROUND_POINTS_CANDIDATES)
    return fail(NVB_ERR_INVALID_ARGUMENT, "which must be NVB_GROUND_POINTS_CROSSINGS or NVB_GROUND_POINTS_CANDIDATES");
  return m->ground.points(m, which, xyz, cap, n, valid);
}

int32_t nvb_ransac_fit_plane(NvbMapper* m, const float* points, int32_t memory, int32_t n, int32_t num_ransac_iterations,
                             float ransac_distance_threshold_m, float plane[4], int32_t* found) {
  if (!m || !plane || !found) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  if (n < 0 || (n > 0 && !points)) return fail(NVB_ERR_INVALID_ARGUMENT, "bad point list");
  if (int rc = checkMemoryKind(memory)) return rc;
  if (num_ransac_iterations < 1) return fail(NVB_ERR_INVALID_ARGUMENT, "num_ransac_iterations must be >= 1");
  *found = 0;
  if (n < 3) return NVB_OK;
  return m->ground.fitPoints(m, points, memory, n, num_ransac_iterations, ransac_distance_threshold_m, plane, found);
}

}  // extern "C"

namespace {
constexpr long long kMaxDynamicsPixels = 1ll << 28;  // 3-byte overlay and 12-byte points per pixel stay below 2^32

int DynamicsOutputs::reserve(NvbMapper* m, int pixels) {
  const size_t n = pixels;
  NVB_CUDA(depth_.grow(m, n, n));
  NVB_CUDA(mask_.grow(m, n, n));
  NVB_CUDA(clean_.grow(m, n, n));
  NVB_CUDA(overlay_.grow(m, 3 * n, 3 * n));
  NVB_CUDA(points_.grow(m, 3 * n, 3 * n));
  const size_t tiles = dynamicsNumTiles(pixels);
  NVB_CUDA(counts_.grow(m, tiles, tiles));
  NVB_CUDA(totals_.grow(m, 2, 2, 0));
  return NVB_OK;
}

int DynamicsOutputs::compute(NvbMapper* m, const float* depth, int32_t memory, DynamicsArgs a) {
  const int pixels = a.rows * a.cols;
  if (int rc = reserve(m, pixels)) return rc;
  // The freespace layer is written on `stream` only (nvb_mapper_update_freespace); the detection follows it there.
  NVB_CUDA(cudaMemcpyAsync(depth_.get(), depth, (size_t)pixels * sizeof(float),
                           memory == NVB_MEM_HOST ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice, m->stream));
  a.depth = depth_.get();
  a.mask = mask_.get(), a.overlay = overlay_.get(), a.counts = counts_.get(), a.points = points_.get();
  launchDynamicsDetect(a, totals_.get(), m->stream);
  m->launches += 3;
  rows_ = a.rows, cols_ = a.cols;
  return NVB_OK;
}

int DynamicsOutputs::reserveComponents(NvbMapper* m, CcArgs* a) {
  const size_t down = std::max(a->drows * a->dcols, 1);
  NVB_CUDA(cc_labels_.growDoubling(m, down));
  NVB_CUDA(cc_sizes_.growDoubling(m, down));
  a->labels = cc_labels_.get(), a->sizes = cc_sizes_.get();
  return NVB_OK;
}

int DynamicsOutputs::pointCount(int* n, cudaStream_t st) const {
  *n = 0;
  if (!totals_.get()) return NVB_OK;  // never computed
  NVB_CUDA(cudaMemcpyAsync(n, totals_.get(), sizeof(int), cudaMemcpyDeviceToHost, st));
  NVB_CUDA(cudaStreamSynchronize(st));
  return NVB_OK;
}

int MaskerOutputs::split(NvbMapper* m, const float* depth, const uint8_t* mask, int32_t memory, MaskerArgs a,
                         bool with_overlay) {
  const size_t n = (size_t)a.rows * a.cols, mn = (size_t)a.mrows * a.mcols;
  // Growing synchronises the mapper's streams first, so no pending split still uses the old buffers.
  NVB_CUDA(background_.grow(m, n, n));
  NVB_CUDA(foreground_.grow(m, n, n));
  if (with_overlay) NVB_CUDA(overlay_.grow(m, 3 * n, 3 * n));
  NVB_CUDA(min_depth_.grow(m, mn, mn));
  CallerBuffers bufs(memory, m->stream, m->stage_pool);  // released behind the split: the call does not synchronise
  NVB_CUDA(bufs.in(depth, n * sizeof(float), &a.depth));
  NVB_CUDA(bufs.in(mask, mn, &a.mask));
  a.min_depth = min_depth_.get();
  a.unmasked = background_.get(), a.masked = foreground_.get();
  a.overlay = with_overlay ? overlay_.get() : nullptr;
  launchSplitDepth(a, m->num_sms, m->stream);
  NVB_CUDA(cudaGetLastError());
  m->launches += 3;
  rows_ = a.rows, cols_ = a.cols, has_overlay_ = with_overlay;
  return NVB_OK;
}

int MaskerOutputs::output(int32_t which, DeviceBytes* out, int32_t* rows, int32_t* cols) const {
  const size_t n = (size_t)rows_ * cols_;
  if (which == NVB_SPLIT_BACKGROUND) *out = {background_.get(), n * sizeof(float)};
  else if (which == NVB_SPLIT_FOREGROUND) *out = {foreground_.get(), n * sizeof(float)};
  else if (which == NVB_SPLIT_OVERLAY) *out = {overlay_.get(), has_overlay_ ? 3 * n : 0};
  else return fail(NVB_ERR_INVALID_ARGUMENT, "bad split output");
  *rows = out->bytes ? rows_ : 0, *cols = out->bytes ? cols_ : 0;
  return NVB_OK;
}

// Copies one of the mapper's published outputs to the caller's `out` (in `memory`) on the mapper's stream; a host copy
// waits for it.
int copyToCaller(NvbMapper* m, void* out, DeviceBytes src, int32_t memory) {
  if (!out || src.bytes == 0 || !src.p) return NVB_OK;
  CallerBuffers bufs(memory, m->stream, m->stage_pool);
  void* dev;
  NVB_CUDA(bufs.out(out, src.bytes, &dev));
  NVB_CUDA(cudaMemcpyAsync(dev, src.p, src.bytes, cudaMemcpyDeviceToDevice, m->stream));
  NVB_CUDA(bufs.finish());
  return NVB_OK;
}
}  // namespace

extern "C" {

int32_t nvb_mapper_compute_dynamics(NvbMapper* m, const float* depth, int32_t memory, int32_t rows, int32_t cols,
                                    const float* T_L_C, const NvbCamera* cam) {
  int rc = validateFrameArgs(m, depth, memory, rows, cols, T_L_C, cam);
  if (rc) return rc;
  if (m->projective_layer_type != NVB_PROJECTIVE_TSDF_WITH_FREESPACE)
    return fail(NVB_ERR_INVALID_ARGUMENT, "the mapper has no freespace layer");
  if ((long long)rows * cols > kMaxDynamicsPixels) return fail(NVB_ERR_INVALID_ARGUMENT, "depth image too large");
  NVB_CUDA(cudaSetDevice(m->device));
  DynamicsArgs a{};
  a.rows = rows, a.cols = cols;
  a.T_L_C = rigidFromColMajor(T_L_C);
  a.cam = *cam;
  a.fs = m->freespace.dev();
  a.block_size = m->block_size;
  a.voxel_size_inv = (float)(1.0 / (double)(m->block_size * (1.0f / kVps)));  // 1.0 / blockSizeToVoxelSize(block_size)
  return m->dynamics.compute(m, depth, memory, a);
}

int32_t nvb_mapper_remove_small_components(NvbMapper* m, const uint8_t* mask_in, uint8_t* mask_out, int32_t memory,
                                           int32_t rows, int32_t cols, int32_t threshold) {
  if (!m || !mask_in || !mask_out) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  if (rows <= 0 || cols <= 0) return fail(NVB_ERR_INVALID_ARGUMENT, "mask must have positive size");
  if (int rc = checkMemoryKind(memory)) return rc;
  if ((long long)rows * cols > kMaxDynamicsPixels) return fail(NVB_ERR_INVALID_ARGUMENT, "mask too large");
  const int pixels = rows * cols;
  if (threshold <= 0) {  // "Simply copy the output if threshold is zero."
    if (memory == NVB_MEM_HOST) {
      if (mask_out != mask_in) std::memmove(mask_out, mask_in, (size_t)pixels);
      return NVB_OK;
    }
    NVB_CUDA(cudaSetDevice(m->device));
    if (mask_out != mask_in)
      NVB_CUDA(cudaMemcpyAsync(mask_out, mask_in, (size_t)pixels, cudaMemcpyDeviceToDevice, m->stream));
    return NVB_OK;
  }
  NVB_CUDA(cudaSetDevice(m->device));
  CcArgs a{};
  a.rows = rows, a.cols = cols, a.drows = rows / 2, a.dcols = cols / 2;
  a.min_size = threshold / 4;  // size_threshold / (kDownScaleFactor * kDownScaleFactor)
  if (int rc = m->dynamics.reserveComponents(m, &a)) return rc;
  CallerBuffers bufs(memory, m->stream, m->stage_pool);
  NVB_CUDA(bufs.in(mask_in, (size_t)pixels, &a.in));
  NVB_CUDA(bufs.out(mask_out, (size_t)pixels, &a.out));
  launchRemoveSmallComponents(a, m->num_sms, m->stream);
  m->launches += a.drows > 0 && a.dcols > 0 ? 4 : 1;
  NVB_CUDA(bufs.finish());
  return NVB_OK;
}

int32_t nvb_mapper_dynamic_mask(NvbMapper* m, uint8_t* out, int32_t memory, int32_t* rows, int32_t* cols) {
  if (!m || !rows || !cols) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  if (int rc = checkMemoryKind(memory)) return rc;
  *rows = m->dynamics.rows(), *cols = m->dynamics.cols();
  NVB_CUDA(cudaSetDevice(m->device));
  return copyToCaller(m, out, m->dynamics.mask(), memory);
}

int32_t nvb_mapper_dynamic_overlay(NvbMapper* m, uint8_t* out, int32_t memory, int32_t* rows, int32_t* cols) {
  if (!m || !rows || !cols) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  if (int rc = checkMemoryKind(memory)) return rc;
  *rows = m->dynamics.rows(), *cols = m->dynamics.cols();
  NVB_CUDA(cudaSetDevice(m->device));
  return copyToCaller(m, out, m->dynamics.overlay(), memory);
}

int32_t nvb_mapper_dynamic_points(NvbMapper* m, float* xyz, int32_t memory, int32_t cap, int32_t* out_count) {
  if (!m || !out_count) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  if (int rc = checkMemoryKind(memory)) return rc;
  *out_count = 0;
  NVB_CUDA(cudaSetDevice(m->device));
  int n = 0;
  if (int rc = m->dynamics.pointCount(&n, m->stream)) return rc;
  *out_count = n;
  const int k = std::min(n, std::max(cap, 0));
  return copyToCaller(m, xyz, m->dynamics.points(k), memory);
}

int32_t nvb_mapper_dynamics_device_buffers(NvbMapper* m, NvbDynamicsBuffers* out) {
  if (!m || !out) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  m->dynamics.deviceBuffers(out);
  return NVB_OK;
}

int32_t nvb_mapper_wait_for(NvbMapper* waiter, NvbMapper* producer) {
  if (!waiter || !producer) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  if (waiter == producer) return NVB_OK;  // one stream: already ordered
  NVB_CUDA(cudaSetDevice(producer->device));
  if (!producer->dyn_event) NVB_CUDA(cudaEventCreateWithFlags(&producer->dyn_event, cudaEventDisableTiming));
  NVB_CUDA(cudaEventRecord(producer->dyn_event, producer->stream));
  NVB_CUDA(cudaSetDevice(waiter->device));
  NVB_CUDA(cudaStreamWaitEvent(waiter->stream, producer->dyn_event, 0));
  return NVB_OK;
}

void nvb_default_image_masker_params(NvbImageMaskerParams* p) {
  if (!p) return;
  p->occlusion_threshold_m = 0.25f;
  p->depth_masked_image_invalid_pixel = -1.0f;
  p->depth_unmasked_image_invalid_pixel = -1.0f;
}

int32_t nvb_mapper_split_depth_image(NvbMapper* m, const float* depth, int32_t depth_rows, int32_t depth_cols,
                                     const uint8_t* mask, int32_t mask_rows, int32_t mask_cols, int32_t memory,
                                     const float* T_CM_CD, const NvbCamera* depth_cam, const NvbCamera* mask_cam,
                                     const NvbImageMaskerParams* params, int32_t with_overlay) {
  if (!m || !depth || !mask || !T_CM_CD || !depth_cam || !mask_cam || !params) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  if (int rc = checkMemoryKind(memory)) return rc;
  if (depth_rows <= 0 || depth_cols <= 0 || mask_rows <= 0 || mask_cols <= 0)
    return fail(NVB_ERR_INVALID_ARGUMENT, "images must have positive size");
  if (depth_rows != depth_cam->height || depth_cols != depth_cam->width)
    return fail(NVB_ERR_INVALID_ARGUMENT, "depth image size does not match the depth camera");
  if (mask_rows != mask_cam->height || mask_cols != mask_cam->width)
    return fail(NVB_ERR_INVALID_ARGUMENT, "mask size does not match the mask camera");
  if ((long long)depth_rows * depth_cols > kMaxDynamicsPixels || (long long)mask_rows * mask_cols > kMaxDynamicsPixels)
    return fail(NVB_ERR_INVALID_ARGUMENT, "image too large");
  NVB_CUDA(cudaSetDevice(m->device));
  MaskerArgs a{};
  a.rows = depth_rows, a.cols = depth_cols, a.mrows = mask_rows, a.mcols = mask_cols;
  a.T_CM_CD = rigidFromColMajor(T_CM_CD);
  a.depth_cam = *depth_cam, a.mask_cam = *mask_cam;
  a.occlusion_threshold_m = params->occlusion_threshold_m;
  a.masked_invalid = params->depth_masked_image_invalid_pixel;
  a.unmasked_invalid = params->depth_unmasked_image_invalid_pixel;
  return m->masker.split(m, depth, mask, memory, a, with_overlay != 0);
}

int32_t nvb_mapper_split_output(NvbMapper* m, int32_t which, void* out, int32_t memory, int32_t* rows, int32_t* cols) {
  if (!m || !rows || !cols) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  if (int rc = checkMemoryKind(memory)) return rc;
  DeviceBytes src;
  if (int rc = m->masker.output(which, &src, rows, cols)) return rc;
  NVB_CUDA(cudaSetDevice(m->device));
  return copyToCaller(m, out, src, memory);
}

int32_t nvb_mapper_split_device_buffers(NvbMapper* m, NvbSplitBuffers* out) {
  if (!m || !out) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  m->masker.deviceBuffers(out);
  return NVB_OK;
}

int32_t nvb_mapper_split_color_image(NvbMapper* m, const uint8_t* rgb, const uint8_t* mask, int32_t memory, int32_t rows,
                                     int32_t cols, uint8_t* unmasked_out, uint8_t* masked_out, uint8_t* overlay_out) {
  if (!m || !rgb || !mask || !unmasked_out || !masked_out) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  if (int rc = checkMemoryKind(memory)) return rc;
  if (rows <= 0 || cols <= 0) return fail(NVB_ERR_INVALID_ARGUMENT, "image must have positive size");
  if ((long long)rows * cols > kMaxDynamicsPixels) return fail(NVB_ERR_INVALID_ARGUMENT, "image too large");
  NVB_CUDA(cudaSetDevice(m->device));
  const size_t n = (size_t)rows * cols;
  ColorSplitArgs a{};
  a.pixels = (long long)n;
  CallerBuffers bufs(memory, m->stream, m->stage_pool);
  NVB_CUDA(bufs.in(rgb, 3 * n, &a.rgb));
  NVB_CUDA(bufs.in(mask, n, &a.mask));
  NVB_CUDA(bufs.out(unmasked_out, 3 * n, &a.unmasked));
  NVB_CUDA(bufs.out(masked_out, 3 * n, &a.masked));
  NVB_CUDA(bufs.out(overlay_out, 3 * n, &a.overlay));
  launchSplitColor(a, m->stream);
  NVB_CUDA(cudaGetLastError());
  m->launches++;
  NVB_CUDA(bufs.finish());
  return NVB_OK;
}

int32_t nvb_esdf_slice_aabb(NvbMapper* m, float slice_height_m, float aabb_out[6], int32_t* empty_out) {
  if (!m || !aabb_out || !empty_out) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  *empty_out = 1;
  NVB_CUDA(cudaSetDevice(m->device));
  NVB_CUDA(syncAll(m));
  const int zb = (int)std::floor(slice_height_m / m->block_size);
  int* box_dev = m->counters.get()->slice_box;
  const int init[4] = {INT32_MAX, INT32_MAX, INT32_MIN, INT32_MIN};
  NVB_CUDA(cudaMemcpyAsync(box_dev, init, sizeof(init), cudaMemcpyHostToDevice, m->stream));
  launchSliceAabb(m->esdf.dev(), zb, box_dev, m->stream);
  int box[4];
  NVB_CUDA(cudaMemcpyAsync(box, box_dev, sizeof(box), cudaMemcpyDeviceToHost, m->stream));
  NVB_CUDA(cudaStreamSynchronize(m->stream));
  m->launches++;
  if (box[0] > box[2]) return NVB_OK;  // no block at that height: empty AABB (:166-168)
  // getAABBOfBlock: [index * block_size, (index + 1) * block_size]
  const float bs = m->block_size;
  aabb_out[0] = (float)box[0] * bs, aabb_out[1] = (float)box[1] * bs, aabb_out[2] = (float)zb * bs;
  aabb_out[3] = ((float)box[2] + 1.0f) * bs, aabb_out[4] = ((float)box[3] + 1.0f) * bs, aabb_out[5] = ((float)zb + 1.0f) * bs;
  *empty_out = 0;
  return NVB_OK;
}

int32_t nvb_esdf_slice_distance_image_in_aabb(NvbMapper* m, float slice_height_m, float unobserved_value, const float aabb[6],
                                              float* image_host, int8_t* grid_host, int32_t cap_pixels, int32_t* rows_out,
                                              int32_t* cols_out) {
  if (!m || !aabb || !rows_out || !cols_out) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  *rows_out = *cols_out = 0;
  NVB_CUDA(cudaSetDevice(m->device));
  NVB_CUDA(syncAll(m));
  const float bs = m->block_size;
  const float voxel_size = bs / (float)kVps;
  const float sx = aabb[3] - aabb[0], sy = aabb[4] - aabb[1];
  if (!(sx > 0.0f) || !(sy > 0.0f)) return NVB_OK;  // aabb.isEmpty() (:175-177)
  const int cols = (int)std::ceil(sx / voxel_size), rows = (int)std::ceil(sy / voxel_size);
  *rows_out = rows, *cols_out = cols;
  const long long npix = (long long)rows * cols;
  if (npix <= 0 || (!image_host && !grid_host) || cap_pixels <= 0) return NVB_OK;
  DeviceArray<float> img_dev;
  DeviceArray<signed char> grid_dev;
  if (image_host) NVB_CUDA(img_dev.grow(m, npix, npix));
  if (grid_host) NVB_CUDA(grid_dev.grow(m, npix, npix));
  launchSliceImage(m->esdf.dev(), bs, aabb[0], aabb[1], slice_height_m, unobserved_value, rows, cols, img_dev.get(), grid_dev.get(),
                   m->stream);
  m->launches++;
  const size_t k = (size_t)std::min<long long>(npix, cap_pixels);
  if (image_host) NVB_CUDA(cudaMemcpyAsync(image_host, img_dev.get(), k * sizeof(float), cudaMemcpyDeviceToHost, m->stream));
  if (grid_host) NVB_CUDA(cudaMemcpyAsync(grid_host, grid_dev.get(), k, cudaMemcpyDeviceToHost, m->stream));
  NVB_CUDA(cudaStreamSynchronize(m->stream));
  return NVB_OK;
}

// robustFloor (nvblox map/internal/cuda/impl/layer_to_3d_grid_impl.cuh): an integer stored as a float with a rounding error
// below 1e-4 is that integer, anything else floors.
static int robustFloor(float x) {
  const int nearest = (int)std::round(x);
  return std::abs(x - (float)nearest) < 1e-4f ? nearest : (int)std::floor(x);
}

int32_t nvb_esdf_dense_grid_in_aabb(NvbMapper* m, const float aabb[6], float default_value, int32_t memory, float* out,
                                    int64_t cap, int32_t min_index_out[3], int32_t dims_out[3]) {
  if (!m || !aabb || !min_index_out || !dims_out) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  if (int rc = checkMemoryKind(memory)) return rc;
  for (int a = 0; a < 3; a++) min_index_out[a] = 0, dims_out[a] = 0;
  for (int a = 0; a < 6; a++)
    if (!std::isfinite(aabb[a])) return fail(NVB_ERR_INVALID_ARGUMENT, "non-finite AABB");
  const float inv_voxel_size = 1.0f / m->voxel_size;
  int mn[3], dims[3];
  long long cells = 1;
  for (int a = 0; a < 3; a++) {
    mn[a] = robustFloor(aabb[a] * inv_voxel_size);
    const long long d = (long long)robustFloor(aabb[3 + a] * inv_voxel_size) - mn[a] + 1;
    if (d <= 0) return NVB_OK;  // an empty box: no cells
    if (d > 65535ll * kVps) return fail(NVB_ERR_CAPACITY, "dense grid longer than 65535 blocks along an axis");
    dims[a] = (int)d, cells *= d;
  }
  if (cells > 0x7fffffffll) return fail(NVB_ERR_CAPACITY, "dense grid with more than 2^31 cells");
  for (int a = 0; a < 3; a++) min_index_out[a] = mn[a], dims_out[a] = dims[a];
  if (!out || cap < cells) return NVB_OK;  // the size only
  NVB_CUDA(cudaSetDevice(m->device));
  NVB_CUDA(syncAll(m));
  CallerBuffers bufs(memory, m->stream, m->stage_pool);
  float* out_dev;
  NVB_CUDA(bufs.out(out, (size_t)cells * sizeof(float), &out_dev));
  launchEsdfDenseGrid(m->esdf.dev(), make_int3(mn[0], mn[1], mn[2]), make_int3(dims[0], dims[1], dims[2]), m->voxel_size,
                      default_value, out_dev, m->stream);
  m->launches++;
  NVB_CUDA(bufs.finish());
  if (memory == NVB_MEM_DEVICE) NVB_CUDA(cudaStreamSynchronize(m->stream));
  return NVB_OK;
}

int32_t nvb_esdf_slice_distance_image(NvbMapper* m, float slice_height_m, float unobserved_value, float aabb_out[6],
                                      float* image_host, int8_t* grid_host, int32_t cap_pixels, int32_t* rows_out,
                                      int32_t* cols_out) {
  if (!m || !rows_out || !cols_out) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  *rows_out = *cols_out = 0;
  float box[6];
  int32_t empty = 1;
  int rc = nvb_esdf_slice_aabb(m, slice_height_m, box, &empty);
  if (rc || empty) return rc;
  if (aabb_out)
    for (int a = 0; a < 6; a++) aabb_out[a] = box[a];
  return nvb_esdf_slice_distance_image_in_aabb(m, slice_height_m, unobserved_value, box, image_host, grid_host, cap_pixels, rows_out,
                                               cols_out);
}

int32_t nvb_mapper_synchronize(NvbMapper* m) {
  if (!m) return fail(NVB_ERR_INVALID_ARGUMENT, "null mapper");
  NVB_CUDA(cudaSetDevice(m->device));
  int rc = enqueueErrorCopies(m);
  if (rc) return rc;
  NVB_CUDA(syncAll(m));
  NVB_CUDA(cudaGetLastError());
  collectStages(m);
  return checkPrefetchedError(m);
}

int32_t nvb_mapper_last_frame_block_count(NvbMapper* m, int32_t* out_count) {
  if (!m || !out_count) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  NVB_CUDA(cudaSetDevice(m->device));
  return m->frame_list.read(m, nullptr, 0, out_count);
}

int32_t nvb_mapper_last_frame_blocks(NvbMapper* m, int32_t* out_xyz_host, int32_t cap, int32_t* out_count) {
  if (!m) return fail(NVB_ERR_INVALID_ARGUMENT, "null mapper");
  NVB_CUDA(cudaSetDevice(m->device));
  return m->frame_list.read(m, out_xyz_host, cap, out_count);
}

}  // extern "C"

namespace {
int BlockUnion::merge(NvbMapper* m, const int32_t* xyz, int n, const ViewGrid& g, int32_t* out_xyz, int32_t cap,
                      int32_t* out_count) {
  int rc;
  if ((rc = m->view.reserve(m, g))) return rc;
  const int need = std::min(n, g.linear_size);
  NVB_CUDA(list_.grow(m, need, (size_t)std::min<long long>((long long)(1.5 * need) + 64, 0x7fffffff)));
  NVB_CUDA(count_.grow(m, 1, 1));
  launchMarkList(xyz, n, g, m->view.bits(), m->stream);
  m->view.compact(g, list_.get(), count_.get(), false, m->tsdf.dev(), TrackerLists{}, m->error_dev, true, m->stream);
  if (out_xyz && cap > 0) launchUnpackList(list_.get(), count_.get(), out_xyz, cap, m->stream);
  m->launches += 4;
  if (out_count) {
    NVB_CUDA(cudaMemcpyAsync(&m->host_words->union_count, count_.get(), sizeof(int), cudaMemcpyDeviceToHost, m->stream));
    NVB_CUDA(cudaStreamSynchronize(m->stream));
    *out_count = m->host_words->union_count;
  }
  return NVB_OK;
}

int BlockUnion::mergeSegments(NvbMapper* m, const int32_t* segments, int32_t num, int32_t stride, int32_t cap_entries,
                              int32_t* out_xyz, int32_t out_cap, int32_t* out_count, cudaStream_t st) {
  // 2^28 cells = 32 MiB of bits: a union AABB of e.g. 1024 x 1024 x 256 blocks (410 m x 410 m x 102 m at 5 cm voxels)
  constexpr long long kUnionCells = 1ll << 28;
  NVB_CUDA(bits_.grow(m, kUnionCells / 32, kUnionCells / 32, 0));
  NVB_CUDA(state_.grow(m, 1, 1, 0));
  launchUnionSegments(segments, num, stride, cap_entries, reinterpret_cast<int*>(state_.get()), bits_.get(), kUnionCells, out_xyz,
                      out_cap, out_count, st);
  m->launches += 5;
  return NVB_OK;
}

int BlockUnion::readError(int32_t* error) const {
  *error = 0;
  if (!state_.get()) return NVB_OK;
  NVB_CUDA(cudaDeviceSynchronize());
  UnionState s;
  NVB_CUDA(cudaMemcpy(&s, state_.get(), sizeof(s), cudaMemcpyDeviceToHost));
  *error = s.error;
  return NVB_OK;
}
}  // namespace

extern "C" {

int32_t nvb_blocks_union(NvbMapper* m, const int32_t* xyz_dev, int32_t n, const int32_t aabb_min[3],
                         const int32_t aabb_max[3], int32_t* out_xyz_dev, int32_t cap, int32_t* out_count_host) {
  if (!m || !aabb_min || !aabb_max || (n > 0 && !xyz_dev)) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  NVB_CUDA(cudaSetDevice(m->device));
  ViewGrid g{};
  g.min_index = make_int3(aabb_min[0], aabb_min[1], aabb_min[2]);
  const long long sx = (long long)aabb_max[0] - aabb_min[0] + 1, sy = (long long)aabb_max[1] - aabb_min[1] + 1,
                  sz = (long long)aabb_max[2] - aabb_min[2] + 1;
  if (n <= 0 || sx <= 0 || sy <= 0 || sz <= 0) {
    if (out_count_host) *out_count_host = 0;
    return NVB_OK;
  }
  if (sx * sy * sz > 0x7fffffffll) return fail(NVB_ERR_CAPACITY, "union AABB has more than 2^31 cells");
  g.size = make_int3((int)sx, (int)sy, (int)sz);
  g.linear_size = (int)(sx * sy * sz);
  g.num_words = (g.linear_size + 31) / 32;
  return m->block_union.merge(m, xyz_dev, n, g, out_xyz_dev, cap, out_count_host);
}

int32_t nvb_mapper_append_frame_blocks(NvbMapper* m, int32_t* segment_dev, int32_t cap_entries) {
  if (!m || !segment_dev || cap_entries <= 0) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  NVB_CUDA(cudaSetDevice(m->device));
  if (!m->frame_list.exists()) return NVB_OK;  // no frame integrated yet
  launchAppendFrame(m->frame_list.blocks(), m->frame_list.count(), segment_dev, cap_entries, m->error_dev, m->stream);
  m->launches++;
  return NVB_OK;
}

int32_t nvb_blocks_union_segments(NvbMapper* m, const int32_t* segments_dev, int32_t num_segments, int32_t segment_stride_ints,
                                  int32_t cap_entries, int32_t* out_xyz_dev, int32_t out_cap, int32_t* out_count_dev, void* stream) {
  if (!m || !segments_dev || !out_xyz_dev || !out_count_dev || num_segments <= 0 || cap_entries <= 0 ||
      segment_stride_ints < 1 + 3 * cap_entries)
    return fail(NVB_ERR_INVALID_ARGUMENT, "bad argument");
  NVB_CUDA(cudaSetDevice(m->device));
  return m->block_union.mergeSegments(m, segments_dev, num_segments, segment_stride_ints, cap_entries, out_xyz_dev, out_cap,
                                      out_count_dev, stream ? (cudaStream_t)stream : m->stream);
}

int32_t nvb_blocks_union_status(NvbMapper* m, int32_t* out_error) {
  if (!m || !out_error) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  NVB_CUDA(cudaSetDevice(m->device));
  return m->block_union.readError(out_error);
}

int32_t nvb_mapper_set_cache_last_viewpoint(NvbMapper* m, int32_t enable) {
  if (!m) return fail(NVB_ERR_INVALID_ARGUMENT, "null mapper");
  m->cache_last_viewpoint = enable ? 1 : 0;
  if (!enable) m->viewpoints.clear();
  return NVB_OK;
}
int32_t nvb_mapper_get_cache_last_viewpoint(const NvbMapper* m) { return m ? m->cache_last_viewpoint : 0; }

int32_t nvb_mapper_set_esdf_reserved_sms(NvbMapper* m, int32_t reserved_sms) {
  if (!m) return fail(NVB_ERR_INVALID_ARGUMENT, "null mapper");
  if (reserved_sms < 0 || reserved_sms > 64) return fail(NVB_ERR_INVALID_ARGUMENT, "reserved_sms must be in [0, 64]");
  return m->esdf_state.setReservedSms(m, reserved_sms);
}
int32_t nvb_mapper_get_esdf_reserved_sms(const NvbMapper* m) { return m ? m->esdf_state.reservedSms() : 0; }

int32_t nvb_mapper_set_depth_preprocessing(NvbMapper* m, int32_t enable, int32_t num_dilations) {
  if (!m) return fail(NVB_ERR_INVALID_ARGUMENT, "null mapper");
  if (num_dilations < 0 || num_dilations > kMaxDilations)
    return fail(NVB_ERR_INVALID_ARGUMENT, "depth_preprocessing_num_dilations must be in [0, 64]");
  m->do_depth_preprocessing = enable ? 1 : 0;
  m->depth_preprocessing_num_dilations = num_dilations;
  return NVB_OK;
}
int32_t nvb_mapper_get_depth_preprocessing(const NvbMapper* m, int32_t* enable, int32_t* num_dilations) {
  if (!m) return fail(NVB_ERR_INVALID_ARGUMENT, "null mapper");
  if (enable) *enable = m->do_depth_preprocessing;
  if (num_dilations) *num_dilations = m->depth_preprocessing_num_dilations;
  return NVB_OK;
}
int32_t nvb_depth_dilate_invalid(NvbMapper* m, const float* depth_dev, float* out_dev, int32_t rows, int32_t cols,
                                 int32_t num_dilations, float invalid_depth_threshold, float invalid_depth_value) {
  if (!m || !depth_dev || !out_dev) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  if (rows < 3 || cols < 3) return fail(NVB_ERR_INVALID_ARGUMENT, "rows and cols must be >= 3");
  if (depth_dev == out_dev) return fail(NVB_ERR_INVALID_ARGUMENT, "the output image must not alias the input");
  if (num_dilations < 0 || num_dilations > kMaxDilations)
    return fail(NVB_ERR_INVALID_ARGUMENT, "num_dilations must be in [0, 64]");
  NVB_CUDA(cudaSetDevice(m->device));
  launchDilateInvalid(depth_dev, out_dev, rows, cols, num_dilations, invalid_depth_threshold, invalid_depth_value, m->stream);
  NVB_CUDA(cudaGetLastError());
  return NVB_OK;
}

int32_t nvb_mapper_join_streams(NvbMapper* m) {
  if (!m) return fail(NVB_ERR_INVALID_ARGUMENT, "null mapper");
  NVB_CUDA(cudaSetDevice(m->device));
  NVB_CUDA(joinEsdf(m));
  return NVB_OK;
}

void* nvb_mapper_stream(NvbMapper* m) { return m ? (void*)m->stream : nullptr; }

// The projective layer is a TsdfLayer or an OccupancyLayer, never both (Mapper allocates the one its
// ProjectiveLayerType names, src/mapper/mapper.cpp:32-52): asking for the other one is an unknown layer.
static LayerSlab* layerOf(NvbMapper* m, int layer) {
  if (layer == NVB_LAYER_TSDF) return m->projective_layer_type != NVB_PROJECTIVE_OCCUPANCY ? &m->tsdf : nullptr;
  if (layer == NVB_LAYER_FREESPACE) return m->freespace.exists() ? &m->freespace : nullptr;
  if (layer == NVB_LAYER_COLOR) {
    // created on first use (integration or query); an occupancy mapper never has one (mapper_impl.h:118-119)
    if (!m->color.exists() && m->projective_layer_type != NVB_PROJECTIVE_OCCUPANCY && ensureColorLayer(m)) return nullptr;
    return m->color.exists() ? &m->color : nullptr;
  }
  if (layer == NVB_LAYER_OCCUPANCY) return m->projective_layer_type == NVB_PROJECTIVE_OCCUPANCY ? &m->tsdf : nullptr;
  if (layer == NVB_LAYER_ESDF) return &m->esdf;
  if (layer == NVB_LAYER_MESH) return m->mesh.exists() ? &m->mesh : nullptr;  // the headers; the geometry: nvb_mesh_get_blocks
  return nullptr;
}

int32_t nvb_layer_block_bytes(int32_t layer) {
  if (layer == NVB_LAYER_TSDF) return kTsdfBlockBytes;
  if (layer == NVB_LAYER_ESDF) return kEsdfBlockBytes;
  if (layer == NVB_LAYER_OCCUPANCY) return kOccBlockBytes;
  if (layer == NVB_LAYER_FREESPACE) return kFreespaceBlockBytes;
  if (layer == NVB_LAYER_COLOR) return kColorBlockBytes;
  return 0;
}

int32_t nvb_layer_num_blocks(NvbMapper* m, int32_t layer, int32_t* out_count) {
  if (!out_count) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  int64_t st[4];
  const int rc = nvb_layer_slab_stats(m, layer, st);
  if (rc == NVB_OK) *out_count = (int32_t)(st[1] - st[2]);  // slots handed out minus deallocated ones
  return rc;
}

int32_t nvb_layer_slab_stats(NvbMapper* m, int32_t layer, int64_t out[4]) {
  if (!m || !out) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  const LayerSlab* L = layerOf(m, layer);
  if (!L) return fail(NVB_ERR_INVALID_ARGUMENT, "unknown layer");
  NVB_CUDA(cudaSetDevice(m->device));
  NVB_CUDA(syncAll(m));
  int count = 0, nfree = 0;
  NVB_CUDA(L->fillLevel(&count));
  NVB_CUDA(cudaMemcpy(&nfree, L->dev().free_count, sizeof(int), cudaMemcpyDeviceToHost));
  out[0] = L->capacity(), out[1] = count, out[2] = nfree, out[3] = (int64_t)L->dev().hash.mask + 1;
  return NVB_OK;
}

int32_t nvb_layer_block_indices(NvbMapper* m, int32_t layer, int32_t* out_xyz_host, int32_t cap, int32_t* out_count) {
  int64_t st[4];
  const int rc = nvb_layer_slab_stats(m, layer, st);
  if (rc) return rc;
  const int hw = (int)st[1], n = (int)(st[1] - st[2]);
  if (out_count) *out_count = n;
  if (out_xyz_host && cap > 0 && n > 0) {
    const int* block_index = layerOf(m, layer)->dev().block_index;
    if (hw == n) {  // no deallocated slots below the high-water mark
      NVB_CUDA(cudaMemcpy(out_xyz_host, block_index, (size_t)std::min(n, cap) * 3 * sizeof(int), cudaMemcpyDeviceToHost));
    } else {
      std::vector<int> all((size_t)hw * 3);
      NVB_CUDA(cudaMemcpy(all.data(), block_index, all.size() * sizeof(int), cudaMemcpyDeviceToHost));
      int k = 0;
      for (int sl = 0; sl < hw && k < cap; sl++) {
        if (all[3 * sl] == kDeadSlotX) continue;
        out_xyz_host[3 * k] = all[3 * sl], out_xyz_host[3 * k + 1] = all[3 * sl + 1], out_xyz_host[3 * k + 2] = all[3 * sl + 2];
        k++;
      }
    }
  }
  return NVB_OK;
}

int32_t nvb_layer_get_blocks(NvbMapper* m, int32_t layer, const int32_t* xyz_host, int32_t n, void* out_host,
                             uint8_t* found_host) {
  if (!m || (n > 0 && !out_host)) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  if (int rc = takeBlockList(BlockList::kLookup, &xyz_host, &n)) return rc;
  const LayerSlab* L = layerOf(m, layer);
  if (!L) return fail(NVB_ERR_INVALID_ARGUMENT, "unknown layer");
  if (n == 0) return NVB_OK;
  NVB_CUDA(cudaSetDevice(m->device));
  NVB_CUDA(syncAll(m));
  std::vector<uint8_t> found_tmp(found_host ? 0 : n);  // the gather writes every block's flag
  CallerBuffers host(NVB_MEM_HOST, m->stream, m->stage_pool);
  const int* xyz_dev;
  unsigned char *out_dev, *found_dev;
  NVB_CUDA(host.in(xyz_host, (size_t)n * 3 * sizeof(int), &xyz_dev));
  NVB_CUDA(host.out(static_cast<unsigned char*>(out_host), (size_t)n * L->dev().block_bytes, &out_dev));
  NVB_CUDA(host.out(found_host ? found_host : found_tmp.data(), (size_t)n, &found_dev));
  launchGatherBlocks(L->dev(), L == &m->esdf, xyz_dev, n, out_dev, found_dev, m->stream);
  m->launches++;
  NVB_CUDA(host.finish());
  return NVB_OK;
}

int32_t nvb_layer_set_blocks(NvbMapper* m, int32_t layer, const int32_t* xyz_host, int32_t n, const void* in_host) {
  if (!m || (n > 0 && !in_host)) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  // Each index carries its own payload, so a repeat cannot be dropped; find-or-insert needs unique keys per launch.
  std::vector<std::array<int, 3>> set;
  const int32_t* unique = xyz_host;
  int32_t n_unique = n;
  if (int rc = takeBlockList(BlockList::kInsertSet, &unique, &n_unique, &set)) return rc;
  if (n_unique != n) return fail(NVB_ERR_INVALID_ARGUMENT, "repeated block index");
  LayerSlab* L = layerOf(m, layer);
  if (!L) return fail(NVB_ERR_INVALID_ARGUMENT, "unknown layer");
  if (n == 0) return NVB_OK;
  NVB_CUDA(cudaSetDevice(m->device));
  const bool projective = L == &m->tsdf, esdf = L == &m->esdf;
  const int rc = projective ? reserveProjective(m, n) : esdf ? reserveEsdf(m, n) : reserveDerived(m, L, n);
  if (rc) return rc;
  NVB_CUDA(syncAll(m));
  CallerBuffers host(NVB_MEM_HOST, m->stream, m->stage_pool);
  const int* xyz_dev;
  const unsigned char* in_dev;
  NVB_CUDA(host.in(xyz_host, (size_t)n * 3 * sizeof(int), &xyz_dev));
  NVB_CUDA(host.in(static_cast<const unsigned char*>(in_host), (size_t)n * L->dev().block_bytes, &in_dev));
  launchScatterBlocks(L->dev(), esdf, xyz_dev, n, in_dev, m->error_dev, m->stream);
  m->launches++;
  NVB_CUDA(syncAll(m));
  if (projective) {
    // a later updateEsdf must see these blocks: the ESDF consumer's next update covers every block. Only the ESDF is
    // told; the freespace and mesh consumers keep their lists.
    m->tracker[kEsdfBlocks].initialized = false;
  } else if (esdf) {
    if (int rc = m->esdf_state.blocksWritten(m)) return rc;
  }
  return checkDeviceError(m);
}

int32_t nvb_layer_block_device_ptr(NvbMapper* m, int32_t layer, const int32_t xyz[3], void** out_ptr) {
  if (!m || !xyz || !out_ptr) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  const LayerSlab* S = layerOf(m, layer);
  if (!S) return fail(NVB_ERR_INVALID_ARGUMENT, "unknown layer");
  const DevLayer* L = &S->dev();
  NVB_CUDA(cudaSetDevice(m->device));
  NVB_CUDA(syncAll(m));
  // host-side probe of the device hash (small, synchronous): copy the probe window
  *out_ptr = nullptr;
  if (!indexInRange(xyz[0], xyz[1], xyz[2])) return NVB_OK;
  const unsigned long long key = packIndex(xyz[0], xyz[1], xyz[2]);
  unsigned int p = hashKey(key) & L->hash.mask;
  for (unsigned int probes = 0; probes <= L->hash.mask; probes++) {
    unsigned long long k = 0;
    NVB_CUDA(cudaMemcpy(&k, L->hash.keys + p, sizeof(k), cudaMemcpyDeviceToHost));
    if (k == key) {
      int slot = -1;
      NVB_CUDA(cudaMemcpy(&slot, L->hash.vals + p, sizeof(int), cudaMemcpyDeviceToHost));
      if (slot >= 0) *out_ptr = L->blocks + (size_t)slot * L->block_bytes;
      return NVB_OK;
    }
    if (k == kEmptyKey) return NVB_OK;
    p = (p + 1) & L->hash.mask;
  }
  return NVB_OK;
}

// The layer a map file's table k (NvbLayer id, kMapFileLayers) is saved from, or null when the mapper does not hold it.
// Unlike layerOf, a colour layer is not created for this.
static LayerSlab* savedLayerOf(NvbMapper* m, int k) {
  if (k == NVB_LAYER_TSDF) return m->projective_layer_type != NVB_PROJECTIVE_OCCUPANCY ? &m->tsdf : nullptr;
  if (k == NVB_LAYER_OCCUPANCY) return m->projective_layer_type == NVB_PROJECTIVE_OCCUPANCY ? &m->tsdf : nullptr;
  if (k == NVB_LAYER_ESDF) return &m->esdf;
  if (k == NVB_LAYER_FREESPACE) return m->freespace.exists() ? &m->freespace : nullptr;
  if (k == NVB_LAYER_COLOR) return m->color.exists() ? &m->color : nullptr;
  return nullptr;  // the feature layer
}

int32_t nvb_mapper_save_map(NvbMapper* m, const char* path) {
  if (!m || !path) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  NVB_CUDA(cudaSetDevice(m->device));
  NVB_CUDA(syncAll(m));
  std::vector<int> xyz[kMapFileLayers], order[kMapFileLayers];
  std::vector<unsigned char> voxels[kMapFileLayers];
  MapFileLayerOut out[kMapFileLayers] = {};
  for (int k = 0; k < kMapFileLayers; k++) {
    const LayerSlab* S = savedLayerOf(m, k);
    if (!S) continue;
    // the slab below the high-water mark in one copy each, dead slots skipped, rows in (x, y, z) order
    int hw = 0;
    NVB_CUDA(S->fillLevel(&hw));
    const DevLayer* L = &S->dev();
    xyz[k].resize(3 * (size_t)hw);
    voxels[k].resize((size_t)hw * L->block_bytes);
    NVB_CUDA(cudaMemcpy(xyz[k].data(), L->block_index, xyz[k].size() * sizeof(int), cudaMemcpyDeviceToHost));
    NVB_CUDA(cudaMemcpy(voxels[k].data(), L->blocks, voxels[k].size(), cudaMemcpyDeviceToHost));
    if (S == &m->esdf) esdfBlocksToRecords(voxels[k].data(), (size_t)hw);  // the file holds EsdfVoxel records
    const int* b = xyz[k].data();
    for (int sl = 0; sl < hw; sl++)
      if (b[3 * sl] != kDeadSlotX) order[k].push_back(sl);
    std::sort(order[k].begin(), order[k].end(), [b](int i, int j) {
      return std::lexicographical_compare(b + 3 * i, b + 3 * i + 3, b + 3 * j, b + 3 * j + 3);
    });
    out[k] = {b, voxels[k].data(), order[k].data(), (int)order[k].size(), L->block_bytes};
  }
  std::string err;
  const int rc = writeMapFile(path, out, m->block_size, &err);
  return rc ? fail(rc, "saving " + std::string(path) + ": " + err) : NVB_OK;
}

// Slots [0, n) of the emptied layer L get the file's blocks in order: one copy of the voxels, one of the indices, the fill
// level and the hash.
static int uploadLoadedLayer(NvbMapper* m, LayerSlab* S, const MapFileLayerIn& in) {
  if (in.n == 0) return NVB_OK;
  const DevLayer& L = S->dev();
  if (S == &m->esdf) esdfBlocksFromRecords(in.voxels.get(), (size_t)in.n);  // the file holds EsdfVoxel records
  NVB_CUDA(cudaMemcpyAsync(L.blocks, in.voxels.get(), (size_t)in.n * L.block_bytes, cudaMemcpyHostToDevice, m->stream));
  NVB_CUDA(cudaMemcpyAsync(L.block_index, in.xyz.data(), in.xyz.size() * sizeof(int), cudaMemcpyHostToDevice, m->stream));
  NVB_CUDA(cudaMemcpyAsync(L.count, &in.n, sizeof(int), cudaMemcpyHostToDevice, m->stream));
  S->rehash(in.n, m->stream);
  m->launches++;
  return NVB_OK;
}

int32_t nvb_mapper_load_map(NvbMapper* m, const char* path, int32_t loaded_blocks[6]) {
  if (!m || !path) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  NVB_CUDA(cudaSetDevice(m->device));
  const bool occupancy = m->projective_layer_type == NVB_PROJECTIVE_OCCUPANCY;
  const int proj = occupancy ? NVB_LAYER_OCCUPANCY : NVB_LAYER_TSDF;
  bool want[kMapFileLayers] = {};
  want[proj] = want[NVB_LAYER_ESDF] = true;
  want[NVB_LAYER_COLOR] = !occupancy;
  want[NVB_LAYER_FREESPACE] = m->projective_layer_type == NVB_PROJECTIVE_TSDF_WITH_FREESPACE;
  MapFileLayerIn in[kMapFileLayers];
  std::string err;
  int rc = readMapFile(path, want, in, &err);
  if (rc) return fail(rc, "loading " + std::string(path) + ": " + err);
  // the slabs' growth, checked before the map changes (colour and freespace follow the projective slab)
  const int n_proj = in[proj].n, n_esdf = in[NVB_LAYER_ESDF].n;
  const long long need_t = std::max({n_proj, in[NVB_LAYER_COLOR].n, in[NVB_LAYER_FREESPACE].n});
  int cap_t = 0, cap_e = 0;
  if ((rc = grownCapacity(m->tsdf.capacity(), need_t, "the map", &cap_t)) ||
      (rc = grownCapacity(m->esdf.capacity(), n_esdf, "the map", &cap_e)))
    return rc;

  // Mapper::loadMap: the file's voxel size, a new cake and a fresh tracker (mapper.cpp:661-671)
  if ((rc = resetLayers(m))) return rc;
  const float voxel_size = in[NVB_LAYER_TSDF].block_size / (float)kVps;
  if (voxel_size != m->voxel_size) {
    m->voxel_size = voxel_size;
    m->block_size = voxel_size * (float)kVps;
    m->viewpoints.clear();  // the cached views are sets of blocks of the old size
  }
  if ((rc = ensureTsdfCapacity(m, need_t))) return rc;
  if ((rc = ensureEsdfCapacity(m, n_esdf))) return rc;
  if (m->freespace.exists()) NVB_CUDA(followProjectiveSlab(m, &m->freespace, kFreespaceBlockBytes));
  if (in[NVB_LAYER_COLOR].n > 0 && (rc = ensureColorLayer(m))) return rc;
  for (int k = 0; k < kMapFileLayers; k++) {
    LayerSlab* L = want[k] ? savedLayerOf(m, k) : nullptr;
    if (L && (rc = uploadLoadedLayer(m, L, in[k]))) return rc;
  }
  m->esdf_state.buildParentBoxes(m->esdf.dev(), n_esdf, m->stream);
  m->launches++;
  // the fill-level bounds from the real counts (tightenEsdfBound)
  m->bounds.reset(n_proj, std::max(0, n_esdf - n_proj), 0);
  NVB_CUDA(syncAll(m));
  if ((rc = checkDeviceError(m))) return rc;
  // a new colour mesh layer and a full mesh update (mapper.cpp:673-678)
  if (!occupancy && (rc = nvb_mapper_update_mesh(m, 1))) return rc;
  if (loaded_blocks)
    for (int k = 0; k < kMapFileLayers; k++) loaded_blocks[k] = want[k] ? in[k].n : 0;
  return NVB_OK;
}

int32_t nvb_layer_export_points(NvbMapper* m, int32_t layer, int32_t memory, float* xyzi, int64_t cap, int64_t* n) {
  if (!m || !n) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  if (layer != NVB_LAYER_TSDF && layer != NVB_LAYER_OCCUPANCY && layer != NVB_LAYER_FREESPACE && layer != NVB_LAYER_ESDF)
    return fail(NVB_ERR_INVALID_ARGUMENT, "points are exported from a TSDF, occupancy, freespace or ESDF layer");
  if (int rc = checkMemoryKind(memory)) return rc;
  const LayerSlab* L = layerOf(m, layer);
  if (!L) return fail(NVB_ERR_INVALID_ARGUMENT, "the mapper does not hold that layer");
  NVB_CUDA(cudaSetDevice(m->device));
  NVB_CUDA(syncAll(m));
  int hw = 0;
  NVB_CUDA(L->fillLevel(&hw));
  *n = 0;
  if (hw == 0) return NVB_OK;
  if ((long long)hw * kVpb > 0x7fffffffll) return fail(NVB_ERR_CAPACITY, "more than 2^31 voxels to export");
  SlotOrder order;
  DeviceArray<int> totals;
  DeviceArray<int2> counts;
  NVB_CUDA(counts.grow(m, hw, hw));
  NVB_CUDA(totals.grow(m, 2, 2));
  ExportPointsArgs a{};
  if (int rc = order.sort(m, L->dev(), hw, &a.slots)) return rc;
  a.layer = L->dev(), a.layer_id = layer, a.num_blocks = hw;
  a.counts = counts.get(), a.totals = totals.get();
  a.block_size = m->block_size, a.voxel_size = m->voxel_size;
  launchExportCount(a, m->stream);
  m->launches += 3;
  int total = 0;
  NVB_CUDA(cudaMemcpyAsync(&total, a.totals, sizeof(int), cudaMemcpyDeviceToHost, m->stream));
  NVB_CUDA(cudaStreamSynchronize(m->stream));
  *n = total;
  if (!xyzi || cap < total || total == 0) return NVB_OK;
  CallerBuffers bufs(memory, m->stream, m->stage_pool);
  NVB_CUDA(bufs.out(reinterpret_cast<float4*>(xyzi), (size_t)total * sizeof(float4), &a.out));
  launchExportEmit(a, m->stream);
  m->launches++;
  NVB_CUDA(bufs.finish());
  if (memory == NVB_MEM_DEVICE) NVB_CUDA(cudaStreamSynchronize(m->stream));
  return NVB_OK;
}

int32_t nvb_mapper_last_esdf_stats(NvbMapper* m, int64_t out[8]) {
  if (!m || !out) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  NVB_CUDA(cudaSetDevice(m->device));
  NVB_CUDA(syncAll(m));
  long long s[kNumEsdfStats];
  NVB_CUDA(m->esdf_state.readStats(s));
  std::copy(s + kStatWork, s + kStatRings + 1, out);
  return NVB_OK;
}

int32_t nvb_mapper_esdf_time_split(NvbMapper* m, int64_t out[4]) {
  if (!m || !out) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  NVB_CUDA(cudaSetDevice(m->device));
  NVB_CUDA(syncAll(m));
  long long s[kNumEsdfStats];
  NVB_CUDA(m->esdf_state.readStats(s));
  out[0] = s[kStatBarrierNs], out[1] = s[kStatAxisNs], out[2] = s[kStatSlowestCtaWorkNs], out[3] = s[kStatBarriers];
  return NVB_OK;
}

int32_t nvb_mapper_esdf_clear_blocks_read(NvbMapper* m, int64_t* out) {
  if (!m || !out) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  NVB_CUDA(cudaSetDevice(m->device));
  NVB_CUDA(syncAll(m));
  long long s[kNumEsdfStats];
  NVB_CUDA(m->esdf_state.readStats(s));
  *out = s[kStatClearBlocksRead];
  return NVB_OK;
}

int32_t nvb_mapper_esdf_split_stats(NvbMapper* m, int64_t out[2]) {
  if (!m || !out) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  NVB_CUDA(cudaSetDevice(m->device));
  NVB_CUDA(syncAll(m));
  long long s[kNumEsdfStats];
  NVB_CUDA(m->esdf_state.readStats(s));
  out[0] = s[kStatSplitCandidates], out[1] = s[kStatRestFetches];
  return NVB_OK;
}

int32_t nvb_mapper_debug_phase_max(NvbMapper* m, int64_t* out, int32_t cap) {
  if (!m || !out) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  NVB_CUDA(cudaSetDevice(m->device));
  NVB_CUDA(syncAll(m));
  NVB_CUDA(m->esdf_state.readPhaseMax(out, std::min(cap, (int32_t)kPhaseMaxEntries)));
  return NVB_OK;
}

int32_t nvb_mapper_enable_profiling(NvbMapper* m, int32_t enable) {
  if (!m) return fail(NVB_ERR_INVALID_ARGUMENT, "null mapper");
  NVB_CUDA(cudaSetDevice(m->device));
  NVB_CUDA(syncAll(m));
  collectStages(m);
  m->profiling = enable != 0;
  return NVB_OK;
}

int32_t nvb_mapper_stage_times(NvbMapper* m, double* out_ms, int64_t* out_calls, int32_t reset) {
  if (!m) return fail(NVB_ERR_INVALID_ARGUMENT, "null mapper");
  NVB_CUDA(cudaSetDevice(m->device));
  NVB_CUDA(syncAll(m));
  collectStages(m);
  for (int i = 0; i < kNumStages; i++) {
    if (out_ms) out_ms[i] = m->stage_ms[i];
    if (out_calls) out_calls[i] = m->stage_calls[i];
    if (reset) m->stage_ms[i] = 0, m->stage_calls[i] = 0;
  }
  return NVB_OK;
}

int64_t nvb_mapper_kernel_launches(const NvbMapper* m) { return m ? m->launches : 0; }

}  // extern "C"

// ---------------------------------------------------------------------------
// Mesh (nvb_mesh.cu)
// ---------------------------------------------------------------------------
namespace {

int MeshArena::create(NvbMapper* m) {
  NVB_CUDA(state_.grow(m, kArenaInts, kArenaInts, 0));
  return NVB_OK;
}

void MeshArena::fill(MeshCtx* c) const {
  c->vertices = live_.v.get(), c->normals = live_.n.get(), c->triangles = live_.t.get(), c->colors_raw = live_.c.get();
  c->colors = reinterpret_cast<uchar4*>(live_.c.get());
  c->arena_state = state_.get();
  c->counts = counts_.get(), c->offsets = offsets_.get();
}

int MeshArena::reserveList(NvbMapper* m, size_t list) {
  NVB_CUDA(counts_.growDoubling(m, list));
  NVB_CUDA(offsets_.growDoubling(m, list));
  return NVB_OK;
}

int MeshArena::fitUpdate(NvbMapper* m, MeshCtx* c) {
  // the one number the host needs: does the update fit behind the arena's fill level?
  int state[kArenaInts];
  NVB_CUDA(cudaMemcpyAsync(state, state_.get(), sizeof(state), cudaMemcpyDeviceToHost, m->stream));
  NVB_CUDA(cudaStreamSynchronize(m->stream));
  if ((long long)state[kArenaLastBase] + state[kArenaLastTotal] <= (long long)capacity()) return NVB_OK;
  if (int rc = repack(m, state[kArenaLastTotal], *c)) return rc;
  fill(c);
  launchMeshScan(*c, m->stream);  // the offsets move with the fill level
  m->launches++;
  return NVB_OK;
}

// Growth and garbage collection are the same operation: a segment is live while a header points at it.
int MeshArena::repack(NvbMapper* m, long long need, const MeshCtx& c) {
  NVB_CUDA(cudaStreamSynchronize(m->stream));
  int nslots = 0;
  NVB_CUDA(m->mesh.fillLevel(&nslots));
  DeviceArray<int> sizes, new_off;
  NVB_CUDA(sizes.grow(m, (size_t)nslots + 1, (size_t)nslots + 1));
  NVB_CUDA(new_off.grow(m, (size_t)nslots + 1, (size_t)nslots + 1));
  launchMeshCompactSizes(c, nslots, sizes.get(), m->stream);
  std::vector<int> h((size_t)nslots + 1, 0), o((size_t)nslots + 1, 0);
  NVB_CUDA(cudaMemcpyAsync(h.data(), sizes.get(), (size_t)nslots * sizeof(int), cudaMemcpyDeviceToHost, m->stream));
  NVB_CUDA(cudaStreamSynchronize(m->stream));
  long long live = 0;
  for (int i = 0; i < nslots; i++) o[i] = (int)live, live += h[i];
  // at least half of the arena is free behind the live data after a repack: with an update re-emitting ~1/5 of the live
  // vertices, that is several updates between repacks
  long long cap = std::max<long long>(capacity(), 1 << 20);
  while (cap < 2 * (live + need)) cap *= 2;
  if (cap > 0x7fffffffll) return fail(NVB_ERR_CAPACITY, "mesh arena beyond 2^31 vertices");
  // The spare arena is the one the previous repack moved out of, never larger than `cap`: when it has the right size it
  // is reused (no cudaMalloc in the steady state).
  NVB_CUDA(spare_.grow(m, cap));
  NVB_CUDA(cudaMemcpyAsync(new_off.get(), o.data(), (size_t)nslots * sizeof(int), cudaMemcpyHostToDevice, m->stream));
  if (hasGeometry())
    launchMeshCompactMove(c, nslots, new_off.get(), spare_.v.get(), spare_.n.get(), spare_.t.get(), spare_.c.get(), m->num_sms,
                          m->stream);
  const int state[kArenaInts] = {(int)live, 0, (int)live, 0};
  NVB_CUDA(cudaMemcpyAsync(state_.get(), state, sizeof(state), cudaMemcpyHostToDevice, m->stream));
  NVB_CUDA(cudaStreamSynchronize(m->stream));
  std::swap(live_, spare_);
  m->launches += 2;
  return NVB_OK;
}

int MeshArena::upload(NvbMapper* m, const int32_t* xyz, int n, const int** dev) {
  const size_t ints = 3 * (size_t)n;
  NVB_CUDA(xyz_.growDoubling(m, ints));
  NVB_CUDA(cudaMemcpyAsync(xyz_.get(), xyz, ints * sizeof(int), cudaMemcpyHostToDevice, m->stream));
  NVB_CUDA(cudaStreamSynchronize(m->stream));
  *dev = xyz_.get();
  return NVB_OK;
}

int ensureMeshLayer(NvbMapper* m) {
  NVB_CUDA(followProjectiveSlab(m, &m->mesh, kMeshHeaderBytes));
  // The arena state and the mesh consumer's tracker arrays: allocated with the layer, or by the next call when that failed
  // part-way. Once they exist, both calls return at once.
  int rc;
  if ((rc = m->mesh_arena.create(m))) return rc;
  return growTracker(m, m->tsdf.capacity());
}

MeshCtx makeMeshCtx(NvbMapper* m) {
  MeshCtx c{};
  c.tsdf = m->tsdf.dev(), c.color = m->color.dev(), c.mesh = m->mesh.dev();
  m->mesh_arena.fill(&c);
  c.block_size = m->block_size, c.voxel_size = m->voxel_size;
  c.min_weight = m->mp.min_weight, c.cutoff_distance_m = m->mp.cutoff_distance_vox * m->voxel_size;
  c.weld = m->mp.weld_vertices ? 1 : 0;
  c.error = m->error_dev;
  return c;
}

// One mesh update over a device list (explicit indices, or TSDF slots from the tracker).
int meshUpdateImpl(NvbMapper* m, const int* xyz_dev, const TrackerList& todo, int upper, bool color) {
  int rc;
  if (upper <= 0) return NVB_OK;
  if ((rc = m->mesh_arena.reserveList(m, upper))) return rc;
  MeshCtx c = makeMeshCtx(m);
  c.in_xyz = xyz_dev, c.todo = todo, c.in_count_host = upper;
  launchMeshCount(c, upper, m->num_sms, m->stream);
  m->launches += 2;
  if ((rc = m->mesh_arena.fitUpdate(m, &c))) return rc;
  launchMeshEmit(c, upper, m->num_sms, m->stream);
  m->launches += c.weld ? 2 : 1;
  if (color) {
    launchMeshColor(c, upper, m->num_sms, m->stream);
    m->launches++;
  }
  return NVB_OK;
}

}  // namespace

extern "C" {

void nvb_default_mesh_params(NvbMeshParams* p) {
  if (!p) return;
  p->min_weight = 1e-4f;          // mesh/mesh_integrator_params.h:22-24
  p->weld_vertices = 1;           // mesh/mesh_integrator_params.h:25-27
  p->cutoff_distance_vox = 5.0f;  // MeshIntegrator::cutoff_distance_vox_, mesh/mesh_integrator.h:129
}
int32_t nvb_mapper_set_mesh_params(NvbMapper* m, const NvbMeshParams* p) {
  if (!m || !p) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  m->mp = *p;
  return NVB_OK;
}
int32_t nvb_mapper_get_mesh_params(const NvbMapper* m, NvbMeshParams* p) {
  if (!m || !p) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  *p = m->mp;
  return NVB_OK;
}

int32_t nvb_mapper_update_mesh(NvbMapper* m, int32_t update_full_layer) {
  if (!m) return fail(NVB_ERR_INVALID_ARGUMENT, "null mapper");
  // "Mesh is only updated for Tsdf layers (not for occupancy)" (src/mapper/mapper.cpp:380-383)
  if (m->projective_layer_type == NVB_PROJECTIVE_OCCUPANCY) return NVB_OK;
  NVB_CUDA(cudaSetDevice(m->device));
  int rc;
  if ((rc = ensureMeshLayer(m))) return rc;
  const int upper = m->bounds.projectiveUpper(m->tsdf.capacity());
  if ((rc = startTrackerUpdate(m, kColorMeshBlocks, update_full_layer))) return rc;
  // integrateBlocksGPU + updateAppearance over the tracker's blocks, then markBlocksAsUpdated (mapper.cpp:385-395)
  const TrackerList todo = m->tracker[kColorMeshBlocks].list();
  if ((rc = meshUpdateImpl(m, nullptr, todo, upper, true))) return rc;
  NVB_CUDA(cudaMemsetAsync(todo.count, 0, sizeof(int), m->stream));
  NVB_CUDA(cudaStreamSynchronize(m->stream));
  return checkDeviceError(m);
}

int32_t nvb_mesh_integrate_blocks(NvbMapper* m, const int32_t* blocks_xyz_host, int32_t num_blocks, int32_t update_color) {
  if (!m) return fail(NVB_ERR_INVALID_ARGUMENT, "null mapper");
  if (m->projective_layer_type == NVB_PROJECTIVE_OCCUPANCY) return fail(NVB_ERR_INVALID_ARGUMENT, "the mapper has no TSDF layer");
  // a set, like the tracker's list in the reference
  std::vector<std::array<int, 3>> set;
  int rc = takeBlockList(BlockList::kInsertSet, &blocks_xyz_host, &num_blocks, &set);
  if (rc) return rc;
  NVB_CUDA(cudaSetDevice(m->device));
  if ((rc = ensureMeshLayer(m))) return rc;
  if (num_blocks == 0) return NVB_OK;  // (:73-75)
  const int* xyz_dev;
  if ((rc = m->mesh_arena.upload(m, blocks_xyz_host, num_blocks, &xyz_dev))) return rc;
  if ((rc = meshUpdateImpl(m, xyz_dev, TrackerList{}, num_blocks, update_color != 0))) return rc;
  NVB_CUDA(cudaStreamSynchronize(m->stream));
  return checkDeviceError(m);
}

int32_t nvb_mesh_update_color(NvbMapper* m, const int32_t* blocks_xyz_host, int32_t num_blocks) {
  if (!m) return fail(NVB_ERR_INVALID_ARGUMENT, "null mapper");
  std::vector<std::array<int, 3>> set;
  int rc = takeBlockList(BlockList::kInsertSet, &blocks_xyz_host, &num_blocks, &set);
  if (rc) return rc;
  NVB_CUDA(cudaSetDevice(m->device));
  if ((rc = ensureMeshLayer(m))) return rc;
  if (num_blocks == 0 || !m->mesh_arena.hasGeometry()) return NVB_OK;
  MeshCtx c = makeMeshCtx(m);
  if ((rc = m->mesh_arena.upload(m, blocks_xyz_host, num_blocks, &c.in_xyz))) return rc;
  c.in_count_host = num_blocks;
  launchMeshColor(c, num_blocks, m->num_sms, m->stream);
  m->launches++;
  NVB_CUDA(cudaStreamSynchronize(m->stream));
  return NVB_OK;
}

int32_t nvb_mesh_block_sizes(NvbMapper* m, const int32_t* blocks_xyz_host, int32_t num_blocks, int32_t* sizes_out) {
  if (!m || (num_blocks > 0 && !sizes_out)) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  if (int rc = takeBlockList(BlockList::kLookup, &blocks_xyz_host, &num_blocks)) return rc;
  if (num_blocks == 0) return NVB_OK;
  NVB_CUDA(cudaSetDevice(m->device));
  for (int i = 0; i < 3 * num_blocks; i++) sizes_out[i] = -1;
  if (!m->mesh.exists()) return NVB_OK;
  NVB_CUDA(syncAll(m));
  DeviceArray<int> dev;  // headers[4n] (int4-aligned)
  NVB_CUDA(dev.grow(m, (size_t)num_blocks * 4, (size_t)num_blocks * 4));
  CallerBuffers host(NVB_MEM_HOST, m->stream, m->stage_pool);
  const int* xyz_dev;
  NVB_CUDA(host.in(blocks_xyz_host, (size_t)num_blocks * 3 * sizeof(int), &xyz_dev));
  launchMeshHeaders(makeMeshCtx(m), xyz_dev, num_blocks, dev.get(), m->stream);
  std::vector<int> h((size_t)num_blocks * 4);
  NVB_CUDA(cudaMemcpyAsync(h.data(), dev.get(), h.size() * sizeof(int), cudaMemcpyDeviceToHost, m->stream));
  NVB_CUDA(cudaStreamSynchronize(m->stream));
  for (int i = 0; i < num_blocks; i++)
    if (h[4 * i] >= 0) sizes_out[3 * i] = h[4 * i + 1], sizes_out[3 * i + 1] = h[4 * i + 2], sizes_out[3 * i + 2] = h[4 * i + 3];
  return NVB_OK;
}

int32_t nvb_mesh_get_blocks(NvbMapper* m, const int32_t* blocks_xyz_host, int32_t num_blocks, float* vertices_out,
                            float* normals_out, int32_t* triangles_out, uint8_t* colors_out, const int64_t caps[3]) {
  if (!m || !caps) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  if (int rc = takeBlockList(BlockList::kLookup, &blocks_xyz_host, &num_blocks)) return rc;
  if (num_blocks == 0 || !m->mesh.exists()) return NVB_OK;
  NVB_CUDA(cudaSetDevice(m->device));
  NVB_CUDA(syncAll(m));
  const size_t n = (size_t)num_blocks;
  DeviceArray<int> dev;  // headers[4n] (int4-aligned)
  NVB_CUDA(dev.grow(m, n * 4, n * 4));
  CallerBuffers host(NVB_MEM_HOST, m->stream, m->stage_pool);
  const int *xyz_dev, *dst_dev;
  NVB_CUDA(host.in(blocks_xyz_host, n * 3 * sizeof(int), &xyz_dev));
  MeshCtx c = makeMeshCtx(m);
  launchMeshHeaders(c, xyz_dev, num_blocks, dev.get(), m->stream);
  std::vector<int> h(n * 4), dst(n * 3);
  NVB_CUDA(cudaMemcpyAsync(h.data(), dev.get(), h.size() * sizeof(int), cudaMemcpyDeviceToHost, m->stream));
  NVB_CUDA(cudaStreamSynchronize(m->stream));
  long long tv = 0, tt = 0, tc = 0;
  for (size_t i = 0; i < n; i++) {
    dst[3 * i] = (int)tv, dst[3 * i + 1] = (int)tt, dst[3 * i + 2] = (int)tc;
    if (h[4 * i] >= 0) tv += h[4 * i + 1], tt += h[4 * i + 2], tc += h[4 * i + 3];
  }
  if (tv > caps[0] || tt > caps[1] || tc > caps[2])
    return fail(NVB_ERR_CAPACITY, "output buffers smaller than the listed mesh blocks");
  // 3 floats per vertex and normal, one int per triangle index, 4 bytes per colour; at least one element each
  DeviceArray<float> pv, pn;
  DeviceArray<int> pt;
  DeviceArray<unsigned char> pc;
  NVB_CUDA(pv.grow(m, std::max<size_t>(1, (size_t)tv * 3), std::max<size_t>(1, (size_t)tv * 3)));
  NVB_CUDA(pn.grow(m, std::max<size_t>(1, (size_t)tv * 3), std::max<size_t>(1, (size_t)tv * 3)));
  NVB_CUDA(pt.grow(m, std::max<size_t>(1, (size_t)tt), std::max<size_t>(1, (size_t)tt)));
  NVB_CUDA(pc.grow(m, std::max<size_t>(1, (size_t)tc * 4), std::max<size_t>(1, (size_t)tc * 4)));
  NVB_CUDA(host.in(dst.data(), n * 3 * sizeof(int), &dst_dev));
  launchMeshPack(c, dev.get(), dst_dev, num_blocks, pv.get(), pn.get(), pt.get(), pc.get(), m->num_sms, m->stream);
  if (vertices_out && tv) NVB_CUDA(cudaMemcpyAsync(vertices_out, pv.get(), (size_t)tv * 12, cudaMemcpyDeviceToHost, m->stream));
  if (normals_out && tv) NVB_CUDA(cudaMemcpyAsync(normals_out, pn.get(), (size_t)tv * 12, cudaMemcpyDeviceToHost, m->stream));
  if (triangles_out && tt) NVB_CUDA(cudaMemcpyAsync(triangles_out, pt.get(), (size_t)tt * 4, cudaMemcpyDeviceToHost, m->stream));
  if (colors_out && tc) NVB_CUDA(cudaMemcpyAsync(colors_out, pc.get(), (size_t)tc * 4, cudaMemcpyDeviceToHost, m->stream));
  NVB_CUDA(cudaStreamSynchronize(m->stream));
  return NVB_OK;
}

int32_t nvb_mesh_arena_stats(NvbMapper* m, int64_t out[4]) {
  if (!m || !out) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  out[0] = (int64_t)m->mesh_arena.capacity(), out[1] = out[2] = out[3] = 0;
  if (!m->mesh.exists()) return NVB_OK;
  NVB_CUDA(cudaSetDevice(m->device));
  NVB_CUDA(syncAll(m));
  int state[kArenaInts];
  NVB_CUDA(m->mesh_arena.readState(state));
  out[1] = state[kArenaUsed], out[2] = state[kArenaLastTotal], out[3] = state[kArenaGarbage];
  return NVB_OK;
}

}  // extern "C"

// ---------------------------------------------------------------------------
// Point queries (nvb_query.cu)
// ---------------------------------------------------------------------------
namespace {

constexpr long long kMaxQueryPoints = 1ll << 40;

QueryLayer queryLayerOf(const NvbMapper* m, const DevLayer& L) {
  QueryLayer q;
  q.layer = L;
  q.block_size = m->block_size;
  q.voxel_size = m->voxel_size;
  q.voxel_size_inv = voxelSizeInv(m->block_size);
  return q;
}

// Orders a query on `qs` between the mappers' work: it runs after everything already enqueued on each mapper (its stream and
// a pending ESDF wavefront), and each mapper's later work runs after it. Device-side event hops only.
template <typename Launch>
int runOrdered(NvbMapper* const* ms, int k, cudaStream_t qs, Launch launch) {
  for (int i = 0; i < k; i++) {
    NvbMapper* m = ms[i];
    if (!m->query_event) NVB_CUDA(cudaEventCreateWithFlags(&m->query_event, cudaEventDisableTiming));
    if (m->esdf_in_flight) NVB_CUDA(cudaStreamWaitEvent(qs, m->esdf_done, 0));
    if (m->stream != qs) {
      NVB_CUDA(cudaEventRecord(m->query_event, m->stream));
      NVB_CUDA(cudaStreamWaitEvent(qs, m->query_event, 0));
    }
  }
  launch(qs);
  NVB_CUDA(cudaGetLastError());
  for (int i = 0; i < k; i++) {
    NvbMapper* m = ms[i];
    m->launches++;
    if (m->stream == qs) continue;
    NVB_CUDA(cudaEventRecord(m->query_event, qs));
    NVB_CUDA(cudaStreamWaitEvent(m->stream, m->query_event, 0));
  }
  return NVB_OK;
}

// A per-layer query (nvb_layer_query_voxels, nvb_layer_interpolate) on the mapper's stream. Host buffers are staged on the
// device and the call returns when the outputs are written back; device buffers are enqueued without synchronising.
// launch(xyz_dev, out_dev, flags_dev, stream)
template <typename Launch>
int runLayerQuery(NvbMapper* m, const float* xyz, int32_t memory, long long n, void* out, size_t out_bytes_per_point,
                  uint8_t* flags, Launch launch) {
  NVB_CUDA(cudaSetDevice(m->device));
  CallerBuffers bufs(memory, m->stream, m->stage_pool);
  const float* xyz_dev;
  void* out_dev;
  uint8_t* flags_dev;
  NVB_CUDA(bufs.in(xyz, (size_t)n * 3 * sizeof(float), &xyz_dev));
  // the outputs the kernel does not write come back unchanged
  NVB_CUDA(bufs.out(out, (size_t)n * out_bytes_per_point, &out_dev, true));
  NVB_CUDA(bufs.out(flags, (size_t)n, &flags_dev));
  const int rc = runOrdered(&m, 1, m->stream, [&](cudaStream_t st) { launch(xyz_dev, out_dev, flags_dev, st); });
  if (rc) return rc;
  NVB_CUDA(bufs.finish());
  return NVB_OK;
}

int checkLayerQueryArgs(NvbMapper* m, const float* xyz, int32_t memory, int64_t n, const void* out, const void* flags) {
  if (!m) return fail(NVB_ERR_INVALID_ARGUMENT, "null mapper");
  if (int rc = checkMemoryKind(memory)) return rc;
  if (n < 0 || n > kMaxQueryPoints) return fail(NVB_ERR_INVALID_ARGUMENT, "bad number of query points");
  if (n > 0 && (!xyz || !out || !flags)) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  return NVB_OK;
}

// The layers of a multi-mapper device query (nvb_query_*), all on one device.
int gatherQueryLayers(NvbMapper* const* mappers, int32_t num_mappers, int32_t layer, int64_t n, const void* in, const void* out,
                      QueryLayers* q) {
  if (!mappers || num_mappers < 1) return fail(NVB_ERR_INVALID_ARGUMENT, "no mappers to query");
  if (num_mappers > kMaxQueryMappers) return fail(NVB_ERR_INVALID_ARGUMENT, "at most 16 mappers per query");
  if (n < 0 || n > kMaxQueryPoints) return fail(NVB_ERR_INVALID_ARGUMENT, "bad number of query points");
  if (n > 0 && (!in || !out)) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  q->n = num_mappers;
  for (int i = 0; i < num_mappers; i++) {
    NvbMapper* m = mappers[i];
    if (!m) return fail(NVB_ERR_INVALID_ARGUMENT, "null mapper");
    if (m->device != mappers[0]->device) return fail(NVB_ERR_INVALID_ARGUMENT, "the mappers of one query must share a device");
    const LayerSlab* L = layerOf(m, layer);
    if (!L) return fail(NVB_ERR_INVALID_ARGUMENT, "a mapper of the query has no such layer");
    q->l[i] = queryLayerOf(m, L->dev());
  }
  return NVB_OK;
}

int runMapperQuery(NvbMapper* const* mappers, int32_t num_mappers, int64_t n, void* caller_stream,
                   const std::function<void(cudaStream_t)>& launch) {
  if (n == 0) return NVB_OK;
  NVB_CUDA(cudaSetDevice(mappers[0]->device));
  return runOrdered(mappers, num_mappers, static_cast<cudaStream_t>(caller_stream), launch);
}

}  // namespace

extern "C" {

int32_t nvb_layer_query_voxels(NvbMapper* m, int32_t layer, const float* xyz, int32_t memory, int64_t n, void* out_voxels,
                               uint8_t* out_success) {
  int rc = checkLayerQueryArgs(m, xyz, memory, n, out_voxels, out_success);
  if (rc) return rc;
  if (layer == NVB_LAYER_MESH) return fail(NVB_ERR_INVALID_ARGUMENT, "the mesh layer has no voxels");
  const LayerSlab* L = layerOf(m, layer);
  if (!L) return fail(NVB_ERR_INVALID_ARGUMENT, "unknown layer");
  if (n == 0) return NVB_OK;
  const QueryLayer q = queryLayerOf(m, L->dev());
  const int voxel_bytes = q.layer.block_bytes / kVpb;
  return runLayerQuery(m, xyz, memory, n, out_voxels, (size_t)voxel_bytes, out_success,
                       [&](const float* x, void* o, uint8_t* f, cudaStream_t st) {
                         launchQueryVoxels(q, voxel_bytes, L == &m->esdf, x, n, o, f, m->num_sms, st);
                       });
}

int32_t nvb_layer_interpolate(NvbMapper* m, int32_t layer, const float* xyz, int32_t memory, int64_t n, float* out_values,
                              uint8_t* out_success) {
  int rc = checkLayerQueryArgs(m, xyz, memory, n, out_values, out_success);
  if (rc) return rc;
  const int kind = layer == NVB_LAYER_TSDF ? kInterpTsdf : layer == NVB_LAYER_ESDF ? kInterpEsdf
                   : layer == NVB_LAYER_OCCUPANCY ? kInterpOccupancy : -1;
  const LayerSlab* L = kind >= 0 ? layerOf(m, layer) : nullptr;
  if (!L) return fail(NVB_ERR_INVALID_ARGUMENT, "interpolation needs the mapper's TSDF, ESDF or occupancy layer");
  if (n == 0) return NVB_OK;
  const QueryLayer q = queryLayerOf(m, L->dev());
  return runLayerQuery(m, xyz, memory, n, out_values, sizeof(float), out_success,
                       [&](const float* x, void* o, uint8_t* f, cudaStream_t st) {
                         launchInterpolate(q, kind, x, n, static_cast<float*>(o), f, m->num_sms, st);
                       });
}

int32_t nvb_query_esdf(NvbMapper* const* mappers, int32_t num_mappers, const float* spheres_xyzr, int64_t n,
                       int32_t with_gradient, float* out, void* caller_stream) {
  QueryLayers q;
  int rc = gatherQueryLayers(mappers, num_mappers, NVB_LAYER_ESDF, n, spheres_xyzr, out, &q);
  if (rc) return rc;
  return runMapperQuery(mappers, num_mappers, n, caller_stream, [&](cudaStream_t st) {
    launchQueryEsdf(q, num_mappers > 1, spheres_xyzr, n, with_gradient != 0, out, mappers[0]->num_sms, st);
  });
}

int32_t nvb_query_tsdf(NvbMapper* const* mappers, int32_t num_mappers, const float* xyz, int64_t n, float* out,
                       void* caller_stream) {
  QueryLayers q;
  int rc = gatherQueryLayers(mappers, num_mappers, NVB_LAYER_TSDF, n, xyz, out, &q);
  if (rc) return rc;
  return runMapperQuery(mappers, num_mappers, n, caller_stream, [&](cudaStream_t st) {
    launchQueryTsdf(q, num_mappers > 1, xyz, n, out, mappers[0]->num_sms, st);
  });
}

int32_t nvb_query_occupancy(NvbMapper* const* mappers, int32_t num_mappers, const float* xyz, int64_t n, float* out,
                            void* caller_stream) {
  QueryLayers q;
  int rc = gatherQueryLayers(mappers, num_mappers, NVB_LAYER_OCCUPANCY, n, xyz, out, &q);
  if (rc) return rc;
  // logOddsFromProbability(0), on the host like the mapper's other log-odds constants
  const float initial = logOddsFromProbability(0.0f);
  return runMapperQuery(mappers, num_mappers, n, caller_stream, [&](cudaStream_t st) {
    launchQueryOccupancy(q, num_mappers > 1, initial, xyz, n, out, mappers[0]->num_sms, st);
  });
}

}  // extern "C"

// ---------------------------------------------------------------------------
// SphereTracer renders (nvb_color.cu)
// ---------------------------------------------------------------------------
namespace {

// Depth (out_rgb == nullptr) or RGBD. Device outputs are ordered like the point queries (runOrdered on `stream`); host
// outputs are rendered into temporaries on `stream` and copied back before the call returns.
int renderImpl(NvbMapper* m, const NvbSphereTracerParams* p, const float* T_L_C, const NvbCamera* cam, float trunc_m, int f,
               int32_t memory, float* out_depth, uint8_t* out_rgb, void* stream) {
  if (m->projective_layer_type == NVB_PROJECTIVE_OCCUPANCY)
    return fail(NVB_ERR_INVALID_ARGUMENT, "the sphere tracer needs a TSDF layer");
  if (p->maximum_steps <= 0 || !(p->maximum_ray_length_m > 0.0f) || !(p->surface_distance_epsilon_vox > 0.0f))
    return fail(NVB_ERR_INVALID_ARGUMENT, "sphere tracer parameter out of range");  // CHECK_GT, sphere_tracer.cu:319-333
  if (int rc = checkMemoryKind(memory)) return rc;
  if (cam->width <= 0 || cam->height <= 0) return fail(NVB_ERR_INVALID_ARGUMENT, "the camera must have a positive size");
  if (f <= 0 || cam->width % f != 0 || cam->height % f != 0)
    return fail(NVB_ERR_INVALID_ARGUMENT, "the ray subsampling factor must divide the image size");  // CHECK_EQ, :432-433
  NVB_CUDA(cudaSetDevice(m->device));
  RenderArgs a{};
  a.tsdf = m->tsdf.dev();
  a.color = m->color.dev();
  a.T_L_C = rigidFromColMajor(T_L_C);
  a.cam = *cam;
  a.block_size = m->block_size;
  a.voxel_size_inv = voxelSizeInv(m->block_size);
  a.trunc_m = trunc_m;
  a.max_steps = p->maximum_steps;
  a.max_ray_len = p->maximum_ray_length_m;
  a.eps_m = p->surface_distance_epsilon_vox * m->voxel_size;
  a.subsample = f;
  a.drows = cam->height / f, a.dcols = cam->width / f;  // getSubsampledImageSize (:335-339)
  const size_t n = (size_t)a.drows * a.dcols;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  CallerBuffers bufs(memory, st, m->stage_pool);
  NVB_CUDA(bufs.out(out_depth, n * sizeof(float), &a.depth));
  NVB_CUDA(bufs.out(out_rgb, 3 * n, &a.rgb));
  const int rc = runOrdered(&m, 1, st, [&](cudaStream_t s) { launchRender(a, s); });
  if (rc) return rc;
  NVB_CUDA(bufs.finish());
  return NVB_OK;
}

}  // namespace

extern "C" {

void nvb_default_sphere_tracer_params(NvbSphereTracerParams* p) {
  if (!p) return;
  p->maximum_steps = 100;  // rays/sphere_tracer.h:216-218
  p->maximum_ray_length_m = 15.0f;
  p->surface_distance_epsilon_vox = 0.1f;
}

int32_t nvb_render_depth(NvbMapper* m, const NvbSphereTracerParams* p, const float* T_L_C, const NvbCamera* cam,
                         float truncation_distance_m, int32_t ray_subsampling_factor, int32_t memory, float* out_depth,
                         void* stream) {
  if (!m || !p || !T_L_C || !cam || !out_depth) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  return renderImpl(m, p, T_L_C, cam, truncation_distance_m, ray_subsampling_factor, memory, out_depth, nullptr, stream);
}

int32_t nvb_render_rgbd(NvbMapper* m, const NvbSphereTracerParams* p, const float* T_L_C, const NvbCamera* cam,
                        float truncation_distance_m, int32_t ray_subsampling_factor, int32_t memory, float* out_depth,
                        uint8_t* out_rgb, void* stream) {
  if (!m || !p || !T_L_C || !cam || !out_depth || !out_rgb) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  return renderImpl(m, p, T_L_C, cam, truncation_distance_m, ray_subsampling_factor, memory, out_depth, out_rgb, stream);
}

}  // extern "C"

// ---------------------------------------------------------------------------
// primitives::Scene (nvb_scene.cu)
// ---------------------------------------------------------------------------
namespace {

// The scene's own checks: the Plane constructor's CHECK_NEAR(normal.norm(), 1.0, 1e-3) (primitives.h), evaluated in double
// like glog's, and Primitive::toString's LOG(FATAL) on an unknown type.
int validateScene(const NvbScene* s) {
  if (!s) return fail(NVB_ERR_INVALID_ARGUMENT, "null scene");
  if (s->num_primitives < 0 || (s->num_primitives > 0 && !s->primitives)) return fail(NVB_ERR_INVALID_ARGUMENT, "bad primitive list");
  for (int i = 0; i < s->num_primitives; i++) {
    const NvbPrimitive& q = s->primitives[i];
    if (q.type < NVB_PRIM_PLANE || q.type > NVB_PRIM_CYLINDER) return fail(NVB_ERR_INVALID_ARGUMENT, "unknown primitive type");
    if (q.type == NVB_PRIM_PLANE) {
      const double norm = std::sqrt(sum3(q.params[0] * q.params[0], q.params[1] * q.params[1], q.params[2] * q.params[2]));
      if (!(norm <= 1.0 + 1e-3 && norm >= 1.0 - 1e-3)) return fail(NVB_ERR_INVALID_ARGUMENT, "a plane's normal is not unit length");
    }
  }
  return NVB_OK;
}

// The scene with its primitives staged on the device by `host`, a CallerBuffers of host memory.
cudaError_t deviceScene(const NvbScene& scene, CallerBuffers* host, NvbScene* out) {
  *out = scene;
  return host->in(scene.primitives, (size_t)scene.num_primitives * sizeof(NvbPrimitive), &out->primitives);
}

int deviceSms() {
  int dev = 0, sms = kHelperCtas;
  if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  return sms;
}

// getBlockIndicesTouchedByBoundingBox (geometry/internal/impl/bounding_boxes_impl.h:28-53): the block-index box of the scene's
// AABB and its number of blocks, which must be at most 2^28, with indices inside the hash key's +-2^20.
int sceneBlockBox(const NvbMapper* m, const NvbScene* scene, int3* lo_out, int3* size_out, long long* cells) {
  const int3 lo = blockIndexFromPosition(m->block_size, Vec3{scene->aabb_min[0], scene->aabb_min[1], scene->aabb_min[2]});
  const int3 hi = blockIndexFromPosition(m->block_size, Vec3{scene->aabb_max[0], scene->aabb_max[1], scene->aabb_max[2]});
  const int3 size = make_int3(std::max(0, hi.x - lo.x + 1), std::max(0, hi.y - lo.y + 1), std::max(0, hi.z - lo.z + 1));
  *cells = (long long)size.x * size.y * size.z;
  if (*cells > (1ll << 28)) return fail(NVB_ERR_CAPACITY, "the scene's AABB covers more than 2^28 blocks");
  if (*cells > 0 && (!indexInRange(lo.x, lo.y, lo.z) || !indexInRange(hi.x, hi.y, hi.z)))
    return fail(NVB_ERR_INDEX_RANGE, "the scene's AABB reaches a block index outside +-2^20");
  if (lo_out) *lo_out = lo, *size_out = size;
  return NVB_OK;
}

// Scene::generateLayerFromScene on L (the mapper's layer layer_id): allocation, then the fill, on m->stream.
int generateLayerImpl(NvbMapper* m, LayerSlab* L, int layer_id, const NvbScene* scene, float max_dist) {
  SceneLayerArgs a{};
  int rc;
  if ((rc = sceneBlockBox(m, scene, &a.box_lo, &a.box_size, &a.cells))) return rc;
  if (L == &m->tsdf) {
    if ((rc = reserveProjective(m, a.cells))) return rc;
  } else {  // the freespace slab: at least the TSDF slab's capacity, doubled until the AABB's blocks fit
    NVB_CUDA(syncAll(m));
    int count = 0, cap = 0;
    NVB_CUDA(L->fillLevel(&count));
    if ((rc = grownCapacity(std::max(L->capacity(), m->tsdf.capacity()), count + a.cells, "the freespace layer", &cap)))
      return rc;
    NVB_CUDA(L->grow(m, cap));
  }
  NVB_CUDA(cudaSetDevice(m->device));
  NVB_CUDA(joinEsdf(m));  // an update_esdf_async may still be reading the layer
  CallerBuffers host(NVB_MEM_HOST, m->stream, m->stage_pool);
  NVB_CUDA(deviceScene(*scene, &host, &a.scene));
  a.layer = L->dev();
  a.layer_id = layer_id;
  a.block_size = m->block_size;
  a.max_dist = max_dist;
  // getVoxelGroundTruthValue: sqrt(3.0) * voxel_size rounded to float, halved in double (exact)
  a.occupied_threshold_m = (float)(std::sqrt(3.0) * (double)m->voxel_size) / 2.0f;
  a.occupied_log_odds = logOddsFromProbability(1.0f);
  a.free_log_odds = logOddsFromProbability(0.0f);
  a.error = m->error_dev;
  launchSceneAllocate(a, m->num_sms, m->stream);
  launchSceneFill(a, m->num_sms, m->stream);
  m->launches += 2;
  NVB_CUDA(cudaStreamSynchronize(m->stream));
  return checkDeviceError(m);
}

// The projective layer as VoxelBlockLayer::copyFrom leaves it before the copy: no blocks, with room for `cells` new ones. Its
// slots are zeroed and handed out again from 0, so every consumer's dirty words are cleared too. The ESDF, colour, mesh and
// freespace layers keep their blocks, so the slab bounds count them as extra: the ESDF's on its own, the others' (which
// follow the projective slab) as the derived slabs' extra blocks. Both slabs are grown first, keeping their contents, so that
// a failed growth leaves the map as it was.
int emptyProjectiveLayer(NvbMapper* m, long long cells) {
  NVB_CUDA(syncAll(m));
  int esdf_n = 0, derived = 0, cap = 0, rc;  // derived: the most blocks a layer that follows the projective slab holds
  for (const LayerSlab* L : m->layers()) {
    if (L == &m->tsdf) continue;
    int n = 0;
    NVB_CUDA(L->fillLevel(&n));
    if (L == &m->esdf) esdf_n = n;
    else derived = std::max(derived, n);
  }
  if ((rc = grownCapacity(m->tsdf.capacity(), cells + derived, "TSDF layer", &cap))) return rc;
  NVB_CUDA(m->tsdf.grow(m, cap));
  if ((rc = growTracker(m, cap)) || (rc = ensureEsdfCapacity(m, cells + esdf_n))) return rc;
  NVB_CUDA(m->tsdf.empty(m->stream));
  m->launches++;
  for (TrackedBlocks& t : m->tracker) {
    if (!t.dirty.get()) continue;
    NVB_CUDA(cudaMemsetAsync(t.dirty.get(), 0, t.dirty.size() * sizeof(int), m->stream));
    NVB_CUDA(cudaMemsetAsync(t.count, 0, sizeof(int), m->stream));
  }
  m->bounds.reset(0, esdf_n, derived);
  NVB_CUDA(cudaStreamSynchronize(m->stream));
  return NVB_OK;
}

}  // namespace

extern "C" {

int32_t nvb_scene_render_depth(const NvbScene* scene, const NvbCamera* cam, const float* T_S_C, float max_dist,
                               float invalid_depth, int32_t memory, float* out_depth, void* stream) {
  int rc;
  if ((rc = validateScene(scene))) return rc;
  if (!cam || !T_S_C || !out_depth) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  if ((rc = checkMemoryKind(memory))) return rc;
  if (cam->width <= 0 || cam->height <= 0) return fail(NVB_ERR_INVALID_ARGUMENT, "the camera must have a positive size");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  SceneDepthArgs a{};
  a.cam = *cam;
  a.T_S_C = rigidFromColMajor(T_S_C);
  a.T_C_S = invertRigid(a.T_S_C);
  a.max_dist = max_dist, a.invalid_depth = invalid_depth;
  a.rows = cam->height, a.cols = cam->width;
  CallerBuffers host(NVB_MEM_HOST, st, nullptr), bufs(memory, st, nullptr);  // no mapper: the device's default pool
  NVB_CUDA(deviceScene(*scene, &host, &a.scene));
  NVB_CUDA(bufs.out(out_depth, (size_t)a.rows * a.cols * sizeof(float), &a.depth));
  launchSceneDepth(a, st);
  NVB_CUDA(cudaGetLastError());
  NVB_CUDA(bufs.finish());
  return NVB_OK;
}

int32_t nvb_scene_signed_distance(const NvbScene* scene, const float* xyz, int32_t memory, int64_t n, float max_dist,
                                  float* out, void* stream) {
  int rc;
  if ((rc = validateScene(scene))) return rc;
  if (n < 0 || (n > 0 && (!xyz || !out))) return fail(NVB_ERR_INVALID_ARGUMENT, "null argument");
  if ((rc = checkMemoryKind(memory))) return rc;
  if (n == 0) return NVB_OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  CallerBuffers host(NVB_MEM_HOST, st, nullptr), bufs(memory, st, nullptr);  // no mapper: the device's default pool
  NvbScene s;
  const float* in_dev;
  float* out_dev;
  NVB_CUDA(deviceScene(*scene, &host, &s));
  NVB_CUDA(bufs.in(xyz, (size_t)n * 3 * sizeof(float), &in_dev));
  NVB_CUDA(bufs.out(out, (size_t)n * sizeof(float), &out_dev));
  launchSceneDistance(s, in_dev, n, max_dist, out_dev, deviceSms(), st);
  NVB_CUDA(cudaGetLastError());
  NVB_CUDA(bufs.finish());
  return NVB_OK;
}

int32_t nvb_scene_generate_layer(NvbMapper* m, int32_t layer_id, const NvbScene* scene, float max_dist) {
  if (!m) return fail(NVB_ERR_INVALID_ARGUMENT, "null mapper");
  int rc;
  if ((rc = validateScene(scene))) return rc;
  // scene_impl.h defines setVoxel for TsdfVoxel, OccupancyVoxel and FreespaceVoxel only
  if (layer_id != NVB_LAYER_TSDF && layer_id != NVB_LAYER_OCCUPANCY && layer_id != NVB_LAYER_FREESPACE)
    return fail(NVB_ERR_INVALID_ARGUMENT, "scenes generate TSDF, occupancy or freespace layers only");
  LayerSlab* L = layerOf(m, layer_id);
  if (!L) return fail(NVB_ERR_INVALID_ARGUMENT, "the mapper has no such layer");
  NVB_CUDA(cudaSetDevice(m->device));
  return generateLayerImpl(m, L, layer_id, scene, max_dist);
}

int32_t nvb_scene_to_mapper(NvbMapper* m, const NvbScene* scene) {
  if (!m) return fail(NVB_ERR_INVALID_ARGUMENT, "null mapper");
  int rc;
  if ((rc = validateScene(scene))) return rc;
  NVB_CUDA(cudaSetDevice(m->device));
  const int layer_id = m->projective_layer_type == NVB_PROJECTIVE_OCCUPANCY ? NVB_LAYER_OCCUPANCY : NVB_LAYER_TSDF;
  // generateLayerImpl's checks, and every slab growth, before the layer is emptied
  long long cells = 0;
  if ((rc = sceneBlockBox(m, scene, nullptr, nullptr, &cells))) return rc;
  // py_scene.cu: copyFrom of the scene's layer with max_distance = 4 voxels
  if ((rc = emptyProjectiveLayer(m, cells))) return rc;
  if ((rc = generateLayerImpl(m, &m->tsdf, layer_id, scene, 4.0f * m->voxel_size))) return rc;
  // markBlocksForUpdate(all blocks): every started consumer's list becomes every block (launchTodoAll); the others start with
  // every block on their first update anyway
  for (int k = 0; k < kNumBlocksToUpdateTypes; k++) {
    TrackedBlocks& t = m->tracker[k];
    if (!t.initialized) continue;
    launchTodoAll(m->tsdf.dev(), t.list(), m->stream);
    m->launches++;
  }
  return nvb_mapper_update_esdf(m, 0);
}

}  // extern "C"
