// comm.cu -- NCCL plumbing and the distributed inner join driver (include/dj_b200.h).
//
// Replaces NCCLCommunicator (src/communicator.cpp:799-875), communicate_sizes
// (src/all_to_all_comm.cpp:54-111), the table all-to-all (:126-189,307-356) and the
// orchestration of distributed_inner_join (src/distributed_join.cpp:134-340):
//   * no MPI: counts travel by ncclAllGather, the unique id comes from the launcher;
//   * no staging copies: buckets are sent from / received into their final buffers;
//   * one ncclGroup per batch covering every column of both tables;
//   * the reference's spinning join thread + std::atomic flags (:100-132,283-322) become two
//     CUDA streams and events: batch b+1's exchange overlaps batch b's local join;
//   * batch results are appended into one output (no cudf::concatenate, :333-339).
#include <cuda.h>
#include <nccl.h>

#include <algorithm>
#include <chrono>
#include <condition_variable>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <mutex>
#include <vector>

#include "dj_device.cuh"
#include "dj_internal.h"

// In-process rank group (dj_comm_create_local_group): the host-side meeting point that replaces
// NCCL's control collectives when every rank is a thread of one process on one device.
struct LocalGroup {
  explicit LocalGroup(int n) : size(n), here(n, 0), in(n), out(n) {}
  int size;
  std::mutex mu;
  std::condition_variable cv;
  uint64_t gen = 0;  // completed all-gathers
  int arrived  = 0;
  std::vector<char> here;                   // [size] arrived in the current generation
  std::vector<std::vector<int64_t>> in, out;  // [size] words being gathered / of the last generation
};

struct dj_comm {
  ncclComm_t nccl = nullptr;
  int rank = 0, size = 1, device = 0;
  ncclComm_t nccl_ctrl     = nullptr;  // duplicate communicator for counts / verdicts, so that tiny
                                       // control collectives never queue behind the bulk exchange
  cudaStream_t comm_stream = nullptr;
  cudaStream_t ctrl_stream = nullptr;
  cudaEvent_t ev_ready     = nullptr;
  cudaEvent_t ev_hist      = nullptr;
  cudaEvent_t ev_part[2]   = {nullptr, nullptr};
  cudaEvent_t ev_seg[2]    = {nullptr, nullptr};
  std::vector<cudaEvent_t> ev_batch;
  // Peer-memory exchange (copy engines over NVLink, no SMs): every rank maps every peer's flag
  // block and -- per call -- workspace through CUDA IPC, pushes its buckets with cudaMemcpyAsync
  // and signals with a stream write; receivers wait with a stream wait-value.
  bool peer_ok = false;
  uint32_t* d_flags = nullptr;               // [size][kFlagSlots], written by peers
  std::vector<uint32_t*> peer_flags;         // peers' d_flags mapped here
  int64_t* d_inbox = nullptr;                // [size][kInbox] control messages deposited by peers (same allocation)
  std::vector<int64_t*> peer_inbox;          // peers' d_inbox mapped here
  uint32_t cseq = 0;                         // control-message sequence number
  std::vector<cudaStream_t> peer_stream;     // one push stream per peer
  struct IpcEntry { cudaIpcMemHandle_t h; char* base; };
  std::vector<std::vector<IpcEntry>> ipc_cache;  // per peer: opened workspace allocations (most recent last)
  std::vector<int64_t> last_handle;              // [size][8] workspace handles seen in the previous call
  uint32_t** d_peer_flags = nullptr;             // device copy of peer_flags (verdict_kernel)
  std::vector<cudaEvent_t> ev_xbeg, ev_xend;     // [2][size] timing events around the pushes (measure_exchange)
  uint32_t seq = 0;
  bool flag_by_memcpy = false;
  bool wait_flush = true;  // CU_STREAM_WAIT_VALUE_FLUSH is dropped if the driver refuses it  // fallback when stream write-value is refused on peer memory
  CUresult (*fn_wait32)(CUstream, CUdeviceptr, cuuint32_t, unsigned int) = nullptr;
  CUresult (*fn_write32)(CUstream, CUdeviceptr, cuuint32_t, unsigned int) = nullptr;
  CUresult (*fn_addr_range)(CUdeviceptr*, size_t*, CUdeviceptr) = nullptr;
  int64_t* h_pinned = nullptr;  // pinned scratch
  int64_t* d_small  = nullptr;  // device scratch for tiny collectives
  size_t small_elems = 0;
  // Set on the members of an in-process group: control all-gathers meet here instead of in NCCL,
  // peer memory is the siblings' own allocations, and nothing synchronises the whole device.
  std::shared_ptr<LocalGroup> group;
};

namespace dj {

#define DJ_NCCL_TRY(expr)                                                                     \
  do {                                                                                        \
    ncclResult_t _r = (expr);                                                                 \
    if (_r != ncclSuccess) {                                                                  \
      dj::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, ncclGetErrorString(_r));    \
      return DJ_ERR_NCCL;                                                                     \
    }                                                                                         \
  } while (0)

constexpr int kFlagSlots = 64;      // per source rank: data flags 0..61, control inbox flag 62, verdict 63
constexpr int kCtrlSlot  = kFlagSlots - 2;
constexpr int kDataSlots = kFlagSlots - 2;
constexpr int kInbox     = 4096;  // int64 words every source rank may deposit per control message
// Messages of one join call (hello, mapping ack, bucket counts) land in separate banks of the inbox: a
// fast rank may already send its NEXT message while a slow peer has not yet read the previous one.
enum { kBankHello = 0, kBankAck = 1, kBankCounts = 2, kBankMisc = 3, kInboxBanks = 4 };
constexpr size_t kSmallElems = 1 << 20;  // int64 entries of pinned + device scratch per communicator

static int ensure_events(dj_comm* c, int n)
{
  while ((int)c->ev_batch.size() < n) {
    cudaEvent_t e;
    DJ_CUDA_TRY(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    c->ev_batch.push_back(e);
  }
  return DJ_OK;
}

}  // namespace dj

using namespace dj;

static int ctrl_allgather(dj_comm* c, const int64_t* h_mine, int n, int64_t* h_all);
static int create_streams_and_scratch(dj_comm* c);

static int ensure_xevents(dj_comm* c, int n)
{
  while ((int)c->ev_xbeg.size() < n) {
    cudaEvent_t a, b;
    DJ_CUDA_TRY(cudaEventCreate(&a));
    DJ_CUDA_TRY(cudaEventCreate(&b));
    c->ev_xbeg.push_back(a);
    c->ev_xend.push_back(b);
  }
  return DJ_OK;
}

// Control all-gather of a local group: each rank's thread deposits its words, the last one to
// arrive publishes the generation.  The wait is bounded so that a rank that never arrives (an
// exception in its thread, a mismatched call sequence) turns into an error, not a hang.
constexpr int kGroupTimeoutS = 120;

static int group_allgather(dj_comm* c, const int64_t* h_mine, int n, int64_t* h_all)
{
  LocalGroup& g = *c->group;
  std::unique_lock<std::mutex> lk(g.mu);
  const uint64_t gen = g.gen;
  g.in[c->rank].assign(h_mine, h_mine + n);
  g.here[c->rank] = 1;
  if (++g.arrived == g.size) {
    // `out` of the previous generation is no longer read: every rank has arrived again since
    g.out.swap(g.in);
    g.arrived = 0;
    std::fill(g.here.begin(), g.here.end(), 0);
    g.gen++;
    g.cv.notify_all();
  } else if (!g.cv.wait_for(lk, std::chrono::seconds(kGroupTimeoutS), [&] { return g.gen != gen; })) {
    int missing = 0;
    while (missing < g.size && g.here[missing]) missing++;
    set_error("local group: rank %d waited %d s at a collective that rank %d never joined", c->rank, kGroupTimeoutS,
              missing);
    return DJ_ERR_NCCL;
  }
  for (int r = 0; r < g.size; r++) {
    DJ_REQUIRE(g.out[r].size() == (size_t)n, "local group: rank %d gathered %d words, rank %d sent %zu", c->rank, n, r,
               g.out[r].size());
    memcpy(h_all + (size_t)r * n, g.out[r].data(), (size_t)n * 8);
  }
  return DJ_OK;
}

// What a local-group rank waits for instead of cudaDeviceSynchronize: a device-wide wait from one
// rank's thread would also wait for a sibling's stream parked on a flag this thread has yet to raise.
static void sync_own_streams(dj_comm* c)
{
  for (cudaStream_t s : {c->comm_stream, c->ctrl_stream})
    if (s) cudaStreamSynchronize(s);
  for (auto ps : c->peer_stream)
    if (ps) cudaStreamSynchronize(ps);
}

// The stream waits until *d_flag >= value (a peer raises it over NVLink).
static int stream_wait_flag(dj_comm* c, cudaStream_t st, const uint32_t* d_flag, uint32_t value)
{
  const CUdeviceptr fa = (CUdeviceptr)d_flag;
  CUresult wr          = CUDA_ERROR_NOT_SUPPORTED;
  if (c->wait_flush) {
    wr = c->fn_wait32((CUstream)st, fa, value, CU_STREAM_WAIT_VALUE_GEQ | CU_STREAM_WAIT_VALUE_FLUSH);
    if (wr != CUDA_SUCCESS) c->wait_flush = false;
  }
  if (wr != CUDA_SUCCESS) wr = c->fn_wait32((CUstream)st, fa, value, CU_STREAM_WAIT_VALUE_GEQ);
  if (wr != CUDA_SUCCESS) {
    set_error("distributed_inner_join: cuStreamWaitValue32 failed with CUresult %d", (int)wr);
    return DJ_ERR_CUDA;
  }
  return DJ_OK;
}

// Control-plane all-gather WITHOUT kernels: every rank deposits `n` int64 words (device or pinned host
// memory) into every peer's inbox with copy-engine copies over NVLink, raises the peer's control
// flag with a stream memory operation, waits for the peers' flags and reads its inbox back.  Unlike
// an NCCL collective it needs no SM, so it is never held up by the persistent partition / join
// kernels that fill the GPU (an NCCL all-gather issued next to them waited for a kernel boundary:
// 4.1 ms measured at N=2).  Every message kind of a call has its own inbox bank (a fast rank's
// counts must not overwrite a hello that a slow peer has not read yet); a bank is safe to reuse in
// the next call because a rank leaves a join only after every peer has published its verdict,
// i.e. long after all banks of that call were read.
static int peer_allgather(dj_comm* c, int bank, const void* src, int n, int64_t* h_all)
{
  DJ_REQUIRE(n >= 1 && n <= kInbox, "control message of %d words exceeds the inbox", n);
  cudaStream_t st    = c->ctrl_stream;
  const uint32_t seq = ++c->cseq;
  const size_t bank_off = (size_t)bank * c->size * kInbox;
  for (int k = 0; k < c->size; k++) {
    const int i = (c->rank + k) % c->size;  // staggered: no two ranks start with the same destination
    DJ_CUDA_TRY(cudaMemcpyAsync(c->peer_inbox[i] + bank_off + (size_t)c->rank * kInbox, src, (size_t)n * 8,
                                cudaMemcpyDefault, st));
    if (i == c->rank) continue;
    uint32_t* flag = c->peer_flags[i] + (size_t)c->rank * kFlagSlots + kCtrlSlot;
    if (!c->flag_by_memcpy && c->fn_write32((CUstream)st, (CUdeviceptr)flag, seq, 0) != CUDA_SUCCESS)
      c->flag_by_memcpy = true;
    if (c->flag_by_memcpy) {
      uint32_t* w = reinterpret_cast<uint32_t*>(c->h_pinned + (910 << 10)) + (seq % 4096);
      *w          = seq;
      DJ_CUDA_TRY(cudaMemcpyAsync(flag, w, 4, cudaMemcpyDefault, st));
    }
  }
  for (int srcr = 0; srcr < c->size; srcr++) {
    if (srcr == c->rank) continue;
    int rc = stream_wait_flag(c, st, c->d_flags + (size_t)srcr * kFlagSlots + kCtrlSlot, seq);
    if (rc) return rc;
  }
  int64_t* land = c->h_pinned + (512 << 10);  // [size][n]
  DJ_REQUIRE((size_t)n * c->size <= (256u << 10), "control message too large for the landing zone");
  DJ_CUDA_TRY(cudaMemcpy2DAsync(land, (size_t)n * 8, c->d_inbox + bank_off, (size_t)kInbox * 8, (size_t)n * 8, c->size,
                                cudaMemcpyDeviceToHost, st));
  DJ_CUDA_TRY(cudaStreamSynchronize(st));
  memcpy(h_all, land, (size_t)n * c->size * 8);
  return DJ_OK;
}

// One thread: this rank's overflow verdict goes into every peer's flag block (slot `slot` of row
// `rank`) as (seq << 1) | overflowed, with system-scope release stores over NVLink.
__global__ void verdict_kernel(const unsigned long long* d_count, unsigned long long capacity,
                               uint32_t* const* peer_flags, int world, int rank, int slots, int slot, uint32_t seq)
{
  if (threadIdx.x != 0) return;
  const uint32_t v = (seq << 1) | (*d_count > capacity ? 1u : 0u);
  for (int p = 0; p < world; p++) {
    uint32_t* f = peer_flags[p] + (size_t)rank * slots + slot;
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(f), "r"(v) : "memory");
  }
}

// Loads the code of every kernel of the library (and the CUB kernels instantiated with it) now.
// Under lazy module loading (CUDA_MODULE_LOADING=LAZY, which PyTorch sets by default) a kernel is
// loaded at its first launch, and the driver may synchronise the whole context to do it.  The
// ranks of a local group share one context: a rank whose stream is parked on a peer's flag then
// holds up the load of a kernel that peer must run before it raises that flag, and neither rank
// moves again, so a group's first join could hang (it is the first launch of most kernels).  Loading everything up
// front, before any rank can wait, removes the load from the ranks' paths.
static int load_all_kernels()
{
  static std::mutex mu;
  static bool done = false;
  std::lock_guard<std::mutex> lock(mu);
  if (done) return DJ_OK;
  cudaDriverEntryPointQueryResult q;
  void* fn = nullptr;
  CUmoduleLoadingMode mode = CU_MODULE_LAZY_LOADING;
  if (cudaGetDriverEntryPoint("cuModuleGetLoadingMode", &fn, cudaEnableDefault, &q) == cudaSuccess && fn &&
      ((CUresult(*)(CUmoduleLoadingMode*))fn)(&mode) == CUDA_SUCCESS && mode == CU_MODULE_EAGER_LOADING) {
    done = true;
    return DJ_OK;
  }
  void *get_module = nullptr, *count = nullptr, *enumerate = nullptr, *load = nullptr;
  const bool found = cudaGetDriverEntryPoint("cuFuncGetModule", &get_module, cudaEnableDefault, &q) == cudaSuccess &&
                     cudaGetDriverEntryPoint("cuModuleGetFunctionCount", &count, cudaEnableDefault, &q) == cudaSuccess &&
                     cudaGetDriverEntryPoint("cuModuleEnumerateFunctions", &enumerate, cudaEnableDefault, &q) ==
                       cudaSuccess &&
                     cudaGetDriverEntryPoint("cuFuncLoad", &load, cudaEnableDefault, &q) == cudaSuccess && get_module &&
                     count && enumerate && load;
  cudaGetLastError();
  if (!found) {
    set_error("the driver cannot load the library's kernels ahead of use (CUDA 12.4 or newer needed); "
              "set CUDA_MODULE_LOADING=EAGER before CUDA starts");
    return DJ_ERR_CUDA;
  }
  const void* anchors[] = {(const void*)verdict_kernel, dj::partition_module_kernel(), dj::join_module_kernel(),
                           dj::generate_module_kernel(), dj::broadcast_module_kernel()};
  for (const void* a : anchors) {
    cudaFunction_t f = nullptr;
    DJ_CUDA_TRY(cudaGetFuncBySymbol(&f, a));
    CUmodule m = nullptr;
    unsigned n = 0;
    bool ok = ((CUresult(*)(CUmodule*, CUfunction))get_module)(&m, (CUfunction)f) == CUDA_SUCCESS &&
              ((CUresult(*)(unsigned*, CUmodule))count)(&n, m) == CUDA_SUCCESS;
    std::vector<CUfunction> fs(n);
    ok = ok && (n == 0 || ((CUresult(*)(CUfunction*, unsigned, CUmodule))enumerate)(fs.data(), n, m) == CUDA_SUCCESS);
    for (unsigned i = 0; ok && i < n; i++) ok = ((CUresult(*)(CUfunction))load)(fs[i]) == CUDA_SUCCESS;
    if (!ok) {
      set_error("cannot load the library's kernels ahead of use; set CUDA_MODULE_LOADING=EAGER before CUDA starts");
      return DJ_ERR_CUDA;
    }
  }
  done = true;
  return DJ_OK;
}

static bool exchange_forced_to_nccl()
{
  const char* mode = getenv("DJ_EXCHANGE");
  return mode && (mode[0] == 'n' || mode[0] == 'N');
}

// The stream memory operations' driver entry points, and this rank's flag block + control inbox
// (zeroed).  *entry_ok: every entry point was found.
static int alloc_ctrl_block(dj_comm* c, bool* entry_ok)
{
  bool ok = true;
  cudaDriverEntryPointQueryResult q;
  void* fn = nullptr;
  if (cudaGetDriverEntryPoint("cuStreamWaitValue32", &fn, cudaEnableDefault, &q) != cudaSuccess || !fn) ok = false;
  c->fn_wait32 = (decltype(c->fn_wait32))fn;
  fn = nullptr;
  if (cudaGetDriverEntryPoint("cuStreamWriteValue32", &fn, cudaEnableDefault, &q) != cudaSuccess || !fn) ok = false;
  c->fn_write32 = (decltype(c->fn_write32))fn;
  fn = nullptr;
  if (cudaGetDriverEntryPoint("cuMemGetAddressRange", &fn, cudaEnableDefault, &q) != cudaSuccess || !fn) ok = false;
  c->fn_addr_range = (decltype(c->fn_addr_range))fn;
  cudaGetLastError();
  *entry_ok = ok;

  const size_t flag_bytes = align_up((size_t)c->size * kFlagSlots * sizeof(uint32_t), 256);
  const size_t ctl_bytes  = flag_bytes + (size_t)kInboxBanks * c->size * kInbox * sizeof(int64_t);
  DJ_CUDA_TRY(cudaMalloc(&c->d_flags, ctl_bytes));
  DJ_CUDA_TRY(cudaMemset(c->d_flags, 0, ctl_bytes));
  c->d_inbox = reinterpret_cast<int64_t*>(reinterpret_cast<char*>(c->d_flags) + flag_bytes);
  return DJ_OK;
}

// Maps every peer's flag block; decides (collectively) whether the copy-engine exchange is usable.
static int setup_peer_exchange(dj_comm* c)
{
  bool ok = !exchange_forced_to_nccl(), entry_ok = false;
  int rc = alloc_ctrl_block(c, &entry_ok);
  if (rc) return rc;
  ok = ok && entry_ok;
  const size_t flag_bytes = align_up((size_t)c->size * kFlagSlots * sizeof(uint32_t), 256);
  cudaIpcMemHandle_t mine;
  if (cudaIpcGetMemHandle(&mine, c->d_flags) != cudaSuccess) {
    ok = false;
    memset(&mine, 0, sizeof(mine));
    cudaGetLastError();
  }
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "CUDA IPC handles are 64 bytes");
  std::vector<int64_t> send(9), all((size_t)c->size * 9);
  send[0] = ok ? 1 : 0;
  memcpy(&send[1], &mine, 64);
  rc = ctrl_allgather(c, send.data(), 9, all.data());
  if (rc) return rc;
  for (int r = 0; r < c->size; r++) ok = ok && all[(size_t)r * 9] == 1;
  c->peer_flags.assign(c->size, nullptr);
  c->peer_inbox.assign(c->size, nullptr);
  c->peer_stream.assign(c->size, nullptr);
  c->ipc_cache.assign(c->size, {});
  int64_t opened = 1;
  if (ok) {
    for (int r = 0; r < c->size; r++) {
      if (r == c->rank) {
        c->peer_flags[r] = c->d_flags;
        c->peer_inbox[r] = c->d_inbox;
        continue;
      }
      cudaIpcMemHandle_t h;
      memcpy(&h, &all[(size_t)r * 9 + 1], 64);
      void* p = nullptr;
      if (cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) {
        opened = 0;
        cudaGetLastError();
        break;
      }
      c->peer_flags[r] = (uint32_t*)p;
      c->peer_inbox[r] = reinterpret_cast<int64_t*>(reinterpret_cast<char*>(p) + flag_bytes);
      DJ_CUDA_TRY(cudaStreamCreateWithFlags(&c->peer_stream[r], cudaStreamNonBlocking));
    }
  }
  std::vector<int64_t> oks(c->size);
  rc = ctrl_allgather(c, &opened, 1, oks.data());
  if (rc) return rc;
  for (int r = 0; r < c->size; r++) ok = ok && oks[r] == 1;
  if (ok) {
    DJ_CUDA_TRY(cudaMalloc(&c->d_peer_flags, (size_t)c->size * sizeof(uint32_t*)));
    DJ_CUDA_TRY(cudaMemcpy(c->d_peer_flags, c->peer_flags.data(), (size_t)c->size * sizeof(uint32_t*),
                           cudaMemcpyHostToDevice));
  }
  c->peer_ok = ok;
  return DJ_OK;
}

// Peer view of rank `peer`'s workspace allocation described by (handle, offset); opened once.
// In a local group the "handle" is the peer's raw workspace pointer: the cache still runs, but
// nothing is opened or closed.
static char* map_peer_workspace(dj_comm* c, int peer, const cudaIpcMemHandle_t& h, int64_t offset)
{
  auto& cache = c->ipc_cache[peer];
  for (size_t i = 0; i < cache.size(); i++)
    if (memcmp(&cache[i].h, &h, sizeof(h)) == 0) {
      const dj_comm::IpcEntry e = cache[i];
      cache.erase(cache.begin() + i);
      cache.push_back(e);  // most recently used last
      return e.base + offset;
    }
  // a peer rarely alternates between more than two live workspaces: older mappings are closed so
  // that the memory behind them can really be released by its owner
  while (cache.size() >= 2) {
    if (!c->group) cudaIpcCloseMemHandle(cache.front().base);
    cache.erase(cache.begin());
  }
  void* p = nullptr;
  if (c->group) {
    memcpy(&p, &h, sizeof(p));
  } else if (cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) {
    cudaGetLastError();
    return nullptr;
  }
  c->ipc_cache[peer].push_back({h, (char*)p});
  return (char*)p + offset;
}

extern "C" int dj_comm_unique_id(void* h_id128)
{
  static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId is expected to be 128 bytes");
  ncclUniqueId id;
  DJ_NCCL_TRY(ncclGetUniqueId(&id));
  memcpy(h_id128, &id, sizeof(id));
  return DJ_OK;
}

extern "C" int dj_comm_create(int rank, int size, const void* h_id128, dj_comm_t** out)
{
  DJ_REQUIRE(out && size >= 1 && rank >= 0 && rank < size, "comm_create: bad rank/size");
  dj_comm* c = new dj_comm();
  c->rank    = rank;
  c->size    = size;
  DJ_CUDA_TRY(cudaGetDevice(&c->device));
  if (size > 1) {
    DJ_REQUIRE(h_id128, "comm_create: unique id missing");
    ncclUniqueId id;
    memcpy(&id, h_id128, sizeof(id));
    DJ_NCCL_TRY(ncclCommInitRank(&c->nccl, size, id, rank));
    DJ_NCCL_TRY(ncclCommSplit(c->nccl, 0, rank, &c->nccl_ctrl, nullptr));
  }
  int rc = create_streams_and_scratch(c);
  if (rc) return rc;
  if (size > 1) {
    rc = load_all_kernels();  // this rank's own streams also park on peer flags
    if (rc) return rc;
    rc = setup_peer_exchange(c);
    if (rc) return rc;
  }
  *out           = c;
  return DJ_OK;
}

extern "C" int dj_comm_create_local_group(int size, dj_comm_t** comms)
{
  DJ_REQUIRE(comms && size >= 1, "comm_create_local_group: bad size");
  if (size == 1) return dj_comm_create(0, 1, nullptr, comms);
  // Every rank queues work on size + 2 streams of one context.  When they share fewer hardware
  // queues, a stream parked on a peer's flag can hold up the write that would raise it.
  const char* e   = getenv("CUDA_DEVICE_MAX_CONNECTIONS");
  const int conns = e && atoi(e) > 0 ? atoi(e) : 8;
  DJ_REQUIRE(size * (size + 2) <= conns,
             "comm_create_local_group: %d ranks use %d streams, more than CUDA_DEVICE_MAX_CONNECTIONS = %d hardware "
             "queues (set it, up to 32, before CUDA starts)", size, size * (size + 2), conns);
  DJ_REQUIRE(!exchange_forced_to_nccl(), "comm_create_local_group: DJ_EXCHANGE=nccl needs NCCL, which a local group "
             "does not have");
  if (int rc = load_all_kernels()) return rc;
  auto g = std::make_shared<LocalGroup>(size);
  std::vector<dj_comm*> cs(size, nullptr);
  auto fail = [&](int rc) {
    for (auto c : cs) dj_comm_destroy(c);
    for (int r = 0; r < size; r++) comms[r] = nullptr;
    return rc;
  };
  bool entry_ok = true;
  for (int r = 0; r < size; r++) {
    dj_comm* c = cs[r] = new dj_comm();
    c->rank = r;
    c->size = size;
    c->group = g;
    int rc = cudaGetDevice(&c->device) == cudaSuccess ? create_streams_and_scratch(c) : DJ_ERR_CUDA;
    bool ok = false;
    if (!rc) rc = alloc_ctrl_block(c, &ok);
    if (rc) return fail(rc);
    entry_ok = entry_ok && ok;
  }
  if (!entry_ok) {
    set_error("comm_create_local_group: the driver lacks the stream memory operations the exchange needs");
    return fail(DJ_ERR_CUDA);
  }
  // peer memory: the siblings' own flag blocks and inboxes, no mapping
  for (int r = 0; r < size; r++) {
    dj_comm* c = cs[r];
    c->peer_flags.assign(size, nullptr);
    c->peer_inbox.assign(size, nullptr);
    c->peer_stream.assign(size, nullptr);
    c->ipc_cache.assign(size, {});
    for (int p = 0; p < size; p++) {
      c->peer_flags[p] = cs[p]->d_flags;
      c->peer_inbox[p] = cs[p]->d_inbox;
      if (p != r && cudaStreamCreateWithFlags(&c->peer_stream[p], cudaStreamNonBlocking) != cudaSuccess) {
        set_error("comm_create_local_group: cudaStreamCreate failed");
        return fail(DJ_ERR_CUDA);
      }
    }
    if (cudaMalloc(&c->d_peer_flags, (size_t)size * sizeof(uint32_t*)) != cudaSuccess ||
        cudaMemcpy(c->d_peer_flags, c->peer_flags.data(), (size_t)size * sizeof(uint32_t*), cudaMemcpyHostToDevice) !=
          cudaSuccess) {
      set_error("comm_create_local_group: cannot allocate the peer flag table");
      return fail(DJ_ERR_CUDA);
    }
    c->peer_ok = true;
  }
  for (int r = 0; r < size; r++) comms[r] = cs[r];
  return DJ_OK;
}

static int create_streams_and_scratch(dj_comm* c)
{
  DJ_CUDA_TRY(cudaStreamCreateWithFlags(&c->comm_stream, cudaStreamNonBlocking));
  DJ_CUDA_TRY(cudaStreamCreateWithFlags(&c->ctrl_stream, cudaStreamNonBlocking));
  DJ_CUDA_TRY(cudaEventCreateWithFlags(&c->ev_ready, cudaEventDisableTiming));
  DJ_CUDA_TRY(cudaEventCreateWithFlags(&c->ev_hist, cudaEventDisableTiming));
  for (int i = 0; i < 2; i++) {
    DJ_CUDA_TRY(cudaEventCreateWithFlags(&c->ev_part[i], cudaEventDisableTiming));
    DJ_CUDA_TRY(cudaEventCreateWithFlags(&c->ev_seg[i], cudaEventDisableTiming));
  }
  DJ_CUDA_TRY(cudaMallocHost(&c->h_pinned, kSmallElems * sizeof(int64_t)));
  DJ_CUDA_TRY(cudaMalloc(&c->d_small, kSmallElems * sizeof(int64_t)));
  c->small_elems = kSmallElems;
  return DJ_OK;
}

extern "C" int dj_comm_destroy(dj_comm_t* c)
{
  if (!c) return DJ_OK;
  if (c->group)
    sync_own_streams(c);
  else
    cudaDeviceSynchronize();
  if (c->nccl_ctrl) ncclCommDestroy(c->nccl_ctrl);
  if (c->nccl) ncclCommDestroy(c->nccl);
  for (int i = 0; i < 2; i++) {
    if (c->ev_part[i]) cudaEventDestroy(c->ev_part[i]);
    if (c->ev_seg[i]) cudaEventDestroy(c->ev_seg[i]);
  }
  if (c->ctrl_stream) cudaStreamDestroy(c->ctrl_stream);
  for (auto ps : c->peer_stream)
    if (ps) cudaStreamDestroy(ps);
  for (int i = 0; i < (int)c->peer_flags.size() && !c->group; i++)
    if (c->peer_flags[i] && i != c->rank) cudaIpcCloseMemHandle(c->peer_flags[i]);
  for (auto& v : c->ipc_cache)
    for (auto& e : v)
      if (!c->group) cudaIpcCloseMemHandle(e.base);
  if (c->d_flags) cudaFree(c->d_flags);
  if (c->d_peer_flags) cudaFree(c->d_peer_flags);
  for (auto e : c->ev_xbeg) cudaEventDestroy(e);
  for (auto e : c->ev_xend) cudaEventDestroy(e);
  if (c->ev_hist) cudaEventDestroy(c->ev_hist);
  for (auto e : c->ev_batch) cudaEventDestroy(e);
  if (c->ev_ready) cudaEventDestroy(c->ev_ready);
  if (c->comm_stream) cudaStreamDestroy(c->comm_stream);
  if (c->h_pinned) cudaFreeHost(c->h_pinned);
  if (c->d_small) cudaFree(c->d_small);
  delete c;
  return DJ_OK;
}

// Collective: every rank closes its mappings of the peers' workspaces, then all ranks meet, so that
// a caller may cudaFree / shrink / regrow its workspace afterwards (freeing memory that an importer
// still has open is undefined behaviour in CUDA IPC).
extern "C" int dj_comm_release_workspace(dj_comm_t* c)
{
  if (!c || c->size == 1) return DJ_OK;
  if (c->group)
    sync_own_streams(c);
  else
    cudaDeviceSynchronize();
  for (auto& v : c->ipc_cache) {
    for (auto& e : v)
      if (!c->group) cudaIpcCloseMemHandle(e.base);
    v.clear();
  }
  c->last_handle.clear();
  cudaGetLastError();
  int64_t one = 1;
  std::vector<int64_t> all(c->size);
  return ctrl_allgather(c, &one, 1, all.data());
}

extern "C" void* dj_comm_nccl_handle(dj_comm_t* c) { return c ? (void*)c->nccl : nullptr; }
extern "C" int dj_comm_rank(const dj_comm_t* c) { return c ? c->rank : 0; }
extern "C" int dj_comm_size(const dj_comm_t* c) { return c ? c->size : 1; }

extern "C" int dj_comm_allgather_i64(dj_comm_t* c, const int64_t* h_mine, int n, int64_t* h_all,
                                     void* stream)
{
  DJ_REQUIRE(c && n >= 0, "allgather: bad argument");
  if (c->size == 1) {
    memcpy(h_all, h_mine, (size_t)n * 8);
    return DJ_OK;
  }
  DJ_REQUIRE((size_t)n * (c->size + 1) <= c->small_elems, "allgather: %d values per rank is too many", n);
  cudaStream_t st = (cudaStream_t)stream;
  if (c->group) {  // same ordering as the NCCL path: the stream's earlier work is done on return
    DJ_CUDA_TRY(cudaStreamSynchronize(st));
    return group_allgather(c, h_mine, n, h_all);
  }
  int64_t* d_send = c->d_small;
  int64_t* d_recv = c->d_small + n;
  memcpy(c->h_pinned, h_mine, (size_t)n * 8);
  DJ_CUDA_TRY(cudaMemcpyAsync(d_send, c->h_pinned, (size_t)n * 8, cudaMemcpyHostToDevice, st));
  DJ_NCCL_TRY(ncclAllGather(d_send, d_recv, (size_t)n, ncclInt64, c->nccl, st));
  DJ_CUDA_TRY(cudaMemcpyAsync(c->h_pinned + n, d_recv, (size_t)n * c->size * 8,
                              cudaMemcpyDeviceToHost, st));
  DJ_CUDA_TRY(cudaStreamSynchronize(st));
  memcpy(h_all, c->h_pinned + n, (size_t)n * c->size * 8);
  return DJ_OK;
}

// Control-plane all-gather on the duplicate communicator and its own stream (blocking, tiny).
static int ctrl_allgather(dj_comm* c, const int64_t* h_mine, int n, int64_t* h_all)
{
  if (c->size == 1) {
    memcpy(h_all, h_mine, (size_t)n * 8);
    return DJ_OK;
  }
  if (c->group) return group_allgather(c, h_mine, n, h_all);
  const size_t half = c->small_elems / 2;  // second half of both scratch areas
  DJ_REQUIRE((size_t)n * (c->size + 1) <= half / 4, "allgather: %d values per rank is too many", n);
  cudaStream_t st = c->ctrl_stream;
  int64_t* hs = c->h_pinned + half + half / 2;
  int64_t* ds = c->d_small + half;
  memcpy(hs, h_mine, (size_t)n * 8);
  DJ_CUDA_TRY(cudaMemcpyAsync(ds, hs, (size_t)n * 8, cudaMemcpyHostToDevice, st));
  DJ_NCCL_TRY(ncclAllGather(ds, ds + n, (size_t)n, ncclInt64, c->nccl_ctrl, st));
  DJ_CUDA_TRY(cudaMemcpyAsync(hs + n, ds + n, (size_t)n * c->size * 8, cudaMemcpyDeviceToHost, st));
  DJ_CUDA_TRY(cudaStreamSynchronize(st));
  memcpy(h_all, hs + n, (size_t)n * c->size * 8);
  return DJ_OK;
}

// Control all-gather of host words: kernel-free peer path when available, NCCL otherwise.
static int ctrl_gather_host(dj_comm* c, int bank, const int64_t* h_mine, int n, int64_t* h_all)
{
  if (c->size > 1 && c->peer_ok && n <= kInbox) {
    int64_t* stage = c->h_pinned + (129 << 10) + (size_t)bank * 64;  // pinned copy: outlives the async copies
    DJ_REQUIRE(n <= 64, "host control message too long");
    memcpy(stage, h_mine, (size_t)n * 8);
    return peer_allgather(c, bank, stage, n, h_all);
  }
  return ctrl_allgather(c, h_mine, n, h_all);
}

extern "C" int dj_comm_barrier(dj_comm_t* c, void* stream)
{
  int64_t mine = 1;
  std::vector<int64_t> all(c ? c->size : 1);
  if (!c || c->size == 1) return cudaStreamSynchronize((cudaStream_t)stream) == cudaSuccess ? DJ_OK : DJ_ERR_CUDA;
  return dj_comm_allgather_i64(c, &mine, 1, all.data(), stream);
}

extern "C" int dj_comm_group_start(dj_comm_t* c)
{
  DJ_REQUIRE(!c || !c->group, "group_start: a local group has no NCCL");
  DJ_NCCL_TRY(ncclGroupStart());
  return DJ_OK;
}
extern "C" int dj_comm_group_end(dj_comm_t* c)
{
  DJ_REQUIRE(!c || !c->group, "group_end: a local group has no NCCL");
  DJ_NCCL_TRY(ncclGroupEnd());
  return DJ_OK;
}
extern "C" int dj_comm_send(dj_comm_t* c, const void* d_buf, int64_t nbytes, int dest, void* stream)
{
  DJ_REQUIRE(c && c->nccl, "send: communicator has no NCCL (size 1 or a local group)");
  DJ_NCCL_TRY(ncclSend(d_buf, (size_t)nbytes, ncclInt8, dest, c->nccl, (cudaStream_t)stream));
  return DJ_OK;
}
extern "C" int dj_comm_recv(dj_comm_t* c, void* d_buf, int64_t nbytes, int source, void* stream)
{
  DJ_REQUIRE(c && c->nccl, "recv: communicator has no NCCL (size 1 or a local group)");
  DJ_NCCL_TRY(ncclRecv(d_buf, (size_t)nbytes, ncclInt8, source, c->nccl, (cudaStream_t)stream));
  return DJ_OK;
}

extern "C" int dj_all_to_all(dj_comm_t* c, int group_size, const int* h_group_ranks, int self_idx,
                             const void* const* h_send_cols, void* const* h_recv_cols,
                             const int64_t* h_send_offsets, const int64_t* h_recv_offsets,
                             const int* h_elem_sizes, int ncols, int include_self, void* stream)
{
  DJ_REQUIRE(c && group_size >= 1 && self_idx >= 0 && self_idx < group_size && ncols >= 0,
             "all_to_all: bad argument");
  DJ_REQUIRE(group_size == 1 || c->nccl, "all_to_all: communicator has no NCCL (size 1 or a local group)");
  cudaStream_t st = (cudaStream_t)stream;
  if (include_self) {
    const int64_t n = h_send_offsets[self_idx + 1] - h_send_offsets[self_idx];
    DJ_REQUIRE(n == h_recv_offsets[self_idx + 1] - h_recv_offsets[self_idx],
               "all_to_all: self send/recv sizes differ");
    for (int col = 0; col < ncols && n > 0; col++) {
      const size_t es = (size_t)h_elem_sizes[col];
      DJ_CUDA_TRY(cudaMemcpyAsync((char*)h_recv_cols[col] + h_recv_offsets[self_idx] * es,
                                  (const char*)h_send_cols[col] + h_send_offsets[self_idx] * es,
                                  (size_t)n * es, cudaMemcpyDeviceToDevice, st));
    }
  }
  if (group_size == 1) return DJ_OK;
  DJ_NCCL_TRY(ncclGroupStart());
  for (int col = 0; col < ncols; col++) {
    const size_t es = (size_t)h_elem_sizes[col];
    for (int i = 0; i < group_size; i++) {
      if (i == self_idx) continue;
      const int64_t ns = h_send_offsets[i + 1] - h_send_offsets[i];
      const int64_t nr = h_recv_offsets[i + 1] - h_recv_offsets[i];
      if (ns > 0)
        DJ_NCCL_TRY(ncclSend((const char*)h_send_cols[col] + h_send_offsets[i] * es, (size_t)ns * es,
                             ncclInt8, h_group_ranks[i], c->nccl, st));
      if (nr > 0)
        DJ_NCCL_TRY(ncclRecv((char*)h_recv_cols[col] + h_recv_offsets[i] * es, (size_t)nr * es,
                             ncclInt8, h_group_ranks[i], c->nccl, st));
    }
  }
  DJ_NCCL_TRY(ncclGroupEnd());
  return DJ_OK;
}

// ------------------------------------------------------------------------- distributed join

static const uint32_t kNvlinkSeed = 12345678u;  // src/distributed_join.cpp:211

// Buckets handed to NCCL start on 32-row (256-byte) boundaries on both the send and the receive
// side: NCCL's peer copies drop to narrow accesses on pointers that are not 16-byte aligned (the
// reference works around the same effect with two staging copies, src/communicator.cpp:820-869).
constexpr int kAlignRows = 32;

static inline int64_t pad_rows(int64_t n) { return (n + kAlignRows - 1) / kAlignRows * kAlignRows; }

// kind 0: inner join; any other kind (semi, anti, left / full outer) builds on the right table with
// the filter plan and a probe-row bit array
static size_t dist_ws_bytes(int64_t nl, int64_t nr, int world, int odf, double slack, int kind = 0)
{
  if (world <= 1 && kind) return local_join_workspace(kind, nr, nl) + 8192;
  if (world <= 1) return local_join_workspace(0, nl < nr ? nl : nr, nl < nr ? nr : nl) + 8192;
  const int nparts = world * odf;
  size_t total     = 1 << 16;
  // partitioned (padded) copies of both tables
  total += align_up((size_t)(nl + (int64_t)nparts * kAlignRows) * sizeof(Row), 256) +
           align_up((size_t)(nr + (int64_t)nparts * kAlignRows) * sizeof(Row), 256);
  total += 2 * pass_workspace_bytes(1, kMaxFanout) + 4 * align_up(((size_t)kMaxFanout + 1) * 8, 256);
  // receive buffers (balanced estimate with slack) + per-(source, sub-bucket) segment tables
  const size_t rl = (size_t)((double)nl * slack) + (size_t)nparts * kAlignRows + 4096;
  const size_t rr = (size_t)((double)nr * slack) + (size_t)nparts * kAlignRows + 4096;
  total += align_up(rl * sizeof(Row), 256) + align_up(rr * sizeof(Row), 256) + (size_t)odf * 8 * 256 +
           (size_t)odf * 2 * 3 * align_up((size_t)kMaxFanout * 8, 256);
  // join scratch for the largest batch (both sides stay alive until the join kernel has run)
  const int64_t bl = (int64_t)(rl / odf) + 4096, br = (int64_t)(rr / odf) + 4096;
  const RadixPlan plan = join_plan(kind, kind ? br : std::min(bl, br));
  total += side_ws_bytes(bl, plan, kMaxFanout) + side_ws_bytes(br, plan, kMaxFanout);
  if (kind) total += filter_bits_bytes(bl, plan);
  return total + 8192;
}

extern "C" size_t dj_distributed_inner_join_workspace_bytes(int64_t nleft, int64_t nright, int world,
                                                            int over_decom_factor)
{
  return dist_ws_bytes(nleft, nright, world, over_decom_factor < 1 ? 1 : over_decom_factor, 1.15);
}

// DJ_TRACE=1: device-side timeline of one call (CUDA event timestamps relative to its start)
struct Trace {
  bool on = false;
  cudaEvent_t base = nullptr;
  std::vector<std::pair<const char*, cudaEvent_t>> marks;
  std::vector<std::pair<const char*, double>> host_marks;  // host wall clock, ms since init
  std::chrono::high_resolution_clock::time_point t0;
  void host(const char* name)
  {
    if (!on) return;
    host_marks.push_back({name, std::chrono::duration<double, std::milli>(
                                  std::chrono::high_resolution_clock::now() - t0).count()});
  }
  void init(cudaStream_t st)
  {
    const char* e = getenv("DJ_TRACE");
    on            = e && e[0] == '1';
    if (!on) return;
    cudaEventCreate(&base);
    cudaEventRecord(base, st);
    t0 = std::chrono::high_resolution_clock::now();
  }
  void mark(const char* name, cudaStream_t st)
  {
    if (!on) return;
    cudaEvent_t ev;
    cudaEventCreate(&ev);
    cudaEventRecord(ev, st);
    marks.push_back({name, ev});
  }
  void dump(int rank)
  {
    if (!on) return;
    for (auto& m : marks) {  // the marks' own events: a device-wide sync could wait on a sibling rank's stream
      float ms = 0;
      cudaEventSynchronize(m.second);
      cudaEventElapsedTime(&ms, base, m.second);
      printf("[trace rank %d] %8.3f ms  %s\n", rank, ms, m.first);
      cudaEventDestroy(m.second);
    }
    cudaEventDestroy(base);
    for (auto& m : host_marks) printf("[trace rank %d] host %8.3f ms  %s\n", rank, m.second, m.first);
    fflush(stdout);
  }
};

static double ms_since(std::chrono::high_resolution_clock::time_point t0)
{
  return std::chrono::duration<double, std::milli>(std::chrono::high_resolution_clock::now() - t0).count();
}

// Words 3..12 of a join's hello: whether peers can map this rank's workspace (3), its offset inside its
// allocation (4) and the allocation's CUDA IPC handle (5..12).
static void workspace_identity(dj_comm* comm, void* d_workspace, int64_t* hello)
{
  if (comm->peer_ok && comm->group) {
    // one address space: the raw workspace pointer stands in for the IPC handle (offset 0)
    hello[3] = 1;
    memcpy(&hello[5], &d_workspace, sizeof(d_workspace));
  } else if (comm->peer_ok) {
    CUdeviceptr base = 0;
    size_t alloc_sz  = 0;
    cudaIpcMemHandle_t wh;
    memset(&wh, 0, sizeof(wh));
    const bool ok = comm->fn_addr_range(&base, &alloc_sz, (CUdeviceptr)d_workspace) == CUDA_SUCCESS &&
                    cudaIpcGetMemHandle(&wh, (void*)base) == cudaSuccess;
    cudaGetLastError();
    hello[3] = ok ? 1 : 0;
    hello[4] = ok ? (int64_t)((CUdeviceptr)d_workspace - base) : 0;
    memcpy(&hello[5], &wh, 64);
  }
}

// Maps every peer's join workspace, described by the call's hello (ipc ok at word 3, offset in the
// allocation at word 4, handle at words 5..12 of every rank's `hello_words`).  Mappings are cached per
// allocation; a peer whose allocation changed since the last call has its old mapping closed first,
// and then every rank agrees that the new mappings worked before anybody pushes.  *use_peer comes in as
// this call's wish for the copy-engine exchange and goes out as the collective decision; peer_ws[r] is
// rank r's workspace as seen from here (nullptr for this rank, or without the peer exchange).
static int map_peer_workspaces(dj_comm* comm, const std::vector<int64_t>& hello, int hello_words, bool* use_peer,
                               std::vector<char*>* peer_ws)
{
  const int world = comm->size, rank = comm->rank;
  auto H = [&](int r, int f) -> int64_t { return hello[(size_t)r * hello_words + f]; };
  for (int r = 0; r < world; r++) *use_peer = *use_peer && H(r, 3) == 1;
  peer_ws->assign(world, nullptr);
  if (!*use_peer) return DJ_OK;
  bool any_new = false;  // identical on every rank: everybody sees the same handles
  if (comm->last_handle.size() != (size_t)world * 8) {
    comm->last_handle.assign((size_t)world * 8, 0);
    any_new = true;
  }
  for (int r = 0; r < world; r++)
    if (memcmp(&comm->last_handle[(size_t)r * 8], &hello[(size_t)r * hello_words + 5], 64) != 0) any_new = true;
  int64_t mapped = 1;
  for (int r = 0; r < world && mapped; r++) {
    if (r == rank) continue;
    cudaIpcMemHandle_t h;
    memcpy(&h, &hello[(size_t)r * hello_words + 5], 64);
    (*peer_ws)[r] = map_peer_workspace(comm, r, h, H(r, 4));
    if (!(*peer_ws)[r]) mapped = 0;
  }
  if (any_new) {
    // a mapping was (re)opened somewhere: agree that it worked before anybody pushes
    std::vector<int64_t> oks(world);
    int rc = ctrl_gather_host(comm, kBankAck, &mapped, 1, oks.data());
    if (rc) return rc;
    for (int r = 0; r < world; r++) *use_peer = *use_peer && oks[r] == 1;
    for (int r = 0; r < world; r++)
      memcpy(&comm->last_handle[(size_t)r * 8], &hello[(size_t)r * hello_words + 5], 64);
  } else if (!mapped) {
    set_error("join exchange: a cached peer mapping disappeared");
    return DJ_ERR_CUDA;
  }
  return DJ_OK;
}

// The collective overflow verdict over peer memory: a one-thread kernel stores this rank's verdict into
// every peer's flag block over NVLink, the stream waits for the peers' words, and their words are
// copied to h_res[1..] (4 bytes per rank) behind the wait.  The caller's one synchronisation of `st`
// then returns the count and every verdict.
static int post_and_await_verdicts(dj_comm* comm, cudaStream_t st, const int64_t* d_count, int64_t out_capacity,
                                   uint32_t seq, int64_t* h_res)
{
  verdict_kernel<<<1, 32, 0, st>>>((const unsigned long long*)d_count, (unsigned long long)out_capacity,
                                   comm->d_peer_flags, comm->size, comm->rank, kFlagSlots, kFlagSlots - 1, seq);
  DJ_LAUNCH_CHECK();
  for (int src = 0; src < comm->size; src++) {
    if (src == comm->rank) continue;
    int rc = stream_wait_flag(comm, st, comm->d_flags + (size_t)src * kFlagSlots + (kFlagSlots - 1), seq << 1);
    if (rc) return rc;
  }
  DJ_CUDA_TRY(cudaMemcpy2DAsync(h_res + 1, 4, comm->d_flags + (kFlagSlots - 1), (size_t)kFlagSlots * 4, 4, comm->size,
                                cudaMemcpyDeviceToHost, st));
  return DJ_OK;
}

// ---- the rank protocol shared by the repartitioned and the broadcast join

namespace dj {

void reset_opts(dj_join_options* opts)
{
  if (!opts) return;
  opts->t_partition_ms = opts->t_comm_ms = opts->t_join_ms = 0;
  opts->bytes_sent = opts->workspace_needed = 0;
  opts->t_exchange_ms[0] = opts->t_exchange_ms[1] = 0;
  opts->t_exchange_total_ms = 0;
}

int single_rank_result(int64_t n, int64_t out_capacity, int64_t* h_out_count)
{
  *h_out_count = n;
  if (n <= out_capacity) return DJ_OK;
  set_error("join output needs %lld rows, capacity %lld", (long long)n, (long long)out_capacity);
  return DJ_ERR_OVERFLOW;
}

}  // namespace dj

constexpr int kHello = 14;  // nleft, nright, workspace bytes, ipc ok, offset in allocation, handle[8], kind word
// A broadcast join's kind word is its kind plus a tag no repartitioned join sends, so that a rank inside
// dj_broadcast_join_i64 and a rank inside a repartitioned join both see a kind mismatch in the one hello
// they both sent, and both return DJ_ERR_ARG.
constexpr int64_t kBroadcastKindTag = 0x100;

// ONE control all-gather opens every multi-rank call: table sizes (from which every rank derives the
// same plan and layouts), workspace size, the CUDA IPC identity of the workspace and the kind word.
// Everything a rank later needs to know about a peer's memory follows from these numbers by pure
// arithmetic.  A kind mismatch is seen identically on every rank.
static int open_call(dj_comm* comm, int64_t kind_word, int64_t nleft, int64_t nright, void* d_workspace,
                     size_t workspace_bytes, std::vector<int64_t>* hello)
{
  int64_t mine[kHello] = {nleft, nright, (int64_t)workspace_bytes, 0, 0};
  mine[13]             = kind_word;
  workspace_identity(comm, d_workspace, mine);
  hello->resize((size_t)comm->size * kHello);
  int rc = ctrl_gather_host(comm, kBankHello, mine, kHello, hello->data());
  if (rc) return rc;
  auto entry = [](int64_t w) { return w >= kBroadcastKindTag ? "broadcast" : "repartitioned"; };
  auto kind  = [](int64_t w) { return (long long)(w >= kBroadcastKindTag ? w - kBroadcastKindTag : w); };
  for (int r = 0; r < comm->size; r++) {
    const int64_t w = (*hello)[(size_t)r * kHello + 13];
    if (w != kind_word) {
      set_error("join: rank %d asked for %s join kind %lld, this rank for %s join kind %lld", r, entry(w), kind(w),
                entry(kind_word), kind(kind_word));
      return DJ_ERR_ARG;
    }
  }
  return DJ_OK;
}

// Raises flag `slot` of this rank's row in rank `peer`'s flag block to `seq`, behind the work queued on
// `ps`: a stream write, or a 4-byte copy from a pinned word where the driver refuses stream writes to
// peer memory.
static int raise_peer_flag(dj_comm* comm, cudaStream_t ps, int peer, int slot, uint32_t seq)
{
  uint32_t* flag = comm->peer_flags[peer] + (size_t)comm->rank * kFlagSlots + slot;
  if (!comm->flag_by_memcpy && comm->fn_write32((CUstream)ps, (CUdeviceptr)flag, seq, 0) != CUDA_SUCCESS)
    comm->flag_by_memcpy = true;
  if (comm->flag_by_memcpy) {
    uint32_t* w = reinterpret_cast<uint32_t*>(comm->h_pinned + (900 << 10)) + (seq % 4096);
    *w          = seq;
    DJ_CUDA_TRY(cudaMemcpyAsync(flag, w, 4, cudaMemcpyDefault, ps));
  }
  return DJ_OK;
}

// The collective overflow verdict once this rank's count n is known: every rank returns DJ_ERR_OVERFLOW
// if any rank's output did not fit, so that callers can retry together.  With peer memory the peers'
// verdicts are in h_res[1..] (post_and_await_verdicts); without, they are all-gathered.
static int overflow_verdict(dj_comm* comm, bool use_peer, int64_t n, int64_t out_capacity, const int64_t* h_res)
{
  int over_rank = -1;
  if (use_peer) {
    const uint32_t* hv = reinterpret_cast<const uint32_t*>(h_res + 1);
    for (int r = 0; r < comm->size; r++)
      if (r != comm->rank && (hv[r] & 1u)) over_rank = r;
    if (n > out_capacity) over_rank = comm->rank;
  } else {
    int64_t over = n > out_capacity ? 1 : 0;
    std::vector<int64_t> overs(comm->size);
    int rc = ctrl_allgather(comm, &over, 1, overs.data());
    if (rc) return rc;
    for (int r = 0; r < comm->size; r++)
      if (overs[r]) over_rank = r;
  }
  if (over_rank < 0) return DJ_OK;
  set_error("join output does not fit on rank %d (this rank: %lld rows, capacity %lld)", over_rank, (long long)n,
            (long long)out_capacity);
  return DJ_ERR_OVERFLOW;
}

// Once a call has issued its exchange, an early return first waits for the exchange's streams: the
// caller may reuse its buffers, and a peer its workspace, as soon as the call has returned.
struct ExchangeDrain {
  dj_comm* comm;
  bool comm_stream;  // the exchange also runs on the communication stream
  bool peers;        // ... and on the peer push streams
  bool armed = false;
  void drain()
  {
    armed = false;
    if (comm_stream) cudaStreamSynchronize(comm->comm_stream);
    if (peers)
      for (int i = 0; i < comm->size; i++)
        if (i != comm->rank) cudaStreamSynchronize(comm->peer_stream[i]);
  }
  ~ExchangeDrain()
  {
    if (armed) drain();
  }
};

// ---- the stages of the repartitioned join

// One rank: the local join is the whole job (src/distributed_join.cpp:186-199).  An anti or outer join
// of an empty right table keeps every left row, a full outer join of an empty left table every right
// row, with the other side null.  *n: the rows of the result; the count lands in h_land first.
static int single_rank_join(int kind, const int64_t* lk, const int64_t* lp, int64_t nl, const int64_t* rk,
                            const int64_t* rp, int64_t nr, int64_t* const out[4], uint8_t* out_sides,
                            int64_t out_capacity, int64_t* d_count, int64_t* h_land, Arena& arena, cudaStream_t st,
                            int64_t* n)
{
  const bool left_only  = (kind == DJ_JOIN_LEFT_ANTI || kind_is_outer(kind)) && nr == 0 && nl > 0;
  const bool right_only = kind == DJ_JOIN_FULL_OUTER && nl == 0 && nr > 0;
  if (left_only || right_only) {
    const int64_t c = std::min(left_only ? nl : nr, out_capacity);
    const int at    = left_only ? 0 : 2;  // columns of the present side
    if (c > 0) {
      DJ_CUDA_TRY(cudaMemcpyAsync(out[at], left_only ? lk : rk, (size_t)c * 8, cudaMemcpyDeviceToDevice, st));
      DJ_CUDA_TRY(cudaMemcpyAsync(out[at + 1], left_only ? lp : rp, (size_t)c * 8, cudaMemcpyDeviceToDevice, st));
    }
    if (c > 0 && kind_is_outer(kind)) {  // the absent side is null
      DJ_CUDA_TRY(cudaMemsetAsync(out[2 - at], 0, (size_t)c * 8, st));
      DJ_CUDA_TRY(cudaMemsetAsync(out[3 - at], 0, (size_t)c * 8, st));
      DJ_CUDA_TRY(cudaMemsetAsync(out_sides, left_only ? DJ_SIDE_LEFT : DJ_SIDE_RIGHT, (size_t)c, st));
    }
  } else if (nl > 0 && nr > 0) {
    int rc = local_join(kind, lk, lp, nl, rk, rp, nr, out, out_sides, out_capacity, d_count, build_on_right(nl, nr),
                        arena, st);
    if (rc) return rc;
  }
  DJ_CUDA_TRY(cudaMemcpyAsync(h_land, d_count, 8, cudaMemcpyDeviceToHost, st));
  DJ_CUDA_TRY(cudaStreamSynchronize(st));
  *n = left_only ? nl : right_only ? nr : *h_land;
  return DJ_OK;
}

// What every rank derives identically from the hello: the radix plan of the batch joins and the shape
// of the rank partition, which may also split every destination's rows into the plan's level-1 buckets.
struct CallPlan {
  int kind, G, odf, nparts;
  RadixPlan plan;
  int sub_bits;  // level-1 bits fused into the rank partition (0: none)
  int F1s;       // sub-buckets per destination in the sender's partition
  int nbk;       // buckets of the sender's partition
  int nseg;      // (source, sub-bucket) segments of a received piece
  size_t pw;     // the rank partition's pass workspace
};

static int agree_plan(int kind, const std::vector<int64_t>& hello, int G, int odf, CallPlan* cp)
{
  const int nparts = G * odf;
  int64_t tot[2]   = {0, 0};
  for (int r = 0; r < G; r++) {
    const int64_t nl = hello[(size_t)r * kHello], nr = hello[(size_t)r * kHello + 1];
    DJ_REQUIRE(nl < ((int64_t)1 << 31) && nr < ((int64_t)1 << 31),
               "distributed_inner_join: per-rank tables are limited to 2^31 rows (rank %d)", r);
    tot[0] += nl;
    tot[1] += nr;
  }
  // rows per rank and batch; every kind but the inner join builds on the right table
  const int64_t est_build = (kind ? tot[1] : std::min(tot[0], tot[1])) / nparts + 1;
  RadixPlan plan          = join_plan(kind, est_build);
  const int bits          = plan.bits1 + plan.bits2;
  int sub_bits            = 0;
  int fit                 = 0;  // largest sub_bits with nparts << sub_bits <= kMaxFanout
  while ((nparts << (fit + 1)) <= kMaxFanout) fit++;
  const char* nofuse = getenv("DJ_NO_FUSE");
  if (plan.bits2 > 0 && fit > 0 && !(nofuse && nofuse[0] == '1')) {
    const int b1 = std::min(plan.bits1, fit);
    if (bits - b1 <= 10) {
      sub_bits   = b1;
      plan.bits1 = b1;
      plan.bits2 = bits - b1;
    }
  }
  *cp = CallPlan{kind, G, odf, nparts, plan, sub_bits, 1 << sub_bits, nparts << sub_bits, G << sub_bits,
                 pass_workspace_bytes(1, nparts << sub_bits)};
  return DJ_OK;
}

// Workspace layout of ANY rank, as offsets from its workspace base: a pure function of that rank's
// table sizes and (for the receive pieces) of the rows it receives -- so every rank can compute where
// its rows go inside every peer without asking.
struct WsLayout {
  size_t count = 0, pws[2] = {0, 0}, prow[2] = {0, 0}, doff[2] = {0, 0}, dcnt[2] = {0, 0}, pbase[2] = {0, 0};
  std::vector<size_t> piece, seg_begin, seg_end, seg_parent;  // [odf*2]
  size_t join_mark = 0, need = 0;
};

// spans[odf*2]: rows of every (batch, table) receive piece; nullptr: the partition part only
static WsLayout ws_layout(const CallPlan& cp, int64_t nl, int64_t nr, const int64_t* spans)
{
  auto off_of = [](const void* p) { return (size_t)reinterpret_cast<uintptr_t>(p); };
  WsLayout L;
  Arena va(nullptr, ~(size_t)0 >> 1);
  L.count = off_of(va.take<int64_t>(32));
  const int64_t n2[2] = {nl, nr};
  for (int t = 0; t < 2; t++) {
    L.pws[t]  = off_of(va.take<char>(cp.pw));
    L.prow[t] = off_of(va.take<Row>((size_t)(n2[t] + (int64_t)cp.nparts * kAlignRows)));
    L.doff[t] = off_of(va.take<int64_t>((size_t)cp.nbk + 1));
    L.pbase[t] = off_of(va.take<Row*>((size_t)cp.nparts));
  }
  L.dcnt[0] = off_of(va.take<int64_t>((size_t)2 * cp.nbk + 2));  // both tables' counts, contiguous: one message
  L.dcnt[1] = L.dcnt[0] + (size_t)cp.nbk * 8;
  L.need = va.used;
  if (!spans) return L;
  L.piece.resize((size_t)cp.odf * 2);
  L.seg_begin.resize((size_t)cp.odf * 2);
  L.seg_end.resize((size_t)cp.odf * 2);
  L.seg_parent.resize((size_t)cp.odf * 2);
  int64_t max_span[2] = {0, 0};
  for (int t = 0; t < 2; t++)
    for (int b = 0; b < cp.odf; b++) {
      const size_t i  = (size_t)b * 2 + t;
      L.piece[i]      = off_of(va.take<Row>((size_t)spans[i] + 8));
      L.seg_begin[i]  = off_of(va.take<int64_t>((size_t)cp.nseg));
      L.seg_end[i]    = off_of(va.take<int64_t>((size_t)cp.nseg));
      L.seg_parent[i] = off_of(va.take<int>((size_t)cp.nseg));
      max_span[t]     = std::max(max_span[t], spans[i]);
    }
  L.join_mark = va.used;
  L.need      = va.used + side_ws_bytes(max_span[0], cp.plan, cp.nseg) + side_ws_bytes(max_span[1], cp.plan, cp.nseg) +
           4096 + (cp.kind ? filter_bits_bytes(max_span[0], cp.plan) : 0);
  return L;
}

// The all-gathered bucket counts of both tables of every rank.
struct Counts {
  const CallPlan& cp;
  std::vector<int64_t> all;  // [source][table][nbk]
  // rows of source `src`'s table t in sub-bucket `sub` of destination bucket q
  int64_t cnt(int src, int t, int q, int sub) const
  {
    return all[((size_t)src * 2 + t) * cp.nbk + ((size_t)q << cp.sub_bits) + sub];
  }
  int64_t sent(int src, int t, int q) const  // rows source `src` sends for destination bucket q
  {
    int64_t c = 0;
    for (int sub = 0; sub < cp.F1s; sub++) c += cnt(src, t, q, sub);
    return c;
  }
  // where source s's rows start inside destination rank r's piece (batch b, table t); s = G: its span
  int64_t piece_begin(int r, int b, int t, int s) const
  {
    int64_t at = 0;
    for (int s2 = 0; s2 < s; s2++) at += pad_rows(sent(s2, t, b * cp.G + r));
    return at;
  }
};

// One received (batch, table) piece: every source's rows, each source padded to kAlignRows, and the
// segment table that splits them into (source, level-1 bucket) segments.
struct Piece {
  std::vector<int64_t> begin, count;  // per source
  int64_t span = 0, rows = 0;
  Row* data = nullptr;
  int64_t *d_seg_begin = nullptr, *d_seg_end = nullptr;
  int* d_seg_parent = nullptr;
};

// This rank's receive pieces in its workspace, and their segment tables copied up on the control stream.
static int receive_pieces(dj_comm* comm, const Counts& C, const WsLayout& my, char* wsb, std::vector<Piece>* pieces)
{
  const CallPlan& cp = C.cp;
  const int G = cp.G, rank = comm->rank, nseg = cp.nseg, F1s = cp.F1s;
  pieces->assign((size_t)cp.odf * 2, Piece{});
  int64_t* hseg = comm->h_pinned + (320 << 10);  // pinned staging for the segment tables
  DJ_REQUIRE(pieces->size() * 3 * (size_t)nseg <= (192u << 10), "distributed_inner_join: too many segments");
  for (int t = 0; t < 2; t++)
    for (int b = 0; b < cp.odf; b++) {
      const size_t i = (size_t)b * 2 + t;
      Piece& pc      = (*pieces)[i];
      pc.begin.resize(G);
      pc.count.resize(G);
      pc.data         = (Row*)(wsb + my.piece[i]);
      pc.d_seg_begin  = (int64_t*)(wsb + my.seg_begin[i]);
      pc.d_seg_end    = (int64_t*)(wsb + my.seg_end[i]);
      pc.d_seg_parent = (int*)(wsb + my.seg_parent[i]);
      int64_t* hb = hseg + i * 3 * nseg;
      int* hpar   = reinterpret_cast<int*>(hb + 2 * (size_t)nseg);
      for (int s = 0; s < G; s++) {
        pc.begin[s] = pc.span;
        pc.count[s] = C.sent(s, t, b * G + rank);
        int64_t at  = pc.span;
        for (int sub = 0; sub < F1s; sub++) {
          const int64_t c          = C.cnt(s, t, b * G + rank, sub);
          hb[s * F1s + sub]        = at;
          hb[nseg + s * F1s + sub] = at + c;
          hpar[s * F1s + sub]      = sub;
          at += c;
        }
        pc.span += pad_rows(pc.count[s]);
        pc.rows += pc.count[s];
      }
      DJ_CUDA_TRY(cudaMemcpyAsync(pc.d_seg_begin, hb, (size_t)nseg * 8, cudaMemcpyHostToDevice, comm->ctrl_stream));
      DJ_CUDA_TRY(cudaMemcpyAsync(pc.d_seg_end, hb + nseg, (size_t)nseg * 8, cudaMemcpyHostToDevice, comm->ctrl_stream));
      DJ_CUDA_TRY(cudaMemcpyAsync(pc.d_seg_parent, hpar, (size_t)nseg * 4, cudaMemcpyHostToDevice, comm->ctrl_stream));
    }
  return DJ_OK;
}

// Fused partition + exchange.  Per table: the bucket cursors restart inside every destination part (a
// part = this rank's slot in one peer's receive piece), the part bases point into the peers'
// workspaces, the scatter kernel runs, and a flag per (batch, table) tells every peer that this rank's
// rows have landed.
static int fused_exchange(dj_comm* comm, const Counts& C, const std::vector<WsLayout>& lay, char* wsb,
                          const std::vector<char*>& peer_ws, PassState pstate[2], uint32_t seq, bool measure,
                          dj_join_options* opts, Trace& trace, cudaStream_t st)
{
  const CallPlan& cp = C.cp;
  const int G = cp.G, rank = comm->rank, nparts = cp.nparts, nbk = cp.nbk;
  int64_t* hcur = comm->h_pinned + (700 << 10);  // [2][nbk] cursors, then [2][nparts] bases
  int64_t* hbas = hcur + 2 * (size_t)nbk;
  for (int t = 0; t < 2; t++) {
    for (int q = 0; q < nparts; q++) {
      const int b = q / G, i = q % G;
      char* base_ws = i == rank ? wsb : peer_ws[i];
      hbas[(size_t)t * nparts + q] =
        (int64_t)(uintptr_t)(base_ws + lay[i].piece[(size_t)b * 2 + t] + (size_t)C.piece_begin(i, b, t, rank) * sizeof(Row));
      int64_t at = 0;
      for (int sub = 0; sub < cp.F1s; sub++) {
        hcur[(size_t)t * nbk + ((size_t)q << cp.sub_bits) + sub] = at;
        at += C.cnt(rank, t, q, sub);
      }
      if (i != rank && opts) opts->bytes_sent += (int64_t)sizeof(Row) * at;
    }
    Row** d_pbase = (Row**)(wsb + lay[rank].pbase[t]);
    DJ_CUDA_TRY(cudaMemcpyAsync(pstate[t].dev.cursor, hcur + (size_t)t * nbk, (size_t)nbk * 8, cudaMemcpyHostToDevice, st));
    DJ_CUDA_TRY(cudaMemcpyAsync(d_pbase, hbas + (size_t)t * nparts, (size_t)nparts * 8, cudaMemcpyHostToDevice, st));
    pstate[t].dev.part_base  = d_pbase;
    pstate[t].dev.part_shift = cp.sub_bits;
    if (measure) DJ_CUDA_TRY(cudaEventRecord(comm->ev_xbeg[t], st));
    int rc = pass_scatter(pstate[t], st);
    if (rc) return rc;
    if (measure) DJ_CUDA_TRY(cudaEventRecord(comm->ev_xend[t], st));
    DJ_CUDA_TRY(cudaEventRecord(comm->ev_part[t], st));
    trace.mark(t ? "partition+exchange(R) done" : "partition+exchange(L) done", st);
    // the flags leave on the communication stream so that the next scatter is not held up
    DJ_CUDA_TRY(cudaStreamWaitEvent(comm->comm_stream, comm->ev_part[t], 0));
    for (int b = 0; b < cp.odf; b++) {
      for (int k = 1; k < G; k++)
        if ((rc = raise_peer_flag(comm, comm->comm_stream, (rank + k) % G, b * 2 + t, seq))) return rc;
      DJ_CUDA_TRY(cudaEventRecord(comm->ev_batch[(size_t)b * 2 + t], comm->comm_stream));
    }
  }
  return DJ_OK;
}

// A batch in which one side received no rows joins nothing (src/distributed_join.cpp:76-82), but an
// anti join keeps its received left rows, and outer joins emit the rows of the non-empty side with the
// other side null.  A piece has padding between its sources, so rows are appended segment by segment.
static int empty_batch_output(int kind, const Piece& L, const Piece& R, int nseg, int64_t* const out[4],
                              uint8_t* out_sides, int64_t out_capacity, int64_t* d_count, cudaStream_t st)
{
  const bool outer = kind_is_outer(kind);
  for (int t = 0; t < 2; t++) {
    const Piece& pc = t ? R : L;
    const bool kept = t ? kind == DJ_JOIN_FULL_OUTER : (kind == DJ_JOIN_LEFT_ANTI || outer);
    if (!kept || pc.rows == 0) continue;
    int64_t longest = 0;
    for (int64_t c : pc.count) longest = std::max(longest, c);
    const int at = t ? 2 : 0;  // columns of this side
    int rc = append_segment_rows(pc.data, pc.d_seg_begin, pc.d_seg_end, nseg, longest, out[at], out[at + 1],
                                 out_capacity, d_count, st, outer ? out[2 - at] : nullptr,
                                 outer ? out[3 - at] : nullptr, outer ? out_sides : nullptr,
                                 outer ? (t ? DJ_SIDE_RIGHT : DJ_SIDE_LEFT) : 0);
    if (rc) return rc;
  }
  return DJ_OK;
}

// measure_exchange: per-direction NVLink throughput of this rank's pushes.  The copy engines work
// through the peer streams one copy after the other, and an event recorded on a waiting stream is
// timestamped when its copy starts -- so a table's window is taken from the FIRST stream's begin event
// to the LATEST end event over all streams, not per stream.
static void read_exchange_windows(dj_comm* comm, bool fused, dj_join_options* opts)
{
  const int G = comm->size, rank = comm->rank;
  const int first = (rank + 1) % G;
  float latest_all = 0;
  for (int t = 0; t < 2; t++) {
    float worst = 0;
    if (fused) {  // the scatter kernel IS the exchange
      if (cudaEventElapsedTime(&worst, comm->ev_xbeg[t], comm->ev_xend[t]) != cudaSuccess) worst = 0;
      opts->t_exchange_ms[t] = worst;
      float ms = 0;
      if (cudaEventElapsedTime(&ms, comm->ev_xbeg[0], comm->ev_xend[t]) == cudaSuccess) latest_all = std::max(latest_all, ms);
      continue;
    }
    for (int i = 0; i < G; i++) {
      if (i == rank) continue;
      float ms = 0;
      if (cudaEventElapsedTime(&ms, comm->ev_xbeg[(size_t)t * G + first], comm->ev_xend[(size_t)t * G + i]) == cudaSuccess)
        worst = std::max(worst, ms);
      if (cudaEventElapsedTime(&ms, comm->ev_xbeg[(size_t)first], comm->ev_xend[(size_t)t * G + i]) == cudaSuccess)
        latest_all = std::max(latest_all, ms);
    }
    opts->t_exchange_ms[t] = worst;
  }
  opts->t_exchange_total_ms = latest_all;  // first push of the left table -> last push of the right table
  cudaGetLastError();
}

// The distributed join of every kind.  kind 0: inner join, out = (left key, left payload, right key,
// right payload).  DJ_JOIN_LEFT_SEMI / DJ_JOIN_LEFT_ANTI: the right table's key column is passed as its
// payload too (d_right_payload == d_right_key), it is always the build side, and out[0..1] receive
// the kept left rows (d_out_rk, d_out_rp are unused).  DJ_JOIN_LEFT_OUTER / DJ_JOIN_FULL_OUTER: the
// right table (with its payload) is always the build side, out as for the inner join, and
// d_out_sides receives every row's DJ_SIDE_* bits.
int dj::distributed_join(dj_comm_t* comm, int kind, const int64_t* d_left_key, const int64_t* d_left_payload,
                         int64_t nleft, const int64_t* d_right_key, const int64_t* d_right_payload, int64_t nright,
                         int64_t* d_out_lk, int64_t* d_out_lp, int64_t* d_out_rk, int64_t* d_out_rp,
                         uint8_t* d_out_sides, int64_t out_capacity, int64_t* h_out_count, dj_join_options* opts,
                         void* d_workspace, size_t workspace_bytes, void* stream)
{
  DJ_REQUIRE(nleft >= 0 && nright >= 0 && h_out_count && d_workspace, "distributed_inner_join: bad argument");
  cudaStream_t st   = (cudaStream_t)stream;
  const int world   = comm ? comm->size : 1;
  const int rank    = comm ? comm->rank : 0;
  const int odf     = (opts && opts->over_decom_factor > 1) ? opts->over_decom_factor : 1;
  const bool timing = opts && opts->report_timing;
  reset_opts(opts);
  Arena arena(d_workspace, workspace_bytes);
  int64_t* d_count = arena.take<int64_t>(32);
  DJ_REQUIRE(d_count, "distributed_inner_join: workspace too small");
  DJ_CUDA_TRY(cudaMemsetAsync(d_count, 0, sizeof(int64_t), st));
  int64_t* const out[4] = {d_out_lk, d_out_lp, d_out_rk, d_out_rp};
  auto t0               = std::chrono::high_resolution_clock::now();

  if (world == 1) {
    int64_t n = 0;
    int rc    = single_rank_join(kind, d_left_key, d_left_payload, nleft, d_right_key, d_right_payload, nright, out,
                                 d_out_sides, out_capacity, d_count, comm ? comm->h_pinned : h_out_count, arena, st, &n);
    if (rc) return rc;
    if (timing) {
      opts->t_join_ms = ms_since(t0);
      // the reference labels this branch's time "Hash partition" (src/distributed_join.cpp:194)
      printf("Rank %d: Hash partition takes %.0fms\n", rank, opts->t_join_ms);
    }
    return single_rank_result(n, out_capacity, h_out_count);
  }

  const int G = world;  // one NVSwitch box: the NVLink group is every rank
  DJ_REQUIRE(G * odf <= kMaxFanout, "distributed_inner_join: %d partitions exceed %d", G * odf, kMaxFanout);
  DJ_REQUIRE(((uintptr_t)d_workspace & 255) == 0, "distributed_inner_join: the workspace must be 256-byte aligned");
  int rc = ensure_events(comm, 2 * odf);
  if (rc) return rc;
  Trace trace;
  trace.init(st);
  // NCCL fallback only: the persistent partition / join kernels leave a couple of SMs idle for the
  // whole call, because the control plane's tiny NCCL all-gathers are kernels too and a GPU
  // saturated by persistent CTAs makes each of them wait for a kernel boundary (measured: up to
  // 4 ms per collective).  The default control plane moves its messages with copy engines.
  struct ReserveGuard {
    explicit ReserveGuard(int dflt)
    {
      const char* e = getenv("DJ_SM_RESERVE");
      set_sm_reserve(e ? atoi(e) : dflt);
    }
    ~ReserveGuard() { set_sm_reserve(0); }
  } reserve_guard(comm->peer_ok ? 0 : 2);  // the peer-memory control plane launches no kernels

  // ---- 0. hello, and the radix plan every rank derives from it
  std::vector<int64_t> hello;
  if ((rc = open_call(comm, kind, nleft, nright, d_workspace, workspace_bytes, &hello))) {
    cudaStreamSynchronize(st);  // nothing is queued but the count reset
    return rc;
  }
  auto H = [&](int r, int f) -> int64_t { return hello[(size_t)r * kHello + f]; };
  CallPlan cp;
  if ((rc = agree_plan(kind, hello, G, odf, &cp))) return rc;
  trace.host("hello gathered, plan agreed");
  const int nparts = cp.nparts, nbk = cp.nbk, nseg = cp.nseg;

  // every rank checks every rank's partition-stage fit: the verdict is identical everywhere
  for (int r = 0; r < world; r++) {
    const WsLayout L = ws_layout(cp, H(r, 0), H(r, 1), nullptr);
    if (L.need > (size_t)H(r, 2)) {
      if (opts) opts->workspace_needed = (int64_t)ws_layout(cp, nleft, nright, nullptr).need;
      set_error("distributed_inner_join: workspace too small on rank %d for the partitioned tables (%zu of %lld bytes)",
                r, L.need, (long long)H(r, 2));
      return DJ_ERR_WORKSPACE;
    }
  }

  // ---- 0b. copy-engine exchange: map every peer's workspace
  bool use_peer = comm->peer_ok && 2 * odf <= kDataSlots;
  std::vector<char*> peer_ws;
  rc = map_peer_workspaces(comm, hello, kHello, &use_peer, &peer_ws);
  if (rc) return rc;
  if (!use_peer && !comm->nccl) {  // identical on every rank: nothing has been queued but the count reset
    set_error("distributed_inner_join: this exchange (odf %d; peer memory carries at most %d) needs NCCL, which a "
              "local group does not have", odf, kDataSlots / 2);
    cudaStreamSynchronize(st);
    return DJ_ERR_ARG;
  }
  trace.host("peer workspaces mapped");
  const uint32_t seq = use_peer ? ++comm->seq : 0;
  // Exchange flavours over peer memory (identical decision on every rank: same environment):
  //   copy   (default) partition into a local table, then copy engines push each bucket to its peer;
  //   fused  the partition kernel's own cp.async.bulk stores write every run straight into the
  //          destination rank's receive piece -- partition and all-to-all are ONE kernel
  //          (src/distributed_join.cpp:211-225 + src/communicator.cpp:811-869 collapsed).
  bool fused = false;
  {
    const char* e = getenv("DJ_EXCHANGE");
    fused         = use_peer && e && (e[0] == 'f' || e[0] == 'F');
  }

  // ---- 1. hash partition (src/distributed_join.cpp:213-225) on the caller's stream, as histogram
  //         halves first: the counts of BOTH tables leave for the host while the scatter kernels run.
  //         Every destination's run of buckets starts on kAlignRows so pushes go straight from it.
  const WsLayout my = ws_layout(cp, nleft, nright, nullptr);
  char* wsb         = (char*)d_workspace;
  const int64_t n_in[2]    = {nleft, nright};
  const int64_t* in_key[2] = {d_left_key, d_right_key};
  const int64_t* in_pay[2] = {d_left_payload, d_right_payload};
  Row* prow[2];
  int64_t* d_cnt[2];
  PassState pstate[2];
  for (int t = 0; t < 2; t++) {
    prow[t]  = (Row*)(wsb + my.prow[t]);
    d_cnt[t] = (int64_t*)(wsb + my.dcnt[t]);
    PassDesc desc{cp.sub_bits ? 2 : 0, kNvlinkSeed, DJ_HASH_MURMUR3, 0, nbk, 1, 1, kAlignRows, nparts, cp.sub_bits};
    PassBuffers pb{};
    pb.in_key = in_key[t]; pb.in_pay[0] = in_pay[t]; pb.out_rows = prow[t];
    pb.nrows = n_in[t]; pb.d_child_off = (int64_t*)(wsb + my.doff[t]); pb.d_child_cnt = d_cnt[t];
    rc = pass_histogram(desc, pb, wsb + my.pws[t], cp.pw, st, &pstate[t]);
    if (rc) return rc;
  }
  DJ_CUDA_TRY(cudaEventRecord(comm->ev_hist, st));
  trace.mark("histograms done", st);
  for (int t = 0; t < 2 && !fused; t++) {
    rc = pass_scatter(pstate[t], st);
    if (rc) return rc;
    DJ_CUDA_TRY(cudaEventRecord(comm->ev_part[t], st));
    trace.mark(t ? "partition(R) done" : "partition(L) done", st);
  }
  trace.host("partition launched");

  // ---- 2. sizes (communicate_sizes, src/all_to_all_comm.cpp:54-111): one all-gather of both
  //         tables' bucket counts, as soon as the histograms are done
  Counts C{cp, std::vector<int64_t>((size_t)world * 2 * nbk)};
  DJ_CUDA_TRY(cudaStreamWaitEvent(comm->ctrl_stream, comm->ev_hist, 0));
  if (comm->peer_ok && 2 * nbk <= kInbox) {
    // device -> every peer's inbox, straight from the histogram's output: no SM, no host hop
    rc = peer_allgather(comm, kBankCounts, d_cnt[0], 2 * nbk, C.all.data());
    if (rc) return rc;
  } else {
    int64_t* hp = comm->h_pinned + (256 << 10);  // D2H landing zone
    DJ_CUDA_TRY(cudaMemcpyAsync(hp, d_cnt[0], (size_t)2 * nbk * 8, cudaMemcpyDeviceToHost, comm->ctrl_stream));
    DJ_CUDA_TRY(cudaStreamSynchronize(comm->ctrl_stream));
    rc = ctrl_allgather(comm, hp, 2 * nbk, C.all.data());
    if (rc) return rc;
  }
  trace.host("counts gathered");
  if (timing) {
    DJ_CUDA_TRY(cudaEventSynchronize(comm->ev_part[1]));
    opts->t_partition_ms = ms_since(t0);
    printf("Rank %d: Hash partition takes %.0fms\n", rank, opts->t_partition_ms);
  }
  auto tcomm = std::chrono::high_resolution_clock::now();
  // my own send offsets: the aligned_offsets_kernel arithmetic restated on the host
  std::vector<int64_t> send_begin((size_t)2 * nparts);
  for (int t = 0; t < 2; t++) {
    int64_t at = 0;
    for (int q = 0; q < nparts; q++) {
      send_begin[(size_t)t * nparts + q] = at;
      at += pad_rows(C.sent(rank, t, q));
    }
  }

  // ---- 3. receive layout of every rank (allocate_communicated_table) + the fit verdict, locally
  std::vector<WsLayout> lay(world);
  std::vector<int64_t> spans((size_t)odf * 2);
  for (int r = 0; r < world; r++) {
    for (int b = 0; b < odf; b++)
      for (int t = 0; t < 2; t++) spans[(size_t)b * 2 + t] = C.piece_begin(r, b, t, G);
    lay[r] = ws_layout(cp, H(r, 0), H(r, 1), spans.data());
  }
  for (int r = 0; r < world; r++)
    if (lay[r].need > (size_t)H(r, 2)) {
      if (opts) opts->workspace_needed = (int64_t)lay[rank].need;
      set_error("distributed_inner_join: workspace too small on rank %d for its received partitions "
                "(needs %zu of %lld bytes; this rank needs %zu)", r, lay[r].need, (long long)H(r, 2), lay[rank].need);
      // nothing has been pushed yet and every rank takes this branch: just drain our own kernels
      cudaStreamSynchronize(st);
      return DJ_ERR_WORKSPACE;
    }
  std::vector<Piece> pieces;
  if ((rc = receive_pieces(comm, C, lay[rank], wsb, &pieces))) return rc;
  DJ_CUDA_TRY(cudaEventRecord(comm->ev_seg[0], comm->ctrl_stream));
  trace.host("pieces laid out");

  // ---- 4. exchange (src/all_to_all_comm.cpp:126-189): every (batch, table) bucket run goes straight
  //         from the partitioned table into the destination's receive piece
  ExchangeDrain drain{comm, true, use_peer};
  const bool measure = opts && opts->measure_exchange && use_peer;
  auto issue_exchange = [&](int b, int t) -> int {
    Piece& pc = pieces[(size_t)b * 2 + t];
    auto sbeg = [&](int dest) { return send_begin[(size_t)t * nparts + (size_t)b * G + dest]; };
    trace.mark(t ? "exchange(R) begin" : "exchange(L) begin", comm->comm_stream);
    // own bucket: device copy (src/all_to_all_comm.cpp:610-653); the rest over NVLink
    if (pc.count[rank] > 0)
      DJ_CUDA_TRY(cudaMemcpyAsync(pc.data + pc.begin[rank], prow[t] + sbeg(rank),
                                  (size_t)pc.count[rank] * sizeof(Row), cudaMemcpyDeviceToDevice, comm->comm_stream));
    if (use_peer) {
      // push every peer's bucket into ITS receive piece with the copy engines (no SMs, so the
      // radix passes running meanwhile keep the whole GPU), then raise that peer's flag
      const int slot = b * 2 + t;
      // destinations in rank+1, rank+2, ... order: at every moment the ranks push along a
      // permutation, so no receiver sees all senders at once (the copy engines work through the
      // peer streams roughly in issue order; starting everybody at rank 0 is an incast)
      for (int k = 1; k < G; k++) {
        const int i     = (rank + k) % G;
        cudaStream_t ps = comm->peer_stream[i];
        DJ_CUDA_TRY(cudaStreamWaitEvent(ps, comm->ev_part[t], 0));
        if (measure && b == 0) DJ_CUDA_TRY(cudaEventRecord(comm->ev_xbeg[(size_t)t * G + i], ps));
        const int64_t ns = C.sent(rank, t, b * G + i);
        if (ns > 0) {
          char* dst = peer_ws[i] + lay[i].piece[(size_t)b * 2 + t] + (size_t)C.piece_begin(i, b, t, rank) * sizeof(Row);
          DJ_CUDA_TRY(cudaMemcpyAsync(dst, prow[t] + sbeg(i), (size_t)ns * sizeof(Row), cudaMemcpyDefault, ps));
          if (opts) opts->bytes_sent += (int64_t)sizeof(Row) * ns;
        }
        if (measure && b == odf - 1) DJ_CUDA_TRY(cudaEventRecord(comm->ev_xend[(size_t)t * G + i], ps));
        int r2 = raise_peer_flag(comm, ps, i, slot, seq);  // ordered behind the data copies on the same stream
        if (r2) return r2;
      }
      DJ_CUDA_TRY(cudaEventRecord(comm->ev_batch[(size_t)b * 2 + t], comm->comm_stream));
      drain.armed = true;
      return DJ_OK;
    }
    DJ_NCCL_TRY(ncclGroupStart());
    for (int i = 0; i < G; i++) {
      if (i == rank) continue;
      const int64_t ns = C.sent(rank, t, b * G + i), nr = pc.count[i];
      if (ns > 0) {
        DJ_NCCL_TRY(ncclSend(prow[t] + sbeg(i), (size_t)ns * sizeof(Row), ncclInt8, i, comm->nccl, comm->comm_stream));
        if (opts) opts->bytes_sent += (int64_t)sizeof(Row) * ns;
      }
      if (nr > 0)
        DJ_NCCL_TRY(ncclRecv(pc.data + pc.begin[i], (size_t)nr * sizeof(Row), ncclInt8, i, comm->nccl,
                             comm->comm_stream));
    }
    DJ_NCCL_TRY(ncclGroupEnd());
    DJ_CUDA_TRY(cudaEventRecord(comm->ev_batch[(size_t)b * 2 + t], comm->comm_stream));
    trace.mark(t ? "exchange(R) end" : "exchange(L) end", comm->comm_stream);
    drain.armed = true;
    return DJ_OK;
  };
  if (measure) {
    rc = ensure_xevents(comm, 2 * G);
    if (rc) return rc;
  }
  if (fused) {
    drain.armed = true;
    if ((rc = fused_exchange(comm, C, lay, wsb, peer_ws, pstate, seq, measure, opts, trace, st))) return rc;
  }
  // batch order (0,L),(0,R),(1,L),...: the left table's pushes start while the right table is
  // still being partitioned
  for (int b = 0; b < odf && !fused; b++)
    for (int t = 0; t < 2; t++) {
      if (b == 0) DJ_CUDA_TRY(cudaStreamWaitEvent(comm->comm_stream, comm->ev_part[t], 0));
      rc = issue_exchange(b, t);
      if (rc) return rc;
    }
  if (timing) {
    DJ_CUDA_TRY(cudaStreamSynchronize(comm->comm_stream));
    if (use_peer)
      for (int i = 0; i < G; i++)
        if (i != rank) DJ_CUDA_TRY(cudaStreamSynchronize(comm->peer_stream[i]));
    opts->t_comm_ms = ms_since(tcomm);
    for (int b = 0; b < odf; b++)
      printf("Rank %d: All-to-all communication on batch %d takes %.0fms\n", rank, b, opts->t_comm_ms / odf);
  }
  trace.host("exchanges issued");
  DJ_CUDA_TRY(cudaStreamWaitEvent(st, comm->ev_seg[0], 0));

  // ---- 5. local join per batch (src/distributed_join.cpp:283-322), appending into one output
  const size_t join_mark = lay[rank].join_mark;
  for (int b = 0; b < odf; b++) {
    auto tj    = std::chrono::high_resolution_clock::now();
    Piece& L   = pieces[(size_t)b * 2];
    Piece& R   = pieces[(size_t)b * 2 + 1];
    arena.used = join_mark;  // join scratch is reused batch after batch (same stream)
    auto await_piece = [&](int t) -> int {
      DJ_CUDA_TRY(cudaStreamWaitEvent(st, comm->ev_batch[(size_t)b * 2 + t], 0));
      if (use_peer) {
        const int slot = b * 2 + t;
        for (int src = 0; src < G; src++) {
          if (src == rank) continue;
          int r2 = stream_wait_flag(comm, st, comm->d_flags + (size_t)src * kFlagSlots + slot, seq);
          if (r2) return r2;
        }
        trace.mark(t ? "arrived(R)" : "arrived(L)", st);
      }
      return DJ_OK;
    };
    if (L.rows == 0 || R.rows == 0) {  // arrivals are still awaited
      for (int t = 0; t < 2; t++)
        if ((rc = await_piece(t))) return rc;
      if ((rc = empty_batch_output(kind, L, R, nseg, out, d_out_sides, out_capacity, d_count, st))) return rc;
      continue;
    }
    const bool right = kind || build_on_right(L.rows, R.rows);  // side[1] is the build side
    PreparedSide side[2];
    for (int t = 0; t < 2; t++) {
      Piece& pc = t ? R : L;
      // each piece is awaited right before ITS radix pass: the left table's pass overlaps the
      // right table's exchange
      if ((rc = await_piece(t))) return rc;
      TableInput in{nullptr, nullptr, pc.data, pc.span, pc.d_seg_begin, pc.d_seg_end, nseg, pc.d_seg_parent,
                    cp.sub_bits > 0};
      trace.mark(t ? "radix(R) begin" : "radix(L) begin", st);
      if ((rc = prepare_side(in, cp.plan, &side[t], arena, st))) return rc;
      trace.mark(t ? "radix(R) end" : "radix(L) end", st);
    }
    rc = join_prepared(kind, side[right], side[!right], cp.plan, out, d_out_sides, out_capacity, d_count, right, arena,
                       st);
    if (rc) return rc;
    trace.mark("join end", st);
    if (timing) {
      DJ_CUDA_TRY(cudaStreamSynchronize(st));
      double ms = ms_since(tj);
      opts->t_join_ms += ms;
      printf("Rank %d: Local join on batch %d takes %.0fms\n", rank, b, ms);
    }
  }
  trace.host("join launched");

  // ---- 6. the overflow verdict is collective and costs no collective: a one-thread kernel stores
  //         this rank's verdict into every peer's flag block over NVLink, the stream waits for the
  //         peers' words, and ONE synchronisation returns count + verdicts.
  int64_t* h_res = comm->h_pinned + (128 << 10);
  if (use_peer) {
    trace.mark("verdict begin", st);
    if ((rc = post_and_await_verdicts(comm, st, d_count, out_capacity, seq, h_res))) return rc;
    trace.mark("verdicts received", st);
  }
  drain.armed = false;
  DJ_CUDA_TRY(cudaMemcpyAsync(h_res, d_count, 8, cudaMemcpyDeviceToHost, st));
  DJ_CUDA_TRY(cudaStreamSynchronize(st));
  trace.host("main stream drained");
  DJ_CUDA_TRY(cudaStreamSynchronize(comm->comm_stream));
  trace.host("streams drained");
  if (use_peer)
    for (int i = 0; i < G; i++)
      if (i != rank) DJ_CUDA_TRY(cudaStreamSynchronize(comm->peer_stream[i]));  // my buckets may be reused now
  *h_out_count = h_res[0];
  if (measure) read_exchange_windows(comm, fused, opts);
  trace.dump(rank);
  return overflow_verdict(comm, use_peer, *h_out_count, out_capacity, h_res);
}

extern "C" int dj_distributed_inner_join_i64(dj_comm_t* comm, const int64_t* d_left_key,
                                             const int64_t* d_left_payload, int64_t nleft,
                                             const int64_t* d_right_key,
                                             const int64_t* d_right_payload, int64_t nright,
                                             int64_t* d_out_lk, int64_t* d_out_lp,
                                             int64_t* d_out_rk, int64_t* d_out_rp,
                                             int64_t out_capacity, int64_t* h_out_count,
                                             dj_join_options* opts, void* d_workspace,
                                             size_t workspace_bytes, void* stream)
{
  return distributed_join(comm, 0, d_left_key, d_left_payload, nleft, d_right_key, d_right_payload, nright, d_out_lk,
                          d_out_lp, d_out_rk, d_out_rp, nullptr, out_capacity, h_out_count, opts, d_workspace,
                          workspace_bytes, stream);
}

extern "C" size_t dj_distributed_left_filter_join_workspace_bytes(int64_t nleft, int64_t nright, int world,
                                                                  int over_decom_factor)
{
  return dist_ws_bytes(nleft, nright, world, over_decom_factor < 1 ? 1 : over_decom_factor, 1.15, DJ_JOIN_LEFT_SEMI);
}

extern "C" int dj_distributed_left_filter_join_i64(dj_comm_t* comm, int kind, const int64_t* d_left_key,
                                                   const int64_t* d_left_payload, int64_t nleft,
                                                   const int64_t* d_right_key, int64_t nright, int64_t* d_out_key,
                                                   int64_t* d_out_payload, int64_t out_capacity,
                                                   int64_t* h_out_count, dj_join_options* opts, void* d_workspace,
                                                   size_t workspace_bytes, void* stream)
{
  DJ_REQUIRE(kind == DJ_JOIN_LEFT_SEMI || kind == DJ_JOIN_LEFT_ANTI, "left_filter_join: unknown join kind %d", kind);
  DJ_REQUIRE(out_capacity >= 0 && (out_capacity == 0 || (d_out_key && d_out_payload)),
             "left_filter_join: bad output columns");
  return distributed_join(comm, kind, d_left_key, d_left_payload, nleft, d_right_key, d_right_key, nright, d_out_key,
                          d_out_payload, nullptr, nullptr, nullptr, out_capacity, h_out_count, opts, d_workspace,
                          workspace_bytes, stream);
}

// An outer join needs what a semi / anti join needs: the same plan, padded sides and probe-row bits
// (the right table's payload travels in the rows either way).
extern "C" size_t dj_distributed_outer_join_workspace_bytes(int64_t nleft, int64_t nright, int world,
                                                            int over_decom_factor)
{
  return dist_ws_bytes(nleft, nright, world, over_decom_factor < 1 ? 1 : over_decom_factor, 1.15, DJ_JOIN_LEFT_OUTER);
}

extern "C" int dj_distributed_outer_join_i64(dj_comm_t* comm, int kind, const int64_t* d_left_key,
                                             const int64_t* d_left_payload, int64_t nleft,
                                             const int64_t* d_right_key, const int64_t* d_right_payload,
                                             int64_t nright, int64_t* d_out_lk, int64_t* d_out_lp,
                                             int64_t* d_out_rk, int64_t* d_out_rp, uint8_t* d_out_sides,
                                             int64_t out_capacity, int64_t* h_out_count, dj_join_options* opts,
                                             void* d_workspace, size_t workspace_bytes, void* stream)
{
  DJ_REQUIRE(kind == DJ_JOIN_LEFT_OUTER || kind == DJ_JOIN_FULL_OUTER, "outer_join: unknown join kind %d", kind);
  DJ_REQUIRE(out_capacity >= 0 && (out_capacity == 0 || (d_out_lk && d_out_lp && d_out_rk && d_out_rp && d_out_sides)),
             "outer_join: bad output columns");
  return distributed_join(comm, kind, d_left_key, d_left_payload, nleft, d_right_key, d_right_payload, nright,
                          d_out_lk, d_out_lp, d_out_rk, d_out_rp, d_out_sides, out_capacity, h_out_count, opts,
                          d_workspace, workspace_bytes, stream);
}

// ------------------------------------------------------------------------- broadcast join

constexpr int kBroadcastFlagSlot = 0;  // data flag: "my right slice has landed in your workspace"
constexpr int kBroadcastBitsFlagSlot = 1;  // full outer: "my match bits for your slice have landed"

// Words of a full outer join's match bits that cover the gathered rows [before, before + n): the words
// [before >> 5, (before + n + 31) >> 5), none for an empty slice.  At most (n + 31) / 32 + 1 words,
// because a slice generally starts inside a word.
static int64_t slice_bit_words(int64_t before, int64_t n) { return n ? ((before + n + 31) >> 5) - (before >> 5) : 0; }

// Workspace of a broadcast join, a pure function of (nleft, R = gathered right rows): count[32] |
// gathered right keys [R] | gathered right payloads [R] | local join scratch.  Every rank's gathered
// columns sit at the same offsets, so every rank knows where its slice goes inside every peer (element
// offset: the right rows of the ranks before it), and every rank can check every rank's fit.  A full
// outer join (`full`) puts two more arrays before the scratch: matched [(R + 31) / 32] words, one bit per
// gathered row that this rank's left rows matched, and the inbox [world][row_words] of the words every
// rank sends for this rank's slice, row_words = (nright + 31) / 32 + 1 for this rank's nright.  The
// inbox's offset depends on R alone, so a sender knows where it lies in every peer.
struct BroadcastLayout {
  size_t count, grk, grp, matched, inbox, scratch, need;
  int64_t row_words;
};
static BroadcastLayout broadcast_layout(int64_t nl, int64_t R, bool full = false, int64_t nright = 0, int world = 1)
{
  BroadcastLayout L{};
  Arena va(reinterpret_cast<void*>(4096), ~(size_t)0 >> 1);  // offsets only
  auto off  = [&](const void* p) { return (size_t)((const char*)p - va.base); };
  L.count   = off(va.take<int64_t>(32));
  L.grk     = off(va.take<int64_t>((size_t)R));
  L.grp     = off(va.take<int64_t>((size_t)R));
  if (full) {
    L.row_words = (nright + 31) / 32 + 1;
    L.matched   = off(va.take<uint32_t>((size_t)(R + 31) / 32));
    L.inbox     = off(va.take<uint32_t>((size_t)world * (size_t)L.row_words));
  }
  L.scratch = align_up(va.used, 256);
  // the ABI's workspace query does not depend on the kind: the larger of the inner and a filter kind
  size_t join = R <= DJ_BROADCAST_TABLE_MAX_ROWS
                  ? broadcast_table_bytes(R, full ? DJ_JOIN_FULL_OUTER : 0)
                  : std::max(local_join_workspace(0, R, nl), local_join_workspace(DJ_JOIN_LEFT_SEMI, R, nl)) + 8192;
  if (full && R > DJ_BROADCAST_TABLE_MAX_ROWS) join = std::max(join, broadcast_radix_mark_bytes(nl, R) + 8192);
  L.need = L.scratch + join;
  return L;
}

extern "C" size_t dj_broadcast_join_workspace_bytes(int64_t nleft, int64_t nright_total)
{
  return broadcast_layout(std::max<int64_t>(nleft, 0), std::max<int64_t>(nright_total, 0)).need;
}

extern "C" size_t dj_broadcast_full_outer_join_workspace_bytes(int64_t nleft, int64_t nright, int64_t nright_total,
                                                               int world)
{
  return broadcast_layout(std::max<int64_t>(nleft, 0), std::max<int64_t>(nright_total, 0), true,
                          std::max<int64_t>(nright, 0), std::max(world, 1))
    .need;
}

// The local join of a broadcast join, chosen from R alone so that every rank takes the same path: the
// hash table while it is small enough to stay in L2, else the radix-partitioned join of that kind with
// the gathered right table as the build side (out = left ++ right).  A full outer join runs as a left
// outer join that also sets d_matched (dj_internal.h).
static int broadcast_local_join(int kind, const int64_t* lk, const int64_t* lp, int64_t nl, const int64_t* grk,
                                const int64_t* grp, int64_t R, int64_t* const out[4], uint8_t* out_sides,
                                int64_t out_capacity, int64_t* d_count, Arena& arena, cudaStream_t st,
                                uint32_t* d_matched = nullptr)
{
  if (R <= DJ_BROADCAST_TABLE_MAX_ROWS)
    return broadcast_hash_join(kind, lk, lp, nl, grk, grp, R, out, out_sides, out_capacity, d_count, arena, st,
                               d_matched);
  if (kind == DJ_JOIN_FULL_OUTER)
    return broadcast_radix_mark_join(lk, lp, nl, grk, grp, R, out, out_sides, out_capacity, d_count, d_matched, arena,
                                     st);
  if (nl == 0) return DJ_OK;
  return local_join(kind, lk, lp, nl, grk, grp, R, out, out_sides, out_capacity, d_count, true, arena, st);
}

// Every rank all-gathers the right table into the same place of its workspace and joins its own left
// rows against it.  Steps: one hello (sizes, workspace, kind), the fit verdict from the layout, the
// peer mappings, the pushes of this rank's right slice into every peer (copy engines and a data flag,
// or grouped NCCL), the local join once every slice has landed, and the overflow verdict.  A full
// outer join adds two steps between the local join and the verdict: every rank sends every peer the
// words of its match bits that cover the peer's slice (copy engines and a second data flag, or
// grouped NCCL), and emits the rows of its own slice whose bit no rank set.
static int broadcast_join(dj_comm_t* comm, int kind, const int64_t* d_left_key, const int64_t* d_left_payload,
                          int64_t nleft, const int64_t* d_right_key, const int64_t* d_right_payload, int64_t nright,
                          int64_t* const out[4], uint8_t* d_out_sides, int64_t out_capacity, int64_t* h_out_count,
                          dj_join_options* opts, void* d_workspace, size_t workspace_bytes, cudaStream_t st)
{
  const bool filter = kind_is_filter(kind), full = kind == DJ_JOIN_FULL_OUTER;
  const int world   = comm ? comm->size : 1;
  const int rank    = comm ? comm->rank : 0;
  const size_t row_bytes = filter ? 8 : 16;  // the key column, and the payload column unless semi / anti
  reset_opts(opts);
  char* wsb = (char*)d_workspace;

  if (world == 1) {
    DJ_REQUIRE(nright < ((int64_t)1 << 31), "broadcast_join: the right table is limited to 2^31 rows");
    const BroadcastLayout L = broadcast_layout(nleft, nright, full, nright, 1);
    if (workspace_bytes < L.need) {
      if (opts) opts->workspace_needed = (int64_t)L.need;
      set_error("broadcast_join: workspace too small (%zu of %zu bytes)", workspace_bytes, L.need);
      return DJ_ERR_WORKSPACE;
    }
    int64_t* d_count = (int64_t*)(wsb + L.count);
    int64_t* grk     = (int64_t*)(wsb + L.grk);
    int64_t* grp     = filter ? grk : (int64_t*)(wsb + L.grp);
    DJ_CUDA_TRY(cudaMemsetAsync(d_count, 0, sizeof(int64_t), st));
    if (nright > 0) {
      DJ_CUDA_TRY(cudaMemcpyAsync(grk, d_right_key, (size_t)nright * 8, cudaMemcpyDeviceToDevice, st));
      if (!filter)
        DJ_CUDA_TRY(cudaMemcpyAsync(grp, d_right_payload, (size_t)nright * 8, cudaMemcpyDeviceToDevice, st));
    }
    Arena arena(wsb + L.scratch, workspace_bytes - L.scratch);
    uint32_t* matched = full ? (uint32_t*)(wsb + L.matched) : nullptr;
    int rc = broadcast_local_join(kind, d_left_key, d_left_payload, nleft, grk, grp, nright, out, d_out_sides,
                                  out_capacity, d_count, arena, st, matched);
    if (rc) return rc;
    if (full && (rc = broadcast_emit_unmatched_right(d_right_key, d_right_payload, nright, matched, 1, 0, 0, out,
                                                     d_out_sides, out_capacity, d_count, st)))
      return rc;
    int64_t n = 0;
    DJ_CUDA_TRY(cudaMemcpyAsync(&n, d_count, 8, cudaMemcpyDeviceToHost, st));
    DJ_CUDA_TRY(cudaStreamSynchronize(st));
    return single_rank_result(n, out_capacity, h_out_count);
  }

  DJ_REQUIRE(((uintptr_t)d_workspace & 255) == 0, "broadcast_join: the workspace must be 256-byte aligned");
  std::vector<int64_t> hello;
  int rc = open_call(comm, kBroadcastKindTag + kind, nleft, nright, d_workspace, workspace_bytes, &hello);
  if (rc) return rc;
  auto H = [&](int r, int f) -> int64_t { return hello[(size_t)r * kHello + f]; };
  int64_t R = 0, before = 0;  // gathered right rows, and those of the ranks before this one
  for (int r = 0; r < world; r++) {
    if (r < rank) before += H(r, 1);
    R += H(r, 1);
  }
  DJ_REQUIRE(R < ((int64_t)1 << 31), "broadcast_join: the gathered right table (%lld rows) is limited to 2^31 rows",
             (long long)R);
  const BroadcastLayout L = broadcast_layout(nleft, R, full, nright, world);
  for (int r = 0; r < world; r++) {
    const size_t need = broadcast_layout(H(r, 0), R, full, H(r, 1), world).need;
    if (need > (size_t)H(r, 2)) {
      if (opts) opts->workspace_needed = (int64_t)L.need;
      set_error("broadcast_join: workspace too small on rank %d (%zu of %lld bytes; this rank needs %zu)", r, need,
                (long long)H(r, 2), L.need);
      return DJ_ERR_WORKSPACE;
    }
  }

  // ---- peer mappings (copy-engine exchange) or NCCL
  bool use_peer = comm->peer_ok;
  std::vector<char*> peer_ws;
  rc = map_peer_workspaces(comm, hello, kHello, &use_peer, &peer_ws);
  if (rc) return rc;
  if (!use_peer && !comm->nccl) {  // identical on every rank: nothing has been queued
    set_error("broadcast_join: the exchange needs peer memory or NCCL, and a local group has no NCCL");
    return DJ_ERR_ARG;
  }
  const uint32_t seq = use_peer ? ++comm->seq : 0;
  int64_t* d_count   = (int64_t*)(wsb + L.count);
  int64_t* grk       = (int64_t*)(wsb + L.grk);
  int64_t* grp       = filter ? grk : (int64_t*)(wsb + L.grp);
  DJ_CUDA_TRY(cudaMemsetAsync(d_count, 0, sizeof(int64_t), st));

  // ---- this rank's right slice into every rank's gathered columns, at element offset `before`
  const int64_t* src_cols[2] = {d_right_key, d_right_payload};
  const size_t dst_off[2]    = {L.grk, L.grp};
  const int ncols            = filter ? 1 : 2;
  for (int c = 0; c < ncols && nright > 0; c++)
    DJ_CUDA_TRY(cudaMemcpyAsync(wsb + dst_off[c] + (size_t)before * 8, src_cols[c], (size_t)nright * 8,
                                cudaMemcpyDeviceToDevice, st));
  ExchangeDrain drain{comm, false, use_peer};  // the NCCL exchange runs on `st`
  if (use_peer) {
    DJ_CUDA_TRY(cudaEventRecord(comm->ev_ready, st));  // the caller's right columns are ready
    // destinations in rank+1, rank+2, ... order, as in the repartitioned exchange: no receiver sees
    // every sender at once
    for (int k = 1; k < world; k++) {
      const int i     = (rank + k) % world;
      cudaStream_t ps = comm->peer_stream[i];
      DJ_CUDA_TRY(cudaStreamWaitEvent(ps, comm->ev_ready, 0));
      for (int c = 0; c < ncols && nright > 0; c++)
        DJ_CUDA_TRY(cudaMemcpyAsync(peer_ws[i] + dst_off[c] + (size_t)before * 8, src_cols[c], (size_t)nright * 8,
                                    cudaMemcpyDefault, ps));
      if ((rc = raise_peer_flag(comm, ps, i, kBroadcastFlagSlot, seq))) return rc;
    }
    drain.armed = true;
    for (int src = 0; src < world; src++) {
      if (src == rank) continue;
      if ((rc = stream_wait_flag(comm, st, comm->d_flags + (size_t)src * kFlagSlots + kBroadcastFlagSlot, seq)))
        return rc;
    }
  } else {
    DJ_NCCL_TRY(ncclGroupStart());
    for (int c = 0; c < ncols; c++) {
      int64_t at = 0;  // first gathered row of rank i
      for (int i = 0; i < world; at += H(i, 1), i++) {
        if (i == rank) continue;
        if (nright > 0) DJ_NCCL_TRY(ncclSend(src_cols[c], (size_t)nright * 8, ncclInt8, i, comm->nccl, st));
        if (H(i, 1) > 0)
          DJ_NCCL_TRY(ncclRecv(wsb + dst_off[c] + (size_t)at * 8, (size_t)H(i, 1) * 8, ncclInt8, i, comm->nccl, st));
      }
    }
    DJ_NCCL_TRY(ncclGroupEnd());
  }
  if (opts) opts->bytes_sent = (int64_t)(world - 1) * nright * (int64_t)row_bytes;

  // ---- local join of this rank's left rows against the gathered right table
  Arena arena(wsb + L.scratch, workspace_bytes - L.scratch);
  uint32_t* matched = full ? (uint32_t*)(wsb + L.matched) : nullptr;
  rc = broadcast_local_join(kind, d_left_key, d_left_payload, nleft, grk, grp, R, out, d_out_sides, out_capacity,
                            d_count, arena, st, matched);
  if (rc) return rc;

  // ---- full outer: every rank's match bits for this rank's slice, then the rows nobody matched
  if (full) {
    std::vector<int64_t> at(world + 1, 0);  // first gathered row of every rank
    for (int r = 0; r < world; r++) at[r + 1] = at[r] + H(r, 1);
    auto words_for = [&](int r) { return slice_bit_words(at[r], H(r, 1)); };
    auto row_of    = [&](int r) { return (H(r, 1) + 31) / 32 + 1; };  // the inbox row length of rank r
    uint32_t* inbox = (uint32_t*)(wsb + L.inbox);
    const int64_t mine = words_for(rank);
    if (mine > 0)  // this rank's own row
      DJ_CUDA_TRY(cudaMemcpyAsync(inbox + (size_t)rank * L.row_words, matched + (before >> 5), (size_t)mine * 4,
                                  cudaMemcpyDeviceToDevice, st));
    if (use_peer) {
      DJ_CUDA_TRY(cudaEventRecord(comm->ev_ready, st));  // `matched` is complete
      for (int k = 1; k < world; k++) {
        const int i     = (rank + k) % world;
        cudaStream_t ps = comm->peer_stream[i];
        DJ_CUDA_TRY(cudaStreamWaitEvent(ps, comm->ev_ready, 0));
        if (words_for(i) > 0)
          DJ_CUDA_TRY(cudaMemcpyAsync(peer_ws[i] + L.inbox + (size_t)rank * row_of(i) * 4, matched + (at[i] >> 5),
                                      (size_t)words_for(i) * 4, cudaMemcpyDefault, ps));
        if ((rc = raise_peer_flag(comm, ps, i, kBroadcastBitsFlagSlot, seq))) return rc;  // also with no words
      }
      for (int src = 0; src < world; src++) {
        if (src == rank) continue;
        if ((rc = stream_wait_flag(comm, st, comm->d_flags + (size_t)src * kFlagSlots + kBroadcastBitsFlagSlot, seq)))
          return rc;
      }
    } else {
      DJ_NCCL_TRY(ncclGroupStart());
      for (int i = 0; i < world; i++) {
        if (i == rank) continue;
        if (words_for(i) > 0)
          DJ_NCCL_TRY(ncclSend(matched + (at[i] >> 5), (size_t)words_for(i) * 4, ncclInt8, i, comm->nccl, st));
        if (mine > 0)
          DJ_NCCL_TRY(ncclRecv(inbox + (size_t)i * L.row_words, (size_t)mine * 4, ncclInt8, i, comm->nccl, st));
      }
      DJ_NCCL_TRY(ncclGroupEnd());
    }
    for (int i = 0; i < world && opts; i++)
      if (i != rank) opts->bytes_sent += words_for(i) * 4;
    rc = broadcast_emit_unmatched_right(d_right_key, d_right_payload, nright, inbox, world, L.row_words,
                                        (int)(before & 31), out, d_out_sides, out_capacity, d_count, st);
    if (rc) return rc;
  }

  // ---- overflow verdict.  Besides agreeing on DJ_ERR_OVERFLOW, it keeps a fast rank from pushing the
  //      NEXT call's right slice into a peer that is still probing this call's gathered columns, and
  //      (full outer) the next call's match bits into a peer that is still emitting from this call's
  //      inbox: a rank's verdict is posted behind its join and emit on its stream, and no rank returns
  //      before it has received every peer's verdict.
  int64_t* h_res = comm->h_pinned + (128 << 10);
  if (use_peer && (rc = post_and_await_verdicts(comm, st, d_count, out_capacity, seq, h_res))) return rc;
  DJ_CUDA_TRY(cudaMemcpyAsync(h_res, d_count, 8, cudaMemcpyDeviceToHost, st));
  DJ_CUDA_TRY(cudaStreamSynchronize(st));
  drain.drain();  // the caller may reuse its right columns once the call returns
  *h_out_count = h_res[0];
  return overflow_verdict(comm, use_peer, *h_out_count, out_capacity, h_res);
}

extern "C" int dj_broadcast_join_i64(dj_comm_t* comm, int kind, const int64_t* d_left_key,
                                     const int64_t* d_left_payload, int64_t nleft, const int64_t* d_right_key,
                                     const int64_t* d_right_payload, int64_t nright, int64_t* d_out_lk,
                                     int64_t* d_out_lp, int64_t* d_out_rk, int64_t* d_out_rp, uint8_t* d_out_sides,
                                     int64_t out_capacity, int64_t* h_out_count, dj_join_options* opts,
                                     void* d_workspace, size_t workspace_bytes, void* stream)
{
  DJ_REQUIRE(kind != DJ_JOIN_FULL_OUTER, "broadcast_join: a full outer join has no broadcast plan (a right row is "
             "unmatched only once every rank's matches are known)");
  DJ_REQUIRE(kind == 0 || kind_is_filter(kind) || kind == DJ_JOIN_LEFT_OUTER, "broadcast_join: unknown join kind %d",
             kind);
  const bool filter = kind_is_filter(kind), outer = kind == DJ_JOIN_LEFT_OUTER;
  DJ_REQUIRE(nleft >= 0 && nright >= 0 && out_capacity >= 0 && h_out_count && d_workspace,
             "broadcast_join: bad argument");
  DJ_REQUIRE((nleft == 0 || (d_left_key && d_left_payload)) &&
               (nright == 0 || (d_right_key && (filter || d_right_payload))),
             "broadcast_join: bad input columns");
  DJ_REQUIRE(out_capacity == 0 || (d_out_lk && d_out_lp && (filter || (d_out_rk && d_out_rp && (!outer || d_out_sides)))),
             "broadcast_join: bad output columns");
  int64_t* const out[4] = {d_out_lk, d_out_lp, d_out_rk, d_out_rp};
  return broadcast_join(comm, kind, d_left_key, d_left_payload, nleft, d_right_key, d_right_payload, nright, out,
                        d_out_sides, out_capacity, h_out_count, opts, d_workspace, workspace_bytes,
                        (cudaStream_t)stream);
}

extern "C" int dj_broadcast_full_outer_join_i64(dj_comm_t* comm, const int64_t* d_left_key,
                                                const int64_t* d_left_payload, int64_t nleft,
                                                const int64_t* d_right_key, const int64_t* d_right_payload,
                                                int64_t nright, int64_t* d_out_lk, int64_t* d_out_lp,
                                                int64_t* d_out_rk, int64_t* d_out_rp, uint8_t* d_out_sides,
                                                int64_t out_capacity, int64_t* h_out_count, dj_join_options* opts,
                                                void* d_workspace, size_t workspace_bytes, void* stream)
{
  DJ_REQUIRE(nleft >= 0 && nright >= 0 && out_capacity >= 0 && h_out_count && d_workspace,
             "broadcast_full_outer_join: bad argument");
  DJ_REQUIRE((nleft == 0 || (d_left_key && d_left_payload)) && (nright == 0 || (d_right_key && d_right_payload)),
             "broadcast_full_outer_join: bad input columns");
  DJ_REQUIRE(out_capacity == 0 || (d_out_lk && d_out_lp && d_out_rk && d_out_rp && d_out_sides),
             "broadcast_full_outer_join: bad output columns");
  int64_t* const out[4] = {d_out_lk, d_out_lp, d_out_rk, d_out_rp};
  return broadcast_join(comm, DJ_JOIN_FULL_OUTER, d_left_key, d_left_payload, nleft, d_right_key, d_right_payload,
                        nright, out, d_out_sides, out_capacity, h_out_count, opts, d_workspace, workspace_bytes,
                        (cudaStream_t)stream);
}
