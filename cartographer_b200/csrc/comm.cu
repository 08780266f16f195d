// Multi-GPU context of the library: one process per GPU, one NCCL communicator, and the
// sharded ConstraintBuilder queue with its single collective.
//
// Reference semantics kept (mapping/internal/constraints/constraint_builder_2d.cc):
//   * every (submap, node) search is independent and only depends on its submap's
//     matcher (:102-111) => submap-major ownership: rank r owns submap s iff
//     owner_of_submap[s] == r, builds only those stacks and runs only those searches;
//   * RunWhenDoneCallback (:279-300) hands the caller ONE vector with all constraints
//     => every rank ends up with the results of ALL jobs, in job order, after exactly one
//     ncclAllGather of fixed-size records on the engine's stream.
#include <dlfcn.h>
#include <nccl.h>

#include <algorithm>
#include <chrono>

#include "engine2d.cuh"

namespace csm {

// libnccl is bound at run time, on the first multi-GPU call, not at link time: a process
// that also hosts PyTorch must end up with ONE libnccl.so.2 (torch's bundled copy, which
// may be newer than the system one), whichever of the two libraries was loaded first.
// RTLD_NOLOAD picks up a copy that is already mapped; otherwise the system library loads.
struct NcclApi {
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t,
                            cudaStream_t) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  bool ok = false;
};

static const NcclApi& Nccl() {
  static const NcclApi api = []() {
    NcclApi a;
    void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD | RTLD_GLOBAL);
    if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    if (!h) return a;
    a.GetUniqueId = reinterpret_cast<decltype(a.GetUniqueId)>(dlsym(h, "ncclGetUniqueId"));
    a.CommInitRank = reinterpret_cast<decltype(a.CommInitRank)>(dlsym(h, "ncclCommInitRank"));
    a.AllGather = reinterpret_cast<decltype(a.AllGather)>(dlsym(h, "ncclAllGather"));
    a.CommDestroy = reinterpret_cast<decltype(a.CommDestroy)>(dlsym(h, "ncclCommDestroy"));
    a.GetErrorString = reinterpret_cast<decltype(a.GetErrorString)>(dlsym(h, "ncclGetErrorString"));
    a.ok = a.GetUniqueId && a.CommInitRank && a.AllGather && a.CommDestroy && a.GetErrorString;
    return a;
  }();
  return api;
}

#define CSM_NCCL_READY()                                                                \
  do {                                                                                  \
    if (!::csm::Nccl().ok) {                                                            \
      ::csm::SetError("libnccl.so.2 could not be loaded: %s", dlerror());               \
      return CSM_E_CUDA;                                                                \
    }                                                                                   \
  } while (0)

#define CSM_NCCL(expr)                                                                  \
  do {                                                                                  \
    ncclResult_t _r = (expr);                                                           \
    if (_r != ncclSuccess) {                                                            \
      ::csm::SetError("%s:%d: %s failed: %s", __FILE__, __LINE__, #expr,                \
                      ::csm::Nccl().GetErrorString(_r));                                \
      return CSM_E_CUDA;                                                                \
    }                                                                                   \
  } while (0)

}  // namespace csm

using namespace csm;

struct csm_ctx {
  int world = 1, rank = 0, device = 0;
  ncclComm_t comm = nullptr;
  cudaStream_t stream = nullptr;
  DevBuf send, recv;
  PinnedBuf h_send, h_recv;
  std::mutex mu;
};

static_assert(sizeof(ncclUniqueId) == CSM_COMM_ID_BYTES, "CSM_COMM_ID_BYTES");

namespace {
// What both csm_cb_batch*_run do with the WHOLE queue (identical on every rank): job j belongs
// to submap submap_of(jobs[j]) and runs on rank submap_owner[that submap] (NULL => submap %
// world_size); `run(jobs, n, results)` runs this rank's share locally.  With more than one rank,
// ONE allgather of fixed-size {job index, result} records, padded to the largest shard, then
// leaves results[0 .. num_jobs) in job order on every rank.
template <typename Job, typename Result, typename SubmapOf, typename HasSubmap, typename Run>
csm_status ShardedQueue(csm_ctx* ctx, const Job* jobs, int32_t num_jobs, int32_t num_submaps,
                        const int32_t* submap_owner, Result* results, csm_stats* stats,
                        SubmapOf submap_of, const char* bad_index, HasSubmap has_submap,
                        const char* not_held, Run run) {
  if (stats) std::memset(stats, 0, sizeof(*stats));
  if (num_jobs == 0) return CSM_OK;
  const int W = ctx->world;
  std::vector<int> mine;
  std::vector<int> per_rank(W, 0);
  for (int j = 0; j < num_jobs; ++j) {
    const int s = submap_of(jobs[j]);
    CSM_REQUIRE(s >= 0 && s < num_submaps, bad_index);
    const int o = submap_owner ? submap_owner[s] : s % W;
    CSM_REQUIRE(o >= 0 && o < W, "submap owner out of range");
    ++per_rank[o];
    if (o == ctx->rank) mine.push_back(j);
  }
  // local searches
  std::vector<Job> my_jobs(mine.size());
  std::vector<Result> my_results(mine.size());
  for (size_t i = 0; i < mine.size(); ++i) {
    my_jobs[i] = jobs[mine[i]];
    CSM_REQUIRE(has_submap(submap_of(my_jobs[i])), not_held);
  }
  if (!mine.empty())
    CSM_TRY(run(my_jobs.data(), static_cast<int32_t>(my_jobs.size()), my_results.data()));
  if (W == 1) {
    for (size_t i = 0; i < mine.size(); ++i) results[mine[i]] = my_results[i];
    return CSM_OK;
  }
  const int max_per_rank = *std::max_element(per_rank.begin(), per_rank.end());
  struct Record { int32_t job; int32_t pad; Result r; };
  static_assert(sizeof(Record) == 8 + sizeof(Result), "record layout");
  std::vector<Record> send(static_cast<size_t>(max_per_rank));
  for (size_t i = 0; i < send.size(); ++i) {
    send[i].job = i < mine.size() ? mine[i] : -1;
    send[i].pad = 0;
    if (i < mine.size()) send[i].r = my_results[i];
    else std::memset(&send[i].r, 0, sizeof(Result));
  }
  std::vector<Record> recv(static_cast<size_t>(max_per_rank) * W);
  const auto t0 = std::chrono::steady_clock::now();
  CSM_TRY(csm_ctx_allgather(ctx, send.data(), static_cast<int64_t>(sizeof(Record)) * max_per_rank,
                            recv.data()));
  if (stats)
    stats->collective_ms +=
        std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count();
  for (const Record& rec : recv)
    if (rec.job >= 0 && rec.job < num_jobs) results[rec.job] = rec.r;
  return CSM_OK;
}
}  // namespace

extern "C" {

csm_status csm_comm_unique_id(uint8_t id[CSM_COMM_ID_BYTES]) {
  CSM_REQUIRE(id != nullptr, "null pointer");
  CSM_NCCL_READY();
  ncclUniqueId u;
  CSM_NCCL(Nccl().GetUniqueId(&u));
  std::memcpy(id, &u, sizeof(u));
  return CSM_OK;
}

csm_status csm_ctx_create(int32_t world_size, int32_t rank, int32_t device,
                          const uint8_t id[CSM_COMM_ID_BYTES], csm_ctx** out) {
  CSM_REQUIRE(out != nullptr, "null pointer");
  CSM_REQUIRE(world_size >= 1 && rank >= 0 && rank < world_size, "rank / world size");
  CSM_REQUIRE(world_size == 1 || id != nullptr, "a unique id is needed for world_size > 1");
  int count = 0;
  CSM_CUDA(cudaGetDeviceCount(&count));
  CSM_REQUIRE(device >= 0 && device < count, "device index out of range");
  CSM_CUDA(cudaSetDevice(device));
  std::unique_ptr<csm_ctx> c(new csm_ctx);
  c->world = world_size;
  c->rank = rank;
  c->device = device;
  CSM_CUDA(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
  if (world_size > 1) {
    CSM_NCCL_READY();
    ncclUniqueId u;
    std::memcpy(&u, id, sizeof(u));
    CSM_NCCL(Nccl().CommInitRank(&c->comm, world_size, u, rank));
  }
  *out = c.release();
  return CSM_OK;
}

csm_status csm_ctx_destroy(csm_ctx* ctx) {
  if (!ctx) return CSM_OK;
  cudaSetDevice(ctx->device);
  if (ctx->stream) cudaStreamSynchronize(ctx->stream);
  if (ctx->comm) Nccl().CommDestroy(ctx->comm);
  if (ctx->stream) cudaStreamDestroy(ctx->stream);
  cudaFree(ctx->send.p);
  cudaFree(ctx->recv.p);
  cudaFreeHost(ctx->h_send.p);
  cudaFreeHost(ctx->h_recv.p);
  delete ctx;
  return CSM_OK;
}

csm_status csm_ctx_info(const csm_ctx* ctx, int32_t* world_size, int32_t* rank, int32_t* device) {
  CSM_REQUIRE(ctx != nullptr, "null context");
  if (world_size) *world_size = ctx->world;
  if (rank) *rank = ctx->rank;
  if (device) *device = ctx->device;
  return CSM_OK;
}

// Gathers `bytes` bytes from every rank into recv (world * bytes, rank-major) with ONE
// ncclAllGather on the context's stream; host buffers in, host buffers out.
csm_status csm_ctx_allgather(csm_ctx* ctx, const void* send, int64_t bytes, void* recv) {
  CSM_REQUIRE(ctx && send && recv && bytes >= 0, "arguments");
  if (bytes == 0) return CSM_OK;
  std::lock_guard<std::mutex> lock(ctx->mu);
  if (ctx->world == 1) {
    std::memcpy(recv, send, static_cast<size_t>(bytes));
    return CSM_OK;
  }
  CSM_CUDA(cudaSetDevice(ctx->device));
  const size_t b = static_cast<size_t>(bytes);
  CSM_TRY(ctx->send.Reserve(b));
  CSM_TRY(ctx->recv.Reserve(b * ctx->world));
  CSM_TRY(ctx->h_send.Reserve(b));
  CSM_TRY(ctx->h_recv.Reserve(b * ctx->world));
  std::memcpy(ctx->h_send.p, send, b);
  CSM_CUDA(cudaMemcpyAsync(ctx->send.p, ctx->h_send.p, b, cudaMemcpyHostToDevice, ctx->stream));
  CSM_NCCL(Nccl().AllGather(ctx->send.p, ctx->recv.p, b, ncclUint8, ctx->comm, ctx->stream));
  CSM_CUDA(cudaMemcpyAsync(ctx->h_recv.p, ctx->recv.p, b * ctx->world, cudaMemcpyDeviceToHost,
                           ctx->stream));
  CSM_CUDA(cudaStreamSynchronize(ctx->stream));
  std::memcpy(recv, ctx->h_recv.p, b * ctx->world);
  return CSM_OK;
}

// The sharded 2D queue.  `jobs` is the WHOLE queue (identical on every rank);
// stacks[s] may be NULL on ranks that do not own submap s.  Job j runs on rank
// submap_owner[jobs[j].stack_index] (NULL => stack_index % world_size).  On return every
// rank holds results[0 .. num_jobs) in job order.
csm_status csm_cb_batch2d_run(csm_ctx* ctx, const csm_stack2d* const* stacks, int32_t num_stacks,
                              const csm_cloud* const* clouds, int32_t num_clouds,
                              const csm_job2d* jobs, int32_t num_jobs,
                              const int32_t* submap_owner, double linear_window,
                              double angular_window, csm_result2d* results, csm_stats* stats) {
  CSM_REQUIRE(ctx && stacks && clouds && jobs && results, "null pointer");
  CSM_REQUIRE(num_jobs >= 0 && num_stacks >= 1 && num_clouds >= 1, "sizes");
  return ShardedQueue(
      ctx, jobs, num_jobs, num_stacks, submap_owner, results, stats,
      [](const csm_job2d& j) { return j.stack_index; }, "stack index",
      [&](int s) { return stacks[s] != nullptr; }, "an owned submap has no stack",
      [&](const csm_job2d* my_jobs, int32_t n, csm_result2d* my_results) {
        // the batch entry needs stacks[0] for its device: pass a dense view of owned stacks
        std::vector<const csm_stack2d*> dense(num_stacks, nullptr);
        const csm_stack2d* any = nullptr;
        for (int s = 0; s < num_stacks; ++s)
          if (stacks[s]) { dense[s] = stacks[s]; any = stacks[s]; }
        for (int s = 0; s < num_stacks; ++s)
          if (!dense[s]) dense[s] = any;  // never dereferenced: no local job points at it
        return csm_match2d_batch(dense.data(), num_stacks, clouds, num_clouds, my_jobs, n,
                                 linear_window, angular_window, my_results, stats);
      });
}

// The sharded 3D queue (constraint_builder_3d.cc:107-116): same ownership rule on
// matcher_index, same single allgather.
csm_status csm_cb_batch3d_run(csm_ctx* ctx, const csm_matcher3d* const* matchers,
                              int32_t num_matchers, const csm_node3d* nodes, int32_t num_nodes,
                              const csm_job3d* jobs, int32_t num_jobs,
                              const int32_t* submap_owner, int32_t max_concurrency,
                              csm_result3d* results, csm_stats* stats) {
  CSM_REQUIRE(ctx && matchers && nodes && jobs && results, "null pointer");
  CSM_REQUIRE(num_jobs >= 0 && num_matchers >= 1 && num_nodes >= 1, "sizes");
  return ShardedQueue(
      ctx, jobs, num_jobs, num_matchers, submap_owner, results, stats,
      [](const csm_job3d& j) { return j.matcher_index; }, "matcher index",
      [&](int m) { return matchers[m] != nullptr; }, "an owned submap has no matcher",
      [&](const csm_job3d* my_jobs, int32_t n, csm_result3d* my_results) {
        return csm_match3d_batch(matchers, num_matchers, nodes, num_nodes, my_jobs, n,
                                 max_concurrency, my_results, stats);
      });
}

}  // extern "C"
