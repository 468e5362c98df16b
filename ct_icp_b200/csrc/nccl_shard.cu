// nccl_shard.cu — keypoint-sharded multi-GPU mode (SURVEY §8e).
//
// One process per GPU. Every rank registers the same scan against its own replica of the map (sampling and map
// update are deterministic, so the replicas stay identical); the K keypoints of a frame are split into contiguous
// chunks [K r / G, K (r+1) / G) and each Gauss-Newton iteration performs ONE exchange: the sum over ranks of the
// 96-double accumulator (78 JTJ + 12 JTr + counters, 768 bytes) over NVLink/NVSwitch, after which every rank solves
// the same 12x12 system and applies the same pose update — no broadcast needed.
//
// The exchange is done by the ICP kernels themselves through peer-mapped mailboxes (peer_exchange.cuh; inside the
// persistent GN kernel, so the sharded GN loop is still ONE launch). This file sets the mailboxes up: NCCL is the
// bootstrap (all-gather of the CUDA IPC handles, agreement on whether every rank could map every peer) and the
// fallback (ncclAllReduce per exchange) when peer mapping is not available (no P2P between the devices, ranks on
// different nodes, CTICP_P2P=0).
//
// NCCL is bound at run time (dlopen "libnccl.so.2"): the process usually already holds torch's bundled NCCL, and a
// link-time dependency on the system copy would put two NCCL versions behind the same symbols.
#include <dlfcn.h>
#include <nccl.h>
#include <unistd.h>

#include <mutex>
#include <vector>

#include "engine.h"
#include "icp.h"

namespace cticp {

struct NcclError : std::runtime_error {
    using std::runtime_error::runtime_error;
};

namespace {
struct NcclApi {
    void *handle = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId *) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*AllReduce)(const void *, void *, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*AllGather)(const void *, void *, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
    const char *(*GetErrorString)(ncclResult_t) = nullptr;
};
NcclApi &Api() {
    static NcclApi api;
    static std::once_flag once;
    std::call_once(once, [] {
        const char *names[] = {"libnccl.so.2", "libnccl.so"};
        for (const char *n : names) {
            api.handle = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
            if (api.handle) break;
        }
        if (!api.handle) return;
        api.GetUniqueId = (decltype(api.GetUniqueId)) dlsym(api.handle, "ncclGetUniqueId");
        api.CommInitRank = (decltype(api.CommInitRank)) dlsym(api.handle, "ncclCommInitRank");
        api.CommDestroy = (decltype(api.CommDestroy)) dlsym(api.handle, "ncclCommDestroy");
        api.AllReduce = (decltype(api.AllReduce)) dlsym(api.handle, "ncclAllReduce");
        api.AllGather = (decltype(api.AllGather)) dlsym(api.handle, "ncclAllGather");
        api.GetErrorString = (decltype(api.GetErrorString)) dlsym(api.handle, "ncclGetErrorString");
    });
    if (!api.handle || !api.GetUniqueId || !api.CommInitRank || !api.AllReduce)
        throw NcclError("NCCL: libnccl.so.2 could not be loaded");
    return api;
}
void Check(ncclResult_t r, const char *what) {
    if (r != ncclSuccess) {
        const char *msg = Api().GetErrorString ? Api().GetErrorString(r) : "?";
        throw NcclError(std::string("NCCL: ") + what + ": " + msg);
    }
}
}  // namespace

void IcpSolver::NcclAllReduceAccumulator(void *nccl_comm) {
    Check(Api().AllReduce(d_acc_.data(), d_acc_.data(), kAcc, ncclDouble, ncclSum, (ncclComm_t) nccl_comm, stream_), "ncclAllReduce");
}

// ---- peer mailboxes ------------------------------------------------------------------------------------------
namespace {
constexpr size_t kMailboxBytes = sizeof(unsigned long long) * 2 * kMaxPeerRanks * 2 * kAcc;   // peer_exchange.cuh layout
struct PeerBlob {   // what every rank tells every other rank (all-gathered through NCCL)
    cudaIpcMemHandle_t handle;
    unsigned long long ptr;       // the mailbox address in the owner's process (used when owner == this process)
    unsigned long long host_tag;  // hash of the host name
    long long pid;
    int device;
    int ok;
};
// Mailboxes are never cudaFree'd while the process lives: a peer may still hold an IPC mapping of one when its owner
// tears its engine down (ranks destroy their handles at their own pace, and freeing exported memory before every
// importer closed it is undefined behaviour). A retired mailbox goes back to this per-device pool and is re-zeroed
// when the next engine of this process adopts it; the exchange protocol is symmetric, so once an owner has finished
// its last exchange no peer writes to its mailbox any more.
struct MailboxPool {
    std::mutex mu;
    std::vector<std::pair<int, void *>> free_list;   // (device, mailbox)
    void *Take(int device) {
        std::lock_guard<std::mutex> lk(mu);
        for (size_t i = 0; i < free_list.size(); ++i)
            if (free_list[i].first == device) {
                void *p = free_list[i].second;
                free_list.erase(free_list.begin() + (long) i);
                return p;
            }
        return nullptr;
    }
    void Give(int device, void *p) {
        std::lock_guard<std::mutex> lk(mu);
        free_list.emplace_back(device, p);
    }
};
MailboxPool &Pool() {
    static MailboxPool pool;
    return pool;
}

unsigned long long HostTag() {
    char name[256] = {0};
    gethostname(name, sizeof(name) - 1);
    unsigned long long h = 1469598103934665603ull;
    for (const char *c = name; *c; ++c) h = (h ^ (unsigned char) *c) * 1099511628211ull;
    return h;
}
}  // namespace

// Returns true when EVERY rank mapped EVERY peer's mailbox (the decision is all-reduced, so all ranks agree).
bool Engine::ConnectPeers() {
    const int world = shard_world_, rank = shard_rank_;
    NcclApi &api = Api();
    auto comm = (ncclComm_t) nccl_comm_;
    int my_ok = 1;
    if (const char *e = getenv("CTICP_P2P")) my_ok = atoi(e) != 0;
    if (world > kMaxPeerRanks || !api.AllGather) my_ok = 0;

    // own mailbox (+ the exchange counter behind it), zeroed before anybody can learn its address
    d_mailbox_ = Pool().Take(device_);
    if (!d_mailbox_ && cudaMalloc(&d_mailbox_, kMailboxBytes + 256) != cudaSuccess) {
        cudaGetLastError();
        d_mailbox_ = nullptr;
        my_ok = 0;
    }
    PeerBlob mine{};
    mine.ptr = (unsigned long long) d_mailbox_;
    mine.host_tag = HostTag();
    mine.pid = (long long) getpid();
    mine.device = device_;
    if (d_mailbox_) {
        if (cudaMemsetAsync(d_mailbox_, 0, kMailboxBytes + 256, stream_.get()) != cudaSuccess ||
            cudaStreamSynchronize(stream_.get()) != cudaSuccess)
            my_ok = 0;
        if (cudaIpcGetMemHandle(&mine.handle, d_mailbox_) != cudaSuccess) {
            cudaGetLastError();
            my_ok = 0;
        }
    }
    mine.ok = my_ok;

    // all-gather of the blobs (NCCL is only the bootstrap here)
    std::vector<PeerBlob> all((size_t) world);
    {
        DeviceArray<PeerBlob> d_all;
        d_all.reserve(world, stream_.get());
        cudaMemcpyAsync(d_all.data() + rank, &mine, sizeof(PeerBlob), cudaMemcpyHostToDevice, stream_.get());
        if (api.AllGather)
            Check(api.AllGather(d_all.data() + rank, d_all.data(), sizeof(PeerBlob), ncclChar, comm, stream_.get()), "ncclAllGather");
        cudaMemcpyAsync(all.data(), d_all.data(), sizeof(PeerBlob) * (size_t) world, cudaMemcpyDeviceToHost, stream_.get());
        if (cudaStreamSynchronize(stream_.get()) != cudaSuccess) throw CudaError("peer bootstrap: stream error");
    }

    PeerLinksHost links;
    links.world = world;
    links.rank = rank;
    for (int p = 0; p < world && my_ok; ++p) {
        if (!all[p].ok) {
            my_ok = 0;
            break;
        }
        if (p == rank) {
            links.inbox[p] = (unsigned long long *) d_mailbox_;
            continue;
        }
        if (all[p].host_tag != mine.host_tag) {   // another node: no load/store path
            my_ok = 0;
            break;
        }
        if (all[p].pid == mine.pid) {   // another engine of this process (one process driving several GPUs)
            if (all[p].device != device_) {
                int can = 0;
                cudaDeviceCanAccessPeer(&can, device_, all[p].device);
                if (!can) {
                    my_ok = 0;
                    break;
                }
                const cudaError_t e = cudaDeviceEnablePeerAccess(all[p].device, 0);
                if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) my_ok = 0;
                cudaGetLastError();
            }
            links.inbox[p] = (unsigned long long *) all[p].ptr;
        } else {
            void *mapped = nullptr;
            if (cudaIpcOpenMemHandle(&mapped, all[p].handle, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) {
                cudaGetLastError();
                my_ok = 0;
                break;
            }
            peer_mapped_.push_back(mapped);
            links.inbox[p] = (unsigned long long *) mapped;
        }
    }
    links.seq = d_mailbox_ ? (unsigned int *) ((char *) d_mailbox_ + kMailboxBytes) : nullptr;

    // agreement: min over ranks of my_ok (the flag serves the rendezvous below as well)
    int agreed = 0;
    DeviceArray<int> d_flag;
    d_flag.reserve(1, stream_.get());
    cudaMemcpyAsync(d_flag.data(), &my_ok, sizeof(int), cudaMemcpyHostToDevice, stream_.get());
    Check(api.AllReduce(d_flag.data(), d_flag.data(), 1, ncclInt, ncclMin, comm, stream_.get()), "ncclAllReduce (peer agreement)");
    cudaMemcpyAsync(&agreed, d_flag.data(), sizeof(int), cudaMemcpyDeviceToHost, stream_.get());
    if (cudaStreamSynchronize(stream_.get()) != cudaSuccess) throw CudaError("peer bootstrap: stream error");
    if (!agreed) {
        DisconnectPeers();
        return false;
    }
    {   // exchange time-out (see peer_exchange.cuh): CTICP_PEER_TIMEOUT_MS, default 30 s, in SM cycles
        double ms = 30000.0;
        if (const char *e = getenv("CTICP_PEER_TIMEOUT_MS")) ms = std::max(1.0, atof(e));
        int khz = 0;
        cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, device_);
        links.timeout_cycles = (long long) (ms * (double) std::max(khz, 1000000));
    }
    icp_->SetPeerLinks(links);
    // every rank loads the sharded kernels' modules NOW, then the ranks meet once more: the first exchange finds all peers
    // warm instead of one of them inside a lazy module load
    icp_->PreloadShardedKernels();
    cudaMemsetAsync(d_flag.data(), 0, sizeof(int), stream_.get());
    Check(api.AllReduce(d_flag.data(), d_flag.data(), 1, ncclInt, ncclMin, comm, stream_.get()), "ncclAllReduce (peer rendezvous)");
    cudaStreamSynchronize(stream_.get());
    if (getenv("CTICP_DEBUG_P2P"))
        fprintf(stderr, "[cticp] rank %d/%d: peer mailboxes connected (%zu IPC mappings)\n", rank, world, peer_mapped_.size());
    return true;
}

void Engine::DisconnectPeers() {
    if (icp_) icp_->SetPeerLinks(PeerLinksHost{});
    for (void *m : peer_mapped_) cudaIpcCloseMemHandle(m);
    peer_mapped_.clear();
    if (d_mailbox_) Pool().Give(device_, d_mailbox_);   // not freed: see MailboxPool
    d_mailbox_ = nullptr;
    cudaGetLastError();
}

void Engine::EnableSharding(const void *unique_id, int rank, int world) {
    if (!unique_id || world < 1 || rank < 0 || rank >= world) throw std::invalid_argument("EnableSharding arguments");
    if (cudaSetDevice(device_) != cudaSuccess) throw CudaError("cudaSetDevice");
    if (stream_.get()) cudaStreamSynchronize(stream_.get());
    DisconnectPeers();
    if (nccl_comm_) {
        Api().CommDestroy((ncclComm_t) nccl_comm_);
        nccl_comm_ = nullptr;
    }
    shard_rank_ = rank;
    shard_world_ = world;
    // every rank of the node runs its own host team: share the machine between them (one node assumed)
    if (HostTeamSize(world) != pool_->size()) pool_ = std::make_unique<HostPool>(HostTeamSize(world));
    if (world == 1) return;
    ncclUniqueId id;
    static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId is 128 bytes");
    memcpy(&id, unique_id, sizeof(id));
    ncclComm_t comm;
    Check(Api().CommInitRank(&comm, world, id, rank), "ncclCommInitRank");
    nccl_comm_ = comm;
    ConnectPeers();   // false: every exchange goes through ncclAllReduce instead
}

void Engine::DestroySharding() {
    DisconnectPeers();
    if (nccl_comm_) {
        try {
            Api().CommDestroy((ncclComm_t) nccl_comm_);
        } catch (...) {
        }
        nccl_comm_ = nullptr;
    }
}

}  // namespace cticp

extern "C" int cticp_nccl_unique_id(void *out_128_bytes) {
    try {
        ncclUniqueId id;
        cticp::Check(cticp::Api().GetUniqueId(&id), "ncclGetUniqueId");
        memcpy(out_128_bytes, &id, sizeof(id));
        return CTICP_OK;
    } catch (const std::exception &) {
        return CTICP_ERR_NCCL;
    }
}
