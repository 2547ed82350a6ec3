// nccl_loopback.cpp -- a test-only stand-in for the NCCL entry points that libconflux_b200.so calls, so that a P-rank
// grid runs as P threads of one process on ONE device.  Loaded with LD_PRELOAD ahead of the real libnccl.so.2; the
// product links NCCL dynamically with unversioned symbols, so these definitions win.
//
// Every call is synchronous and staged through host memory:
//   1. cuStreamSynchronize(stream): the input is final
//   2. the rank copies its input into its slot of the communicator, and the ranks meet (rendezvous 1); the last to
//      arrive checks that every rank issued the same operation (kind, count, type, op, root) as the same call number
//   3. each rank computes its own result from all slots in rank order (sums run rank 0, 1, ..., P-1) and writes it with
//      cuMemcpyHtoDAsync on the caller's stream, then cuStreamSynchronize
//   4. rendezvous 2, so no slot is overwritten by the next call while another rank still reads it
// Inside ncclGroupStart / ncclGroupEnd every operation is deferred; at the outermost ncclGroupEnd the sends are posted
// first, then the collectives run in issue order, then the receives complete (matched by communicator, peer and a
// per-pair sequence number, with count and type checked).
//
// A mismatched schedule gives every rank of that call ncclInvalidUsage and names both calls on stderr.  A rendezvous
// that waits longer than LOOPBACK_TIMEOUT_S seconds (default 120) names, per rank, the call it waits in, and fails.
// Either poisons the communicator: every later call on it fails at once instead of waiting.
//
// -DLOOPBACK_HOST_ONLY replaces the device copies and stream syncs with memcpy, so the CPU tests can drive the library
// through ctypes with host buffers.
#include <nccl.h>

#include <dlfcn.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <tuple>
#include <vector>

namespace {

// ---------------------------------------------------------------------------------------------------- call counters
enum Kind { K_INIT, K_SPLIT, K_ALLREDUCE, K_REDUCE, K_BROADCAST, K_ALLGATHER, K_SEND, K_RECV, K_GROUP, K_DESTROY, K_COUNT };
const char* const KIND_NAMES[K_COUNT] = {"ncclCommInitRank", "ncclCommSplit", "ncclAllReduce", "ncclReduce",
                                         "ncclBroadcast", "ncclAllGather", "ncclSend", "ncclRecv", "ncclGroupEnd",
                                         "ncclCommDestroy"};
std::atomic<unsigned long long> g_stats[K_COUNT];

void say(const char* fmt, ...) {
    char buf[2048];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    fprintf(stderr, "nccl_loopback: %s\n", buf);
    fflush(stderr);
}

const char* type_name(ncclDataType_t t) {
    switch (t) {
        case ncclInt: return "ncclInt";
        case ncclDouble: return "ncclDouble";
        case ncclUint64: return "ncclUint64";
        default: return "unsupported-type";
    }
}
size_t type_size(ncclDataType_t t) {
    switch (t) {
        case ncclInt: return 4;
        case ncclDouble: case ncclUint64: return 8;
        default: return 0;
    }
}
const char* op_name(int op) {
    switch (op) {
        case ncclSum: return "ncclSum";
        case ncclMax: return "ncclMax";
        case ncclMin: return "ncclMin";
        case -1: return "-";
        default: return "unsupported-op";
    }
}

// ------------------------------------------------------------------------------------------------- device access
#ifndef LOOPBACK_HOST_ONLY
typedef int CUresult_;
struct Driver {
    CUresult_ (*ctx_get_current)(void**) = nullptr;
    CUresult_ (*stream_sync)(void*) = nullptr;
    CUresult_ (*dtoh_async)(void*, unsigned long long, size_t, void*) = nullptr;
    CUresult_ (*htod_async)(unsigned long long, const void*, size_t, void*) = nullptr;
    CUresult_ (*err_string)(CUresult_, const char**) = nullptr;
    bool ok = false;
    Driver() {
        void* h = dlopen("libcuda.so.1", RTLD_NOW | RTLD_GLOBAL);
        if (!h) return;
        ctx_get_current = (decltype(ctx_get_current))dlsym(h, "cuCtxGetCurrent");
        stream_sync = (decltype(stream_sync))dlsym(h, "cuStreamSynchronize");
        dtoh_async = (decltype(dtoh_async))dlsym(h, "cuMemcpyDtoHAsync_v2");
        htod_async = (decltype(htod_async))dlsym(h, "cuMemcpyHtoDAsync_v2");
        err_string = (decltype(err_string))dlsym(h, "cuGetErrorString");
        ok = ctx_get_current && stream_sync && dtoh_async && htod_async && err_string;
    }
};
Driver& drv() {
    static Driver d;
    return d;
}
bool cu_ok(CUresult_ r, const char* what, const char* fn) {
    if (r == 0) return true;
    const char* s = "?";
    drv().err_string(r, &s);
    say("%s: %s failed: %s (%d)", fn, what, s, r);
    return false;
}
// the caller's thread must already have a context current (the product selects its device before every call)
bool have_context(const char* fn) {
    if (!drv().ok) {
        say("%s: libcuda.so.1 or one of its entry points could not be loaded", fn);
        return false;
    }
    void* ctx = nullptr;
    if (!cu_ok(drv().ctx_get_current(&ctx), "cuCtxGetCurrent", fn)) return false;
    if (!ctx) {
        say("%s: no CUDA context is current on this thread; the loopback does not create one", fn);
        return false;
    }
    return true;
}
bool sync_stream(cudaStream_t s, const char* fn) { return cu_ok(drv().stream_sync((void*)s), "cuStreamSynchronize", fn); }
bool to_host(void* dst, const void* src, size_t bytes, cudaStream_t s, const char* fn) {
    if (!bytes) return true;
    return cu_ok(drv().dtoh_async(dst, (unsigned long long)(uintptr_t)src, bytes, (void*)s), "cuMemcpyDtoHAsync", fn) &&
           sync_stream(s, fn);
}
bool to_device(void* dst, const void* src, size_t bytes, cudaStream_t s, const char* fn) {
    if (!bytes) return true;
    return cu_ok(drv().htod_async((unsigned long long)(uintptr_t)dst, src, bytes, (void*)s), "cuMemcpyHtoDAsync", fn) &&
           sync_stream(s, fn);
}
#else
bool have_context(const char*) { return true; }
bool sync_stream(cudaStream_t, const char*) { return true; }
bool to_host(void* dst, const void* src, size_t bytes, cudaStream_t, const char*) {
    if (bytes) std::memcpy(dst, src, bytes);
    return true;
}
bool to_device(void* dst, const void* src, size_t bytes, cudaStream_t, const char*) {
    if (bytes) std::memcpy(dst, src, bytes);
    return true;
}
#endif

double timeout_s() {
    const char* e = getenv("LOOPBACK_TIMEOUT_S");
    const double t = e ? atof(e) : 120.0;
    return t > 0 ? t : 120.0;
}

// ------------------------------------------------------------------------------------------------- communicators
// One operation as a rank issued it; the schedule check compares these field by field.
struct Call {
    int kind = -1;
    size_t count = 0;
    int dtype = -1;
    int op = -1;
    int root = -1;
    unsigned long long seq = 0;  // this rank's call number on the communicator
    std::string text() const {
        char b[256];
        snprintf(b, sizeof(b), "call #%llu %s(count=%zu, %s, %s, root=%d)", seq, kind >= 0 ? KIND_NAMES[kind] : "none",
                 count, dtype >= 0 ? type_name((ncclDataType_t)dtype) : "-", op_name(op), root);
        return b;
    }
    bool same(const Call& o) const {
        return kind == o.kind && count == o.count && dtype == o.dtype && op == o.op && root == o.root && seq == o.seq;
    }
};

struct Shared;
struct Slot {
    Call call;               // the call this rank is in (or last left)
    bool waiting = false;    // inside a rendezvous right now
    std::vector<char> data;  // staged input
    int color = 0, key = 0;  // ncclCommSplit arguments
    Shared* split_to = nullptr;
    int split_rank = -1;
};

// The state every rank of one communicator shares.
struct Shared {
    int n;
    int id;
    std::string name;
    std::mutex m;
    std::condition_variable cv;
    int arrived = 0;
    unsigned long long gen = 0;
    bool poisoned = false;
    bool round_bad = false;  // the schedule check of the current call failed
    std::vector<Slot> slots;
    int refs = 0;
    int joined = 0;  // ncclCommInitRank: ranks that have registered
    // point-to-point mailboxes: (src, dst, per-pair sequence) -> message
    struct Msg {
        size_t count;
        int dtype;
        std::vector<char> data;
    };
    std::map<std::tuple<int, int, unsigned long long>, Msg> mail;
    Shared(int n_, std::string nm) : n(n_), name(std::move(nm)), slots(n_) {
        static std::atomic<int> next{1};
        id = next++;
    }
};

}  // namespace

struct ncclComm {
    Shared* sh;
    int rank;
    unsigned long long seq = 0;                       // collective call number on this communicator
    std::vector<unsigned long long> sent, received;  // per-peer message counters
    ncclComm(Shared* s, int r) : sh(s), rank(r), sent(s->n, 0), received(s->n, 0) {}
};

namespace {

std::string state_of(Shared& s) {  // under s.m
    std::string out;
    for (int r = 0; r < s.n; ++r) {
        const Slot& sl = s.slots[r];
        out += "\n    rank " + std::to_string(r) + (sl.waiting ? " waits in " : " has not arrived; last ") + sl.call.text();
    }
    return out;
}

// Meets every rank of `s`.  The last rank to arrive runs `last()` under the lock (with every slot filled) before it
// releases the others.  Returns false on a timeout or a poisoned communicator.
template <class F>
bool rendezvous(Shared& s, int rank, const char* fn, F&& last) {
    std::unique_lock<std::mutex> lk(s.m);
    if (s.poisoned) {
        say("%s: communicator %s (id %d) is poisoned by an earlier failure; rank %d refused", fn, s.name.c_str(), s.id, rank);
        return false;
    }
    s.slots[rank].waiting = true;
    const unsigned long long g = s.gen;
    if (++s.arrived == s.n) {
        s.arrived = 0;
        last();
        for (Slot& sl : s.slots) sl.waiting = false;
        ++s.gen;
        s.cv.notify_all();
        return true;
    }
    const double t = timeout_s();
    const auto deadline = std::chrono::steady_clock::now() + std::chrono::duration<double>(t);
    while (s.gen == g && !s.poisoned) {
        if (s.cv.wait_until(lk, deadline) == std::cv_status::timeout && s.gen == g && !s.poisoned) {
            say("%s: timeout after %.0f s: rank %d of communicator %s (id %d, %d ranks) waits in %s; the ranks:%s", fn, t,
                rank, s.name.c_str(), s.id, s.n, s.slots[rank].call.text().c_str(), state_of(s).c_str());
            s.poisoned = true;
            s.cv.notify_all();
        }
    }
    s.slots[rank].waiting = false;
    return s.gen != g;
}

// rendezvous 1 of a data call: schedule check by the last arriver
bool meet_checked(ncclComm* c, const char* fn) {
    Shared& s = *c->sh;
    const bool ok = rendezvous(s, c->rank, fn, [&] {
        s.round_bad = false;
        for (int r = 1; r < s.n; ++r)
            if (!s.slots[r].call.same(s.slots[0].call)) {
                say("schedule mismatch on communicator %s (id %d): rank 0 issued %s, rank %d issued %s", s.name.c_str(),
                    s.id, s.slots[0].call.text().c_str(), r, s.slots[r].call.text().c_str());
                s.round_bad = true;
            }
        if (s.round_bad) s.poisoned = true;
    });
    if (!ok) return false;
    std::lock_guard<std::mutex> lk(s.m);
    return !s.round_bad;
}

bool check_comm(ncclComm* c, const char* fn) {
    if (!c || !c->sh) {
        say("%s: NULL communicator", fn);
        return false;
    }
    return true;
}

template <class T>
void reduce_into(T* acc, const T* x, size_t n, int op) {
    for (size_t i = 0; i < n; ++i) {
        if (op == ncclSum) acc[i] = acc[i] + x[i];
        else if (op == ncclMax) acc[i] = x[i] > acc[i] ? x[i] : acc[i];
        else acc[i] = x[i] < acc[i] ? x[i] : acc[i];
    }
}
// rank-order reduction of every slot into out (int32 sums wrap like the uint64 ones: they run on the unsigned type)
void reduce_slots(Shared& s, std::vector<char>& out, size_t count, ncclDataType_t t, int op) {
    out = s.slots[0].data;
    for (int r = 1; r < s.n; ++r) {
        const char* x = s.slots[r].data.data();
        switch (t) {
            case ncclDouble: reduce_into((double*)out.data(), (const double*)x, count, op); break;
            case ncclUint64: reduce_into((uint64_t*)out.data(), (const uint64_t*)x, count, op); break;
            default:
                if (op == ncclSum) reduce_into((uint32_t*)out.data(), (const uint32_t*)x, count, op);
                else reduce_into((int32_t*)out.data(), (const int32_t*)x, count, op);
        }
    }
}

bool args_ok(const char* fn, ncclDataType_t t, int op, int root, int n) {
    if (!type_size(t)) {
        say("%s: refused: datatype %d is not one of ncclInt, ncclDouble, ncclUint64", fn, (int)t);
        return false;
    }
    if (op != -1 && op != ncclSum && op != ncclMax && op != ncclMin) {
        say("%s: refused: reduction op %d is not one of ncclSum, ncclMax, ncclMin", fn, op);
        return false;
    }
    if (root != -1 && (root < 0 || root >= n)) {
        say("%s: refused: root %d outside a communicator of %d ranks", fn, root, n);
        return false;
    }
    return true;
}

// ---------------------------------------------------------------------------------------------- deferred operations
struct Op {
    int kind;
    const void* send;
    void* recv;
    size_t count;
    ncclDataType_t dtype;
    int op, root, peer;
    ncclComm* comm;
    cudaStream_t stream;
};
thread_local int t_group_depth = 0;
thread_local std::vector<Op> t_group;
thread_local bool t_group_failed = false;

// one collective, run to completion
ncclResult_t run_collective(const Op& o) {
    const char* fn = KIND_NAMES[o.kind];
    ncclComm* c = o.comm;
    Shared& s = *c->sh;
    const size_t es = type_size(o.dtype);
    if (!have_context(fn) || !sync_stream(o.stream, fn)) return ncclUnhandledCudaError;
    Call call;
    call.kind = o.kind;
    call.count = o.count;
    call.dtype = o.dtype;
    call.op = o.op;
    call.root = o.root;
    call.seq = c->seq++;
    std::vector<char> in;
    const bool stage = o.kind != K_BROADCAST || c->rank == o.root;
    if (stage) {
        in.resize(o.count * es);
        if (!to_host(in.data(), o.send, in.size(), o.stream, fn)) return ncclUnhandledCudaError;
    }
    {
        std::lock_guard<std::mutex> lk(s.m);
        s.slots[c->rank].call = call;
        s.slots[c->rank].data.swap(in);
    }
    g_stats[o.kind]++;
    if (!meet_checked(c, fn)) return ncclInvalidUsage;  // the communicator is poisoned: nobody stages into it again
    std::vector<char> out;
    void* dst = o.recv;
    bool write = true;
    switch (o.kind) {
        case K_ALLREDUCE: reduce_slots(s, out, o.count, o.dtype, o.op); break;
        case K_REDUCE:
            write = c->rank == o.root;
            if (write) reduce_slots(s, out, o.count, o.dtype, o.op);
            break;
        case K_BROADCAST: out = s.slots[o.root].data; break;
        case K_ALLGATHER:
            out.resize((size_t)s.n * o.count * es);
            for (int r = 0; r < s.n; ++r) std::memcpy(out.data() + (size_t)r * o.count * es, s.slots[r].data.data(), o.count * es);
            break;
    }
    const bool copied = !write || to_device(dst, out.data(), out.size(), o.stream, fn);
    if (!rendezvous(s, c->rank, fn, [] {})) return ncclInvalidUsage;
    return copied ? ncclSuccess : ncclUnhandledCudaError;
}

ncclResult_t post_send(const Op& o) {
    const char* fn = "ncclSend";
    ncclComm* c = o.comm;
    Shared& s = *c->sh;
    if (!have_context(fn) || !sync_stream(o.stream, fn)) return ncclUnhandledCudaError;
    Shared::Msg msg{o.count, (int)o.dtype, std::vector<char>(o.count * type_size(o.dtype))};
    if (!to_host(msg.data.data(), o.send, msg.data.size(), o.stream, fn)) return ncclUnhandledCudaError;
    g_stats[K_SEND]++;
    std::lock_guard<std::mutex> lk(s.m);
    s.mail[std::make_tuple(c->rank, o.peer, c->sent[o.peer]++)] = std::move(msg);
    s.cv.notify_all();
    return ncclSuccess;
}

ncclResult_t complete_recv(const Op& o) {
    const char* fn = "ncclRecv";
    ncclComm* c = o.comm;
    Shared& s = *c->sh;
    if (!have_context(fn) || !sync_stream(o.stream, fn)) return ncclUnhandledCudaError;
    const unsigned long long q = c->received[o.peer]++;
    const auto key = std::make_tuple(o.peer, c->rank, q);
    Shared::Msg msg;
    {
        std::unique_lock<std::mutex> lk(s.m);
        const double t = timeout_s();
        const auto deadline = std::chrono::steady_clock::now() + std::chrono::duration<double>(t);
        while (!s.mail.count(key)) {
            if (s.poisoned) {
                say("%s: communicator %s (id %d) is poisoned; rank %d refused", fn, s.name.c_str(), s.id, c->rank);
                return ncclInvalidUsage;
            }
            if (s.cv.wait_until(lk, deadline) == std::cv_status::timeout && !s.mail.count(key)) {
                say("%s: timeout after %.0f s: rank %d of communicator %s (id %d) waits for message #%llu from rank %d "
                    "(count=%zu, %s)", fn, t, c->rank, s.name.c_str(), s.id, q, o.peer, o.count, type_name(o.dtype));
                s.poisoned = true;
                s.cv.notify_all();
                return ncclInvalidUsage;
            }
        }
        msg = std::move(s.mail[key]);
        s.mail.erase(key);
    }
    g_stats[K_RECV]++;
    if (msg.count != o.count || msg.dtype != (int)o.dtype) {
        say("%s: message #%llu from rank %d to rank %d on communicator %s (id %d): sent count=%zu %s, received as "
            "count=%zu %s", fn, q, o.peer, c->rank, s.name.c_str(), s.id, msg.count, type_name((ncclDataType_t)msg.dtype),
            o.count, type_name(o.dtype));
        return ncclInvalidUsage;
    }
    return to_device(o.recv, msg.data.data(), msg.data.size(), o.stream, fn) ? ncclSuccess : ncclUnhandledCudaError;
}

ncclResult_t run_now(const Op& o) {
    switch (o.kind) {
        case K_SEND: return post_send(o);
        case K_RECV: return complete_recv(o);
        default: return run_collective(o);
    }
}

ncclResult_t submit(const Op& o) {
    if (t_group_depth > 0) {
        t_group.push_back(o);
        return ncclSuccess;
    }
    return run_now(o);
}

ncclResult_t data_call(int kind, const void* send, void* recv, size_t count, ncclDataType_t t, int op, int root, int peer,
                       ncclComm_t comm, cudaStream_t stream) {
    const char* fn = KIND_NAMES[kind];
    if (!check_comm(comm, fn)) return ncclInvalidArgument;
    if (!args_ok(fn, t, op, root, comm->sh->n)) return ncclInvalidArgument;
    if (peer != -1 && (peer < 0 || peer >= comm->sh->n || peer == comm->rank)) {
        say("%s: refused: peer %d on a communicator of %d ranks (caller is rank %d)", fn, peer, comm->sh->n, comm->rank);
        return ncclInvalidArgument;
    }
    return submit(Op{kind, send, recv, count, t, op, root, peer, comm, stream});
}

// --------------------------------------------------------------------------------------------- unique-id registry
std::mutex g_reg_m;
std::map<std::string, Shared*> g_registry;
const char ID_MAGIC[8] = {'l', 'o', 'o', 'p', 'b', 'a', 'c', 'k'};

ncclResult_t refuse_entry(const char* fn) {
    say("%s is not implemented by the loopback: refused", fn);
    return ncclInvalidUsage;
}

}  // namespace

extern "C" {

// ------------------------------------------------------------------------------------------------------- exported
__attribute__((visibility("default"))) int loopback_stats(unsigned long long* out, int n) {
    for (int k = 0; k < n && k < K_COUNT; ++k) out[k] = g_stats[k].load();
    return K_COUNT;
}
__attribute__((visibility("default"))) const char* loopback_stat_name(int k) {
    return (k >= 0 && k < K_COUNT) ? KIND_NAMES[k] : nullptr;
}

const char* ncclGetErrorString(ncclResult_t r) {
    switch (r) {
        case ncclSuccess: return "no error (loopback)";
        case ncclUnhandledCudaError: return "unhandled cuda error (loopback)";
        case ncclSystemError: return "unhandled system error (loopback)";
        case ncclInternalError: return "internal error (loopback)";
        case ncclInvalidArgument: return "invalid argument (loopback)";
        case ncclInvalidUsage: return "invalid usage (loopback; see stderr)";
        default: return "unknown result (loopback)";
    }
}

ncclResult_t ncclGetUniqueId(ncclUniqueId* id) {
    static std::atomic<unsigned long long> next{1};
    std::memset(id, 0, sizeof(*id));
    std::memcpy(id->internal, ID_MAGIC, sizeof(ID_MAGIC));
    const unsigned long long v = next++;
    std::memcpy(id->internal + sizeof(ID_MAGIC), &v, sizeof(v));
    return ncclSuccess;
}

ncclResult_t ncclCommInitRank(ncclComm_t* comm, int nranks, ncclUniqueId id, int rank) {
    const char* fn = "ncclCommInitRank";
    if (!comm || nranks < 1 || rank < 0 || rank >= nranks) {
        say("%s: refused: nranks=%d rank=%d", fn, nranks, rank);
        return ncclInvalidArgument;
    }
    if (std::memcmp(id.internal, ID_MAGIC, sizeof(ID_MAGIC)) != 0) {
        say("%s: refused: the unique id was not made by the loopback's ncclGetUniqueId", fn);
        return ncclInvalidArgument;
    }
    const std::string key(id.internal, 16);
    Shared* s;
    {
        std::lock_guard<std::mutex> lk(g_reg_m);
        auto it = g_registry.find(key);
        if (it == g_registry.end()) {
            unsigned long long v;
            std::memcpy(&v, id.internal + sizeof(ID_MAGIC), sizeof(v));
            s = new Shared(nranks, "world#" + std::to_string(v));
            g_registry[key] = s;
        } else {
            s = it->second;
        }
    }
    {
        std::lock_guard<std::mutex> lk(s->m);
        if (s->n != nranks) {
            say("%s: refused: rank %d says %d ranks, the communicator was created with %d", fn, rank, nranks, s->n);
            return ncclInvalidArgument;
        }
        s->refs++;
        s->slots[rank].call = Call{K_INIT, 0, -1, -1, -1, 0};
    }
    g_stats[K_INIT]++;
    if (!rendezvous(*s, rank, fn, [&] {
            std::lock_guard<std::mutex> lk(g_reg_m);
            g_registry.erase(key);
        }))
        return ncclSystemError;
    *comm = new ncclComm(s, rank);
    return ncclSuccess;
}

ncclResult_t ncclCommSplit(ncclComm_t comm, int color, int key, ncclComm_t* newcomm, ncclConfig_t* config) {
    const char* fn = "ncclCommSplit";
    (void)config;
    if (!check_comm(comm, fn) || !newcomm) return ncclInvalidArgument;
    if (t_group_depth > 0) return refuse_entry("ncclCommSplit inside a group");
    if (color < 0 && color != NCCL_SPLIT_NOCOLOR) {
        say("%s: refused: colour %d", fn, color);
        return ncclInvalidArgument;
    }
    Shared& s = *comm->sh;
    {
        std::lock_guard<std::mutex> lk(s.m);
        Slot& sl = s.slots[comm->rank];
        sl.call = Call{K_SPLIT, 0, -1, -1, -1, comm->seq++};
        sl.color = color;
        sl.key = key;
        sl.split_to = nullptr;
        sl.split_rank = -1;
    }
    g_stats[K_SPLIT]++;
    if (!meet_checked(comm, fn)) return ncclInvalidUsage;
    // the first rank of each colour (in parent order) builds the colour's communicator: members ordered by key, ties by
    // parent rank.  Done under the lock, once, by whoever gets there first.
    {
        std::lock_guard<std::mutex> lk(s.m);
        Slot& me = s.slots[comm->rank];
        if (color != NCCL_SPLIT_NOCOLOR && !me.split_to) {
            std::vector<int> members;
            for (int r = 0; r < s.n; ++r)
                if (s.slots[r].color == color) members.push_back(r);
            std::stable_sort(members.begin(), members.end(),
                             [&](int a, int b) { return s.slots[a].key < s.slots[b].key; });
            Shared* ns = new Shared((int)members.size(), s.name + "/split(colour " + std::to_string(color) + ")");
            ns->refs = (int)members.size();
            for (int i = 0; i < (int)members.size(); ++i) {
                s.slots[members[i]].split_to = ns;
                s.slots[members[i]].split_rank = i;
            }
        }
        *newcomm = color == NCCL_SPLIT_NOCOLOR ? nullptr : new ncclComm(me.split_to, me.split_rank);
    }
    if (!rendezvous(s, comm->rank, fn, [] {})) return ncclSystemError;
    return ncclSuccess;
}

ncclResult_t ncclCommCount(const ncclComm_t comm, int* count) {
    if (!check_comm(comm, "ncclCommCount")) return ncclInvalidArgument;
    *count = comm->sh->n;
    return ncclSuccess;
}
ncclResult_t ncclCommUserRank(const ncclComm_t comm, int* rank) {
    if (!check_comm(comm, "ncclCommUserRank")) return ncclInvalidArgument;
    *rank = comm->rank;
    return ncclSuccess;
}
ncclResult_t ncclCommDestroy(ncclComm_t comm) {
    if (!comm) return ncclSuccess;
    g_stats[K_DESTROY]++;
    Shared* s = comm->sh;
    bool last;
    {
        std::lock_guard<std::mutex> lk(s->m);
        last = --s->refs == 0;
    }
    delete comm;
    if (last) delete s;
    return ncclSuccess;
}

ncclResult_t ncclGroupStart() {
    if (t_group_depth++ == 0) {
        t_group.clear();
        t_group_failed = false;
    }
    return ncclSuccess;
}
ncclResult_t ncclGroupEnd() {
    if (t_group_depth == 0) {
        say("ncclGroupEnd: refused: no group is open");
        return ncclInvalidUsage;
    }
    if (--t_group_depth > 0) return ncclSuccess;
    g_stats[K_GROUP]++;
    std::vector<Op> ops;
    ops.swap(t_group);
    ncclResult_t rc = ncclSuccess;
    for (const Op& o : ops)  // sends first: nobody waits on a message posted later in its own group
        if (o.kind == K_SEND && rc == ncclSuccess) rc = post_send(o);
    for (const Op& o : ops)
        if (o.kind != K_SEND && o.kind != K_RECV && rc == ncclSuccess) rc = run_collective(o);
    for (const Op& o : ops)
        if (o.kind == K_RECV && rc == ncclSuccess) rc = complete_recv(o);
    return rc;
}

ncclResult_t ncclSend(const void* sendbuff, size_t count, ncclDataType_t datatype, int peer, ncclComm_t comm,
                      cudaStream_t stream) {
    return data_call(K_SEND, sendbuff, nullptr, count, datatype, -1, -1, peer, comm, stream);
}
ncclResult_t ncclRecv(void* recvbuff, size_t count, ncclDataType_t datatype, int peer, ncclComm_t comm,
                      cudaStream_t stream) {
    return data_call(K_RECV, nullptr, recvbuff, count, datatype, -1, -1, peer, comm, stream);
}
ncclResult_t ncclAllReduce(const void* sendbuff, void* recvbuff, size_t count, ncclDataType_t datatype, ncclRedOp_t op,
                           ncclComm_t comm, cudaStream_t stream) {
    return data_call(K_ALLREDUCE, sendbuff, recvbuff, count, datatype, (int)op, -1, -1, comm, stream);
}
ncclResult_t ncclReduce(const void* sendbuff, void* recvbuff, size_t count, ncclDataType_t datatype, ncclRedOp_t op,
                        int root, ncclComm_t comm, cudaStream_t stream) {
    return data_call(K_REDUCE, sendbuff, recvbuff, count, datatype, (int)op, root, -1, comm, stream);
}
ncclResult_t ncclBroadcast(const void* sendbuff, void* recvbuff, size_t count, ncclDataType_t datatype, int root,
                           ncclComm_t comm, cudaStream_t stream) {
    return data_call(K_BROADCAST, sendbuff, recvbuff, count, datatype, -1, root, -1, comm, stream);
}
ncclResult_t ncclAllGather(const void* sendbuff, void* recvbuff, size_t sendcount, ncclDataType_t datatype,
                           ncclComm_t comm, cudaStream_t stream) {
    return data_call(K_ALLGATHER, sendbuff, recvbuff, sendcount, datatype, -1, -1, -1, comm, stream);
}

// The rest of the communicator API: a product change that starts calling one of these must fail by name rather than
// reach the real library with a loopback communicator.
ncclResult_t ncclBcast(void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) { return refuse_entry("ncclBcast"); }
ncclResult_t ncclReduceScatter(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) {
    return refuse_entry("ncclReduceScatter");
}
ncclResult_t ncclCommInitAll(ncclComm_t*, int, const int*) { return refuse_entry("ncclCommInitAll"); }
ncclResult_t ncclCommInitRankConfig(ncclComm_t*, int, ncclUniqueId, int, ncclConfig_t*) {
    return refuse_entry("ncclCommInitRankConfig");
}
ncclResult_t ncclCommFinalize(ncclComm_t) { return refuse_entry("ncclCommFinalize"); }
ncclResult_t ncclCommAbort(ncclComm_t) { return refuse_entry("ncclCommAbort"); }
ncclResult_t ncclCommGetAsyncError(ncclComm_t, ncclResult_t*) { return refuse_entry("ncclCommGetAsyncError"); }
ncclResult_t ncclCommCuDevice(const ncclComm_t, int*) { return refuse_entry("ncclCommCuDevice"); }

}  // extern "C"
