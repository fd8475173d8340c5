// b200gbm engine implementation: network bootstrap, dataset ingestion/binning, GBDT driver and the
// device-resident leaf-wise tree learner.  See engine.h / kernels.cuh / hist_kernel.cuh.
#include "engine.h"
#include "objective.h"
#include "renew_kernel.cuh"
#include "metrics.h"
#include "predictor.h"

#include <nvtx3/nvToolsExt.h>      // header-only NVTX v3: ranges are no-ops unless a profiler injects itself

#include <arpa/inet.h>
#include <netdb.h>
#include <netinet/in.h>
#include <netinet/tcp.h>
#include <sys/select.h>
#include <sys/socket.h>
#include <unistd.h>
#include <sys/types.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <functional>
#include <random>
#include <mutex>
#include <omp.h>
#include <cstring>
#include <numeric>
#include <thread>

namespace b200gbm {

// NVTX ranges named after the kernel / collective numbering of SURVEY.md §2.5 (K1..K9, C1..C5): `nsys`/`ncu --nvtx` can filter on them
struct NvtxRange {
  explicit NvtxRange(const char* name) { nvtxRangePushA(name); }
  ~NvtxRange() { nvtxRangePop(); }
};

// Device time of the work enqueued on `stream` between construction and Ms() (CUDA events).  The events are destroyed on every
// way out of the scope, a throw included.
class StreamTimer {
 public:
  explicit StreamTimer(cudaStream_t stream) : stream_(stream) {
    B200_CUDA(cudaEventCreate(&start_.e)); B200_CUDA(cudaEventCreate(&stop_.e));
    B200_CUDA(cudaEventRecord(start_.e, stream_));
  }
  StreamTimer(const StreamTimer&) = delete;
  StreamTimer& operator=(const StreamTimer&) = delete;
  float Ms() {
    B200_CUDA(cudaEventRecord(stop_.e, stream_));
    B200_CUDA(cudaEventSynchronize(stop_.e));
    float ms = 0;
    B200_CUDA(cudaEventElapsedTime(&ms, start_.e, stop_.e));
    return ms;
  }

 private:
  struct Event {      // a member, so that an event made before a throw in the constructor is destroyed too
    cudaEvent_t e = nullptr;
    ~Event() { if (e) cudaEventDestroy(e); }
  };
  cudaStream_t stream_;
  Event start_, stop_;
};

// =============================================================================== device / network
static thread_local int t_device = -1;
static thread_local Network t_net;
Network& Net() { return t_net; }

// Host-side OpenMP loops (bin finding on the sample, batch predict) must respect the container's CPU
// quota: a container may show many more logical CPUs than its cgroup quota allows, and oversubscribed
// OpenMP teams are then far slower.
static void CapHostThreadsOnce() {
  static std::once_flag once;
  std::call_once(once, [] {
    int n = omp_get_max_threads();
    FILE* f = std::fopen("/sys/fs/cgroup/cpu.max", "r");
    if (f) {
      char q[64] = {0};
      long long period = 0;
      if (std::fscanf(f, "%63s %lld", q, &period) == 2 && std::strcmp(q, "max") != 0 && period > 0) {
        long long quota = std::atoll(q);
        n = static_cast<int>(std::max<long long>(1, std::min<long long>(n, quota / period)));
      }
      std::fclose(f);
    }
    omp_set_num_threads(n);
  });
}

static int DeviceCountOrDie() {
  CapHostThreadsOnce();
  int cnt = 0;
  cudaError_t e = cudaGetDeviceCount(&cnt);
  if (e != cudaSuccess || cnt <= 0)
    Fatal(std::string("b200gbm: no CUDA device available (") + cudaGetErrorString(e) +
          "). This engine is CUDA-only (sm_90a); there is no CPU fallback.");
  return cnt;
}
int CurrentDevice() {
  if (t_device < 0) {
    int cnt = DeviceCountOrDie();
    const char* lr = std::getenv("LOCAL_RANK");
    t_device = (lr ? std::atoi(lr) : 0) % cnt;
  }
  return t_device;
}
void SetThreadDevice(int ordinal) {
  int cnt = DeviceCountOrDie();
  if (ordinal < 0 || ordinal >= cnt) Fatal("b200gbm: device ordinal out of range");
  t_device = ordinal;
}
void EnsureDevice() { B200_CUDA(cudaSetDevice(CurrentDevice())); }
int DeviceSMs() {
  int sms = 0;
  B200_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, CurrentDevice()));
  return sms;
}

static void SendAll(int fd, const void* buf, size_t n) {
  const char* p = static_cast<const char*>(buf);
  while (n) { ssize_t k = ::send(fd, p, n, 0); if (k <= 0) Fatal("network bootstrap: send failed"); p += k; n -= k; }
}
static void RecvAll(int fd, void* buf, size_t n) {
  char* p = static_cast<char*>(buf);
  while (n) { ssize_t k = ::recv(fd, p, n, 0); if (k <= 0) Fatal("network bootstrap: recv failed"); p += k; n -= k; }
}

// ---- same-device communicator
// Rank-threads of one process that share one CUDA device (numTasks above the GPU count, the reference's local mode) cannot use NCCL, which
// refuses two ranks on one device.  They meet in one SameDeviceComm: a collective posts each rank's device pointer into its slot, and the
// last rank to arrive enqueues the whole collective on the device's shared stream (AcquireStream), then releases the others.  Every rank
// enqueued its earlier work on that stream before arriving, and its later work after being released, so stream order is the only
// synchronisation the device needs; no kernel ever waits on another rank.
struct SameDeviceComm {
  int world = 0;
  cudaStream_t stream = nullptr;
  std::chrono::seconds timeout{120};      // NetworkInit's listen_time_out bounds every wait
  std::mutex mu;
  std::condition_variable cv;
  unsigned long long generation = 0;      // completed collectives
  int arrived = 0;
  int left = -1;                          // the first rank that left the network (LGBM_NetworkFree, a timeout or a failed collective)
  void* buf[kMaxPeers] = {};
  const void* src[kMaxPeers] = {};
  size_t bytes[kMaxPeers] = {};
};

static std::string LeftMessage(int r) {
  return "rank " + std::to_string(r) + " left the network: the same-device collective cannot complete";
}

// The rendezvous of one collective.  The last rank to arrive checks that every rank passed the same size, runs enqueue() under the lock and
// advances the generation; the others wait for that, for a rank leaving, or for the timeout.  A failure marks this rank as left, so that
// no rank waits for it.
template <typename Enqueue>
static void Rendezvous(SameDeviceComm& c, int me, void* buf, const void* src, size_t bytes, Enqueue enqueue) {
  std::unique_lock<std::mutex> lk(c.mu);
  if (c.left >= 0) Fatal(LeftMessage(c.left));
  c.buf[me] = buf; c.src[me] = src; c.bytes[me] = bytes;
  const unsigned long long gen = c.generation;
  if (++c.arrived == c.world) {
    std::string err;
    for (int r = 0; r < c.world; ++r)
      if (c.bytes[r] != bytes) err = "same-device collective: rank " + std::to_string(r) + " passed " + std::to_string(c.bytes[r]) + " bytes, rank " + std::to_string(me) + " " + std::to_string(bytes);
    if (err.empty()) {
      try { enqueue(); } catch (const std::exception& e) { err = e.what(); }
    }
    if (!err.empty()) { c.left = me; c.cv.notify_all(); Fatal(err); }
    c.arrived = 0;
    ++c.generation;
    c.cv.notify_all();
    return;
  }
  const bool woke = c.cv.wait_for(lk, c.timeout, [&] { return c.generation != gen || c.left >= 0; });
  if (c.generation != gen) return;      // completed, even if a rank left afterwards
  if (!woke) {
    c.left = me; c.cv.notify_all();
    Fatal("rank " + std::to_string(me) + ": a same-device collective timed out after " + std::to_string(c.timeout.count()) + " s waiting for the other ranks");
  }
  Fatal(LeftMessage(c.left));
}

static void LaunchAllReduceSameDevice(void* const* bufs, int R, size_t count, ncclDataType_t type, ncclRedOp_t op, cudaStream_t s) {
  SameDevicePtrs t{};
  int vec = 1;
  for (int r = 0; r < R; ++r) { t.p[r] = bufs[r]; vec &= (reinterpret_cast<uintptr_t>(bufs[r]) & 15) == 0 ? 1 : 0; }
  int sms = 0;
  B200_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, CurrentDevice()));
  const size_t esz = type == ncclUint32 ? 4 : 8;
  const size_t work = std::max<size_t>(1, count / (16 / esz) + 16 / esz);      // vectors plus the scalar tail
  const unsigned grid = static_cast<unsigned>(std::min<size_t>((work + 255) / 256, static_cast<size_t>(sms) * 16));
  const long long n = static_cast<long long>(count);
  if (type == ncclDouble && op == ncclSum) k_allreduce_same_device<double, RedSum<double>><<<grid, 256, 0, s>>>(t, R, n, vec);
  else if (type == ncclDouble && op == ncclMax) k_allreduce_same_device<double, RedMax<double>><<<grid, 256, 0, s>>>(t, R, n, vec);
  else if (type == ncclDouble && op == ncclMin) k_allreduce_same_device<double, RedMin<double>><<<grid, 256, 0, s>>>(t, R, n, vec);
  else if (type == ncclInt64 && op == ncclSum) k_allreduce_same_device<long long, RedSum<long long>><<<grid, 256, 0, s>>>(t, R, n, vec);
  else if (type == ncclUint32 && op == ncclMax) k_allreduce_same_device<unsigned, RedMax<unsigned>><<<grid, 256, 0, s>>>(t, R, n, vec);
  else Fatal("same-device all-reduce: unsupported type / operation");
  B200_CUDA(cudaGetLastError());
}

void Network::AllReduce(void* buf, size_t count, ncclDataType_t type, ncclRedOp_t op, cudaStream_t s) const {
  if (!active) Fatal("collective called without an initialised network (LGBM_NetworkInit)");
  if (!same_device) { B200_NCCL(ncclAllReduce(buf, buf, count, type, op, comm, s)); return; }
  SameDeviceComm& c = *same_device;
  if (s != c.stream) Fatal("same-device collective on a stream other than the device's shared stream");
  const size_t esz = type == ncclUint32 ? 4 : 8;
  Rendezvous(c, rank, buf, nullptr, count * esz, [&] { LaunchAllReduceSameDevice(c.buf, c.world, count, type, op, s); });
}

void Network::AllGather(const void* send, void* recv, size_t bytes, cudaStream_t s) const {
  if (!active) Fatal("collective called without an initialised network (LGBM_NetworkInit)");
  if (!same_device) { B200_NCCL(ncclAllGather(send, recv, bytes, ncclChar, comm, s)); return; }
  SameDeviceComm& c = *same_device;
  if (s != c.stream) Fatal("same-device collective on a stream other than the device's shared stream");
  Rendezvous(c, rank, recv, send, bytes, [&] {      // every send into rank 0's recv, then rank 0's recv into the others'
    char* r0 = static_cast<char*>(c.buf[0]);
    for (int r = 0; r < c.world; ++r) B200_CUDA(cudaMemcpyAsync(r0 + r * bytes, c.src[r], bytes, cudaMemcpyDeviceToDevice, s));
    for (int r = 1; r < c.world; ++r) B200_CUDA(cudaMemcpyAsync(c.buf[r], r0, bytes * c.world, cudaMemcpyDeviceToDevice, s));
  });
}

// one non-blocking stream per device for every rank-thread of a same-device network; never destroyed
static std::mutex g_shared_streams_mu;
static std::map<int, cudaStream_t> g_shared_streams;
static cudaStream_t SharedStream(int device) {
  std::lock_guard<std::mutex> lk(g_shared_streams_mu);
  cudaStream_t& s = g_shared_streams[device];
  if (!s) B200_CUDA(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
  return s;
}
cudaStream_t AcquireStream() {
  if (t_net.active && t_net.same_device) return t_net.same_device->stream;
  cudaStream_t s = nullptr;
  B200_CUDA(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
  return s;
}
void ReleaseStream(cudaStream_t s) {
  if (!s) return;
  {
    std::lock_guard<std::mutex> lk(g_shared_streams_mu);
    for (auto& kv : g_shared_streams) if (kv.second == s) return;
  }
  cudaStreamDestroy(s);
}

// same-device communicators between NetworkInit's rank 0 creating one and every other rank attaching to it
static std::mutex g_comm_registry_mu;
static std::map<std::pair<unsigned long long, unsigned long long>, std::shared_ptr<SameDeviceComm>> g_comm_registry;      // (token, sequence)

// A random token of this process, made once when the library loads: it tells rank 0 which ranks are threads of one process (a pid alone
// does not, pids repeat across containers).
static const unsigned long long g_process_token = [] {
  std::random_device rd;
  return (static_cast<unsigned long long>(rd()) << 32) ^ rd() ^ static_cast<unsigned long long>(std::chrono::steady_clock::now().time_since_epoch().count());
}();
static std::atomic<unsigned long long> g_comm_sequence{0};

// what every rank reports to rank 0, and rank 0's decision
struct RankHello { unsigned long long token; unsigned char uuid[16]; };
enum : int { kLayoutNccl = 0, kLayoutSameDevice = 1, kLayoutRejected = 2 };
struct LayoutDecision { int layout; unsigned long long sequence; ncclUniqueId id; char message[1024]; };

static std::string UuidString(const unsigned char* u) {
  char b[48];
  std::snprintf(b, sizeof(b), "GPU-%02x%02x%02x%02x-%02x%02x-%02x%02x-%02x%02x-%02x%02x%02x%02x%02x%02x", u[0], u[1], u[2], u[3], u[4], u[5], u[6], u[7], u[8],
                u[9], u[10], u[11], u[12], u[13], u[14], u[15]);
  return b;
}

// Rank 0's choice from every rank's process token and device UUID: NCCL when all devices differ, the same-device communicator when all
// ranks are threads of one process on one device, a message naming the ranks that share a device otherwise.
static LayoutDecision DecideLayout(const std::vector<RankHello>& h) {
  LayoutDecision d{};
  const int R = static_cast<int>(h.size());
  std::map<std::string, std::vector<int>> by_device;
  bool one_process = true;
  for (int r = 0; r < R; ++r) { by_device[UuidString(h[r].uuid)].push_back(r); one_process &= h[r].token == h[0].token; }
  if (static_cast<int>(by_device.size()) == R) { d.layout = kLayoutNccl; return d; }
  if (by_device.size() == 1 && one_process && R <= kMaxPeers) { d.layout = kLayoutSameDevice; return d; }
  std::string m = "LGBM_NetworkInit: unsupported layout:";
  for (auto& kv : by_device) {
    if (kv.second.size() < 2) continue;
    m += " ranks";
    for (size_t i = 0; i < kv.second.size(); ++i) m += (i ? "," : " ") + std::to_string(kv.second[i]);
    m += " share CUDA device " + kv.first + ";";
  }
  if (by_device.size() == 1 && one_process) m += " more than " + std::to_string(kMaxPeers) + " ranks on one device;";
  m += " supported layouts are one device per rank (NCCL) or every rank a thread of one process on one device (same-device collective)";
  d.layout = kLayoutRejected;
  std::snprintf(d.message, sizeof(d.message), "%s", m.c_str());
  return d;
}

static void SetSocketTimeout(int fd, int sec) {
  timeval tv{std::max(sec, 1), 0};
  setsockopt(fd, SOL_SOCKET, SO_RCVTIMEO, &tv, sizeof(tv));
  setsockopt(fd, SOL_SOCKET, SO_SNDTIMEO, &tv, sizeof(tv));
}

// Replaces LGBM_NetworkInit's TCP mesh (reference call site TrainUtils.scala:279-295): the machine list is only used to agree on ranks.
// Rank 0 connects to every other rank, collects each rank's process token and device UUID, decides the layout (DecideLayout) and sends
// the decision — with its ncclUniqueId when NCCL was chosen — back over the same connections.  NCCL training traffic then goes over
// NVLink / NVSwitch; a same-device network never leaves the process.  A rejected layout fails on every rank with the same message.
void NetworkInit(const char* machines, int local_listen_port, int listen_time_out_sec, int num_machines) {
  NetworkFree();
  if (num_machines <= 1) return;
  std::vector<std::pair<std::string, int>> nodes;
  {
    std::string s(machines ? machines : "");
    for (auto& c : s) if (c == ' ' || c == ';') c = ',';
    std::stringstream ss(s);
    std::string tok;
    while (std::getline(ss, tok, ',')) {
      if (tok.empty()) continue;
      size_t p = tok.rfind(':');
      if (p == std::string::npos) Fatal("machines should be a list of ip:port, got '" + tok + "'");
      nodes.emplace_back(tok.substr(0, p), std::atoi(tok.c_str() + p + 1));
    }
  }
  if (static_cast<int>(nodes.size()) < num_machines) Fatal("machine list shorter than num_machines");
  nodes.resize(num_machines);
  int rank = -1;
  for (int i = 0; i < num_machines; ++i) if (nodes[i].second == local_listen_port) { rank = i; break; }
  if (rank < 0) Fatal("local_listen_port " + std::to_string(local_listen_port) + " is not in the machine list");
  if (t_device < 0) {
    int cnt = DeviceCountOrDie();
    const char* lr = std::getenv("LOCAL_RANK");
    t_device = (lr ? std::atoi(lr) : rank) % cnt;
  }
  EnsureDevice();
  const auto deadline = std::chrono::steady_clock::now() + std::chrono::seconds(std::max(listen_time_out_sec, 1));
  RankHello mine{};
  mine.token = g_process_token;
  {
    cudaDeviceProp prop;
    B200_CUDA(cudaGetDeviceProperties(&prop, t_device));
    std::memcpy(mine.uuid, prop.uuid.bytes, 16);
  }
  LayoutDecision dec{};
  std::shared_ptr<SameDeviceComm> sd;
  if (rank == 0) {
    struct Conns { std::vector<int> fd; ~Conns() { for (int f : fd) ::close(f); } } conns;
    std::vector<RankHello> hello(num_machines);
    hello[0] = mine;
    for (int r = 1; r < num_machines; ++r) {
      int fd = -1;
      while (true) {
        addrinfo hints{}, *res = nullptr;
        hints.ai_family = AF_INET; hints.ai_socktype = SOCK_STREAM;
        std::string port = std::to_string(nodes[r].second);
        if (getaddrinfo(nodes[r].first.c_str(), port.c_str(), &hints, &res) == 0 && res) {
          fd = ::socket(res->ai_family, res->ai_socktype, res->ai_protocol);
          if (fd >= 0 && ::connect(fd, res->ai_addr, res->ai_addrlen) == 0) { freeaddrinfo(res); break; }
          if (fd >= 0) ::close(fd);
          fd = -1;
          freeaddrinfo(res);
        }
        if (std::chrono::steady_clock::now() > deadline) Fatal("network bootstrap: cannot reach " + nodes[r].first + ":" + std::to_string(nodes[r].second));
        std::this_thread::sleep_for(std::chrono::milliseconds(20));
      }
      conns.fd.push_back(fd);
      SetSocketTimeout(fd, listen_time_out_sec);
      RecvAll(fd, &hello[r], sizeof(RankHello));
    }
    dec = DecideLayout(hello);
    if (dec.layout == kLayoutNccl) B200_NCCL(ncclGetUniqueId(&dec.id));
    if (dec.layout == kLayoutSameDevice) {      // created before any rank hears the decision, so every rank finds it
      sd = std::make_shared<SameDeviceComm>();
      sd->world = num_machines;
      sd->stream = SharedStream(t_device);
      sd->timeout = std::chrono::seconds(std::max(listen_time_out_sec, 1));
      dec.sequence = ++g_comm_sequence;
      std::lock_guard<std::mutex> lk(g_comm_registry_mu);
      g_comm_registry[{g_process_token, dec.sequence}] = sd;
    }
    struct Unregister {      // once every rank attached, or when the bootstrap fails; the ranks hold the communicator
      unsigned long long seq;
      ~Unregister() { if (seq) { std::lock_guard<std::mutex> lk(g_comm_registry_mu); g_comm_registry.erase({g_process_token, seq}); } }
    } unregister{dec.sequence};
    for (int fd : conns.fd) {      // the ack comes after the rank attached to a same-device communicator
      SendAll(fd, &dec, sizeof(dec));
      char ack = 0;
      RecvAll(fd, &ack, 1);
    }
  } else {
    int ls = ::socket(AF_INET, SOCK_STREAM, 0);
    if (ls < 0) Fatal("network bootstrap: socket() failed");
    int one = 1;
    setsockopt(ls, SOL_SOCKET, SO_REUSEADDR, &one, sizeof(one));
    sockaddr_in addr{};
    addr.sin_family = AF_INET; addr.sin_addr.s_addr = htonl(INADDR_ANY); addr.sin_port = htons(static_cast<uint16_t>(local_listen_port));
    if (::bind(ls, reinterpret_cast<sockaddr*>(&addr), sizeof(addr)) != 0) { ::close(ls); Fatal("network bootstrap: cannot bind port " + std::to_string(local_listen_port)); }
    ::listen(ls, 4);
    fd_set fds;
    FD_ZERO(&fds); FD_SET(ls, &fds);
    timeval tv{std::max(listen_time_out_sec, 1), 0};
    if (::select(ls + 1, &fds, nullptr, nullptr, &tv) <= 0) { ::close(ls); Fatal("network bootstrap: timed out waiting for rank 0"); }
    int fd = ::accept(ls, nullptr, nullptr);
    ::close(ls);
    if (fd < 0) Fatal("network bootstrap: accept failed");
    struct Conn { int fd; ~Conn() { ::close(fd); } } conn{fd};
    SetSocketTimeout(fd, listen_time_out_sec);
    SendAll(fd, &mine, sizeof(mine));
    RecvAll(fd, &dec, sizeof(dec));
    if (dec.layout == kLayoutSameDevice) {
      std::lock_guard<std::mutex> lk(g_comm_registry_mu);
      auto it = g_comm_registry.find({g_process_token, dec.sequence});
      if (it == g_comm_registry.end()) Fatal("network bootstrap: rank 0's same-device communicator is not in this process");
      sd = it->second;
    }
    char ack = 1;
    SendAll(fd, &ack, 1);
  }
  if (dec.layout == kLayoutRejected) Fatal(std::string(dec.message, strnlen(dec.message, sizeof(dec.message))));
  if (sd) {
    t_net.active = true; t_net.rank = rank; t_net.world = num_machines; t_net.same_device = sd;
    return;
  }
  ncclComm_t comm;
  B200_NCCL(ncclCommInitRank(&comm, num_machines, dec.id, rank));
  t_net.active = true; t_net.rank = rank; t_net.world = num_machines; t_net.comm = comm;
}
// Leaving a same-device network marks the rank as left: ranks waiting in a collective, or entering one later, fail instead of waiting for
// it.  Ranks that already completed every collective are not affected.
void NetworkFree() {
  if (t_net.active && t_net.comm) { ncclCommDestroy(t_net.comm); }
  if (t_net.same_device) {
    SameDeviceComm& c = *t_net.same_device;
    std::lock_guard<std::mutex> lk(c.mu);
    if (c.left < 0) c.left = t_net.rank;
    c.cv.notify_all();
  }
  t_net = Network();
}

void AllReduceHost(double* v, int n, ncclRedOp_t op, cudaStream_t s) {
  if (!Net().active) return;
  DevBuf<double> d; d.Alloc(n);
  d.Upload(v, n, s);
  Net().AllReduce(d.p, n, ncclDouble, op, s);
  d.Download(v, n, s);
  B200_CUDA(cudaStreamSynchronize(s));
}

// =============================================================================== dataset
Dataset::~Dataset() {
  ReleaseIngestStaging();
  ReleaseStream(stream);
}

template <typename T>
__global__ void k_gather_rows(const T* __restrict__ X, long long nrow, int ncol, int row_major, const int* __restrict__ rows, int nsample,
                              double* __restrict__ out) {
  for (long long e = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; e < static_cast<long long>(nsample) * ncol;
       e += static_cast<long long>(gridDim.x) * blockDim.x) {
    int s = static_cast<int>(e / ncol), f = static_cast<int>(e % ncol);
    long long r = rows[s];
    out[e] = row_major ? static_cast<double>(X[r * ncol + f]) : static_cast<double>(X[static_cast<long long>(f) * nrow + r]);
  }
}

static bool IsDevicePointer(const void* p) {
  cudaPointerAttributes a;
  cudaError_t e = cudaPointerGetAttributes(&a, p);
  if (e != cudaSuccess) { cudaGetLastError(); return false; }
  return a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged;
}

static void PackMapper(const FeatureBins& fb, double* r, int slots) {
  r[0] = fb.num_bin; r[1] = fb.missing_type; r[2] = fb.trivial; r[3] = fb.default_bin; r[4] = fb.most_freq_bin;
  r[5] = fb.sparse_rate; r[6] = fb.min_val; r[7] = fb.max_val; r[8] = fb.categorical; r[9] = 0;
  for (int i = 0; i < slots; ++i) {
    if (fb.categorical) r[10 + i] = i < static_cast<int>(fb.bin_to_cat.size()) ? fb.bin_to_cat[i] : 0.0;
    else r[10 + i] = i < static_cast<int>(fb.upper.size()) ? fb.upper[i] : 0.0;
  }
}
static FeatureBins UnpackMapper(const double* r) {
  FeatureBins fb;
  fb.num_bin = static_cast<int>(r[0]); fb.missing_type = static_cast<int>(r[1]); fb.trivial = r[2] != 0;
  fb.default_bin = static_cast<uint32_t>(r[3]); fb.most_freq_bin = static_cast<uint32_t>(r[4]);
  fb.sparse_rate = r[5]; fb.min_val = r[6]; fb.max_val = r[7]; fb.categorical = r[8] != 0;
  if (fb.categorical) {
    for (int b = 0; b < fb.num_bin; ++b) fb.bin_to_cat.push_back(static_cast<int>(r[10 + b]));
    std::vector<std::pair<int, int>> byc;
    for (int b = 1; b < fb.num_bin; ++b) byc.emplace_back(fb.bin_to_cat[b], b);
    std::sort(byc.begin(), byc.end());
    for (auto& p : byc) { fb.sorted_cats.push_back(p.first); fb.sorted_bins.push_back(p.second); }
  } else {
    fb.upper.assign(r + 10, r + 10 + fb.num_bin);
  }
  return fb;
}

// device, stream, sizes and parameters of a new dataset (the caller has run EnsureDevice)
std::unique_ptr<Dataset> Dataset::NewShell(int nrow, int ncol, const char* params) {
  std::unique_ptr<Dataset> d(new Dataset());
  d->device = CurrentDevice();
  d->stream = AcquireStream();
  d->num_data = nrow; d->num_total_features = ncol;
  d->cfg.Parse(params);
  return d;
}

// the rows whose values define the bins
std::vector<int> Dataset::SampleRows() const {
  LcgRandom rnd(cfg.data_random_seed);
  return rnd.Sample(num_data, std::min(num_data, cfg.bin_construct_sample_cnt));
}

// Mappers and feature names of a new dataset.  With a reference they are the reference's and the bin parameters are not checked.
// Otherwise the bin parameters are checked, then sample(&nz, &nz_rows, f0, f1) fills nz[f] with the sampled values of feature f that are
// NaN or have |v| > 1e-35 (at least for this rank's features f0 <= f < f1) and returns the number of sampled rows.  When nz_rows is not
// null (bundling), it fills every feature, and nz_rows[f] with the sample position (0 .. count-1) of each value of nz[f].
// Bundles are grouped on rank 0's sample and broadcast, so every rank starts from the same candidate bundles.
template <typename Sample>
void Dataset::SetMappers(const Dataset* reference, bool may_bundle, Sample sample) {
  const int n = num_data, F = num_total_features;
  if (reference) {
    if (reference->num_total_features != F) Fatal("Validation data has a different number of features than the reference dataset");
    mappers = reference->mappers;
    feature_names = reference->feature_names;
    return;
  }
  if (cfg.max_bin >= kWideMaxBins) Fatal("max_bin >= " + std::to_string(kWideMaxBins) + " is not supported");
  if (cfg.max_bin < 2) Fatal("max_bin should be >= 2");
  if (cfg.zero_as_missing) Fatal("zero_as_missing=true is not supported by this build");
  // feature ownership for distributed bin finding (SURVEY.md fact 9, A.2): contiguous slices of ceil(F/R)
  const int world = Net().active ? Net().world : 1, rank = Net().active ? Net().rank : 0;
  const int step = std::max(1, (F + world - 1) / world);
  const int f0 = world == 1 ? 0 : std::min(F, rank * step), f1 = world == 1 ? F : std::min(F, f0 + step);
  const bool bundle = may_bundle && cfg.enable_bundle;
  std::vector<std::vector<double>> nz(F);
  std::vector<std::vector<int>> nz_rows(bundle ? F : 0);
  const int sample_cnt = sample(&nz, bundle ? &nz_rows : nullptr, f0, f1);
  NvtxRange nvtx("b200gbm:find bins (host) + C5 mapper all-gather");
  const int filter_cnt = static_cast<int>(static_cast<double>(cfg.min_data_in_leaf) * sample_cnt / n);
  mappers.assign(F, FeatureBins());
#pragma omp parallel for schedule(dynamic)
  for (int f = f0; f < f1; ++f) {
    std::vector<double> vals;      // the bin finders reorder their input; bundling needs nz[f] in step with nz_rows[f]
    std::vector<double>* v = &nz[f];
    if (bundle) { vals = nz[f]; v = &vals; }
    const bool is_cat = std::find(cfg.categorical_feature.begin(), cfg.categorical_feature.end(), f) != cfg.categorical_feature.end();
    if (is_cat) mappers[f] = FindCategoricalBins(v, sample_cnt, cfg.max_bin, cfg.min_data_in_bin, filter_cnt, cfg.feature_pre_filter);
    else mappers[f] = FindFeatureBins(v, sample_cnt, cfg.max_bin, cfg.min_data_in_bin, filter_cnt, cfg.feature_pre_filter, cfg.use_missing,
                                      cfg.zero_as_missing);
  }
  for (int f = f0; f < f1; ++f)
    if (mappers[f].num_bin > kWideMaxBins)
      Fatal("categorical feature " + std::to_string(f) + " needs " + std::to_string(mappers[f].num_bin) +
            " bins (a categorical feature keeps categories until 99% of its mass is covered); this build supports at most " + std::to_string(kWideMaxBins) + " bins per feature");
  if (world > 1) {   // C5: all-gather the serialized mappers (record = 10 header doubles + the largest bin count of any rank)
    double maxbins = 256;
    for (int f = f0; f < f1; ++f) maxbins = std::max(maxbins, static_cast<double>(mappers[f].num_bin));
    AllReduceHost(&maxbins, 1, ncclMax, stream);
    const int slots = static_cast<int>(maxbins);
    const size_t kMapperRecord = 10 + static_cast<size_t>(slots);
    std::vector<double> send(static_cast<size_t>(step) * kMapperRecord, 0.0), recv(static_cast<size_t>(world) * step * kMapperRecord);
    for (int f = f0; f < f1; ++f) PackMapper(mappers[f], &send[static_cast<size_t>(f - f0) * kMapperRecord], slots);
    DevBuf<double> ds, dr; ds.Alloc(send.size()); dr.Alloc(recv.size());
    ds.Upload(send.data(), send.size(), stream);
    Net().AllGather(ds.p, dr.p, send.size() * sizeof(double), stream);
    dr.Download(recv.data(), recv.size(), stream);
    B200_CUDA(cudaStreamSynchronize(stream));
    for (int f = 0; f < F; ++f) {
      int owner = f / step, off = f - owner * step;
      mappers[f] = UnpackMapper(&recv[(static_cast<size_t>(owner) * step + off) * kMapperRecord]);
    }
  }
  feature_names.resize(F);
  for (int f = 0; f < F; ++f) feature_names[f] = "Column_" + std::to_string(f);
  bundles.clear();
  if (!bundle) return;
  if (rank == 0) {
    std::vector<std::vector<int>> off_mfb(F);
#pragma omp parallel for schedule(dynamic)
    for (int f = 0; f < F; ++f) {
      const FeatureBins& fb = mappers[f];
      if (!BundleCandidate(fb)) continue;
      for (size_t i = 0; i < nz[f].size(); ++i)
        if (fb.ValueToBin(nz[f][i]) != fb.most_freq_bin) off_mfb[f].push_back(nz_rows[f][i]);
    }
    bundles = FindBundles(mappers, off_mfb, sample_cnt);
  }
  if (world > 1) {      // broadcast rank 0's grouping: bundle index + 1 of every feature, summed over ranks that send zeros
    std::vector<double> of(F, 0.0);
    for (size_t k = 0; k < bundles.size(); ++k) for (int f : bundles[k]) of[f] = static_cast<double>(k + 1);
    AllReduceHost(of.data(), F, ncclSum, stream);
    int nb = 0;
    for (int f = 0; f < F; ++f) nb = std::max(nb, static_cast<int>(of[f]));
    bundles.assign(nb, {});
    for (int f = 0; f < F; ++f) if (of[f] > 0) bundles[static_cast<int>(of[f]) - 1].push_back(f);
  }
}

// The device table of the bundle members (BundleMember, kernels.cuh).  inner / base / the bundle columns are valid after UploadMeta.
void Dataset::UploadBundleMembers() {
  std::vector<BundleMember> mem;
  std::vector<int> start(1, 0), bcol;
  for (const std::vector<int>& b : bundles) {
    int base = 0;
    for (int f : b) {
      const FeatureBins& fb = mappers[f];
      const int db = static_cast<int>(fb.default_bin);
      BundleMember m{};
      m.zlo = db == 0 ? -std::numeric_limits<double>::infinity() : fb.upper[db - 1];
      m.zhi = fb.upper[db];
      m.real_index = f;
      m.inner = inner_of.empty() ? -1 : inner_of[f];
      m.base = base;
      m.bundle = static_cast<int>(start.size()) - 1;
      m.nan_moves = fb.missing_type == MISSING_NAN ? 1 : 0;
      mem.push_back(m);
      base += fb.num_bin - 1;
    }
    start.push_back(static_cast<int>(mem.size()));
    bcol.push_back(inner_of.empty() ? -1 : meta_host[inner_of[b[0]]].hist_off >> 8);
  }
  d_members.Alloc(std::max<size_t>(mem.size(), 1)); d_bundle_start.Alloc(start.size()); d_bundle_col.Alloc(std::max<size_t>(bcol.size(), 1));
  if (!mem.empty()) { d_members.Upload(mem.data(), mem.size(), stream); d_bundle_col.Upload(bcol.data(), bcol.size(), stream); }
  d_bundle_start.Upload(start.data(), start.size(), stream);
  B200_CUDA(cudaStreamSynchronize(stream));
}

// Every row of the input is checked before any bin is written; with data-parallel training the counts of all ranks are combined, so
// every rank keeps the same bundles (and the histogram all-reduce one buffer shape).
template <typename Count>
void Dataset::DissolveConflictingBundles(Count count) {
  const bool parallel = Net().active && Net().world > 1;
  if (bundles.empty()) return;
  NvtxRange nvtx("b200gbm:bundle row check");
  UploadBundleMembers();
  const int nb = static_cast<int>(bundles.size());
  DevBuf<unsigned long long> conflicts; conflicts.Alloc(nb); conflicts.Zero(stream);
  count(conflicts.p);
  B200_CUDA(cudaGetLastError());
  std::vector<unsigned long long> h(nb);
  conflicts.Download(h.data(), nb, stream);
  B200_CUDA(cudaStreamSynchronize(stream));
  std::vector<double> c(h.begin(), h.end());
  if (parallel) AllReduceHost(c.data(), nb, ncclMax, stream);
  std::vector<std::vector<int>> kept;
  for (int k = 0; k < nb; ++k) if (c[k] == 0.0) kept.push_back(std::move(bundles[k]));
  bundles = std::move(kept);
}

void Dataset::UploadMeta() {
  // inner order: features with <= 256 bins first (uint8 tiles of 32), then the wide ones (uint16 columns), each group in real-index order
  used.clear();
  inner_of.assign(num_total_features, -1);
  std::vector<int> wide_real;
  for (int f = 0; f < num_total_features; ++f) {
    if (mappers[f].trivial) continue;
    if (mappers[f].num_bin > 256) wide_real.push_back(f);
    else { inner_of[f] = static_cast<int>(used.size()); used.push_back(f); }
  }
  nfn = static_cast<int>(used.size());
  for (int f : wide_real) { inner_of[f] = static_cast<int>(used.size()); used.push_back(f); }
  nf = static_cast<int>(used.size());
  nw = nf - nfn;
  sample_order.clear();
  for (int f = 0; f < num_total_features; ++f) if (inner_of[f] >= 0) sample_order.push_back(inner_of[f]);
  // storage columns in inner-feature order: a plain feature's column, or its bundle's column where the bundle's first feature comes
  std::vector<int> bundle_of(num_total_features, -1), col_of(nfn, 0), base_of(nfn, -1), bundle_col(bundles.size(), -1);
  for (size_t k = 0; k < bundles.size(); ++k) {
    int base = 0;
    for (int f : bundles[k]) { bundle_of[f] = static_cast<int>(k); base_of[inner_of[f]] = base; base += mappers[f].num_bin - 1; }
  }
  num_columns = 0;
  for (int u = 0; u < nfn; ++u) {
    const int k = bundle_of[used[u]];
    if (k < 0) col_of[u] = num_columns++;
    else { if (bundle_col[k] < 0) bundle_col[k] = num_columns++; col_of[u] = bundle_col[k]; }
  }
  num_tiles = std::max(1, (num_columns + 31) / 32);
  col_feat.assign(static_cast<size_t>(num_tiles) * 32, -1);
  for (int u = 0; u < nfn; ++u) if (base_of[u] < 0) col_feat[col_of[u]] = u;
  const int nft = std::max(1, (nfn + 31) / 32) * 32;      // inner slots of the tile features
  nf_pad = nft + nw;
  meta_host.assign(nf_pad, FeatMeta{1, 0, 0, 0, 0, 0, 0, 0, 0});
  bundle_base.assign(nf_pad, -1);
  for (int u = 0; u < nfn; ++u) bundle_base[u] = base_of[u];
  // bin tables: tile slot u's row at u * 256 (k_bin_rows stages a tile's rows in shared memory), then one row per wide feature
  std::vector<double> ubh(static_cast<size_t>(nft) * 256, 0.0);
  std::vector<uint16_t> cbh(ubh.size(), 0);
  has_categorical = false;
  hist_pairs = static_cast<size_t>(num_tiles) * 32 * 256;
  for (int u = 0; u < nf; ++u) {
    const FeatureBins& fb = mappers[used[u]];
    const size_t row_len = fb.categorical ? fb.sorted_cats.size() : static_cast<size_t>(fb.num_bin);
    int hist_off = u < nfn ? col_of[u] * 256 : 0;
    size_t table_off = static_cast<size_t>(u) * 256;
    if (u >= nfn) {
      hist_off = static_cast<int>(hist_pairs);
      hist_pairs += (static_cast<size_t>(fb.num_bin) + 255) / 256 * 256;
      if (hist_pairs > (1u << 30)) Fatal("histogram of the wide features is too large");
      table_off = ubh.size();
      ubh.resize(table_off + row_len, 0.0);
      cbh.resize(table_off + row_len, 0);
    }
    meta_host[u] = FeatMeta{fb.num_bin, fb.missing_type, static_cast<int>(fb.default_bin), fb.most_freq_bin == 0 ? 1 : 0, used[u],
                            fb.categorical ? 1 : 0, static_cast<int>(fb.sorted_cats.size()), hist_off, static_cast<int>(table_off)};
    if (fb.categorical) {
      has_categorical = true;
      for (size_t i = 0; i < row_len; ++i) { ubh[table_off + i] = fb.sorted_cats[i]; cbh[table_off + i] = static_cast<uint16_t>(fb.sorted_bins[i]); }
    } else {
      for (size_t b = 0; b < row_len; ++b) ubh[table_off + b] = fb.upper[b];
    }
  }
  meta.Alloc(nf_pad); ub.Alloc(ubh.size()); catbin.Alloc(cbh.size());
  meta.Upload(meta_host.data(), nf_pad, stream);
  d_col_feat.Alloc(col_feat.size()); d_col_feat.Upload(col_feat.data(), col_feat.size(), stream);
  d_bundle_base.Alloc(nf_pad); d_bundle_base.Upload(bundle_base.data(), nf_pad, stream);
  if (!bundles.empty()) UploadBundleMembers();
  ub.Upload(ubh.data(), ubh.size(), stream);
  catbin.Upload(cbh.data(), cbh.size(), stream);
  B200_CUDA(cudaStreamSynchronize(stream));
}

// last step of every create once the mappers are set: their device tables, and the bins (tiles + wide columns) of num_data rows
void Dataset::AllocBins() {
  UploadMeta();
  rows_stride = static_cast<size_t>(num_data);
  bins.Alloc(static_cast<size_t>(num_tiles) * rows_stride * 32);
  if (nw > 0) bins16.Alloc(static_cast<size_t>(nw) * rows_stride);
}

template <typename T>
static void LaunchBin(const T* X, long long nrow, int ncol, int row_major, long long ld, const Dataset& d, long long row_offset, cudaStream_t s) {
  // function attributes are per device/context: set on every call (rank-threads drive different GPUs)
  B200_CUDA(cudaFuncSetAttribute(k_bin_rows<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, 65536));
  const int sms = DeviceSMs();
  dim3 grid(static_cast<unsigned>(std::min<long long>((nrow + 7) / 8, sms * 8)), d.num_tiles);
  if (grid.x == 0) grid.x = 1;
  k_bin_rows<T><<<grid, 256, 65536, s>>>(X, nrow, ncol, row_major, ld, d.meta.p, d.ub.p, d.catbin.p, d.d_col_feat.p, d.bins.p, static_cast<long long>(d.rows_stride), row_offset);
  if (!d.bundles.empty())      // after k_bin_rows (same stream): it left the bundle columns at slot 0
    k_bin_bundles<T><<<sms * 8, 256, 0, s>>>(X, nrow, row_major, ld, d.d_members.p, d.d_bundle_start.p, d.d_bundle_col.p, static_cast<int>(d.bundles.size()),
                                             d.meta.p, d.ub.p, d.bins.p, static_cast<long long>(d.rows_stride), row_offset);
  if (d.nw > 0)
    k_bin_wide<T><<<sms * 8, 256, 0, s>>>(X, nrow, row_major, ld, d.meta.p + d.nfn, d.nw, d.ub.p, d.catbin.p, d.bins16.p, d.rows_stride, row_offset);
  B200_CUDA(cudaGetLastError());
}

void Dataset::BinBlock(const std::vector<MatPart>& parts, int data_type, int is_row_major, long long start_row) {
  NvtxRange nvtx("b200gbm:K0 bin rows (H2D + value->bin)");
  const int F = num_total_features;
  long long n = 0, host_rows = 0;
  for (const MatPart& p : parts) { n += p.nrow; if (!p.on_device) host_rows += p.nrow; }
  if (start_row < 0 || start_row + n > num_data) Fatal("row block out of range");
  {
    std::lock_guard<std::mutex> lock(block_bound_mu_);
    block_bound_.Free();      // a bound of earlier bins would let K4 overflow a cell
  }
  ForEachDeviceBlock(parts, data_type, is_row_major, [&](const void* x, long long rows, long long ld, long long r0) {
    if (data_type == 0) LaunchBin<float>(static_cast<const float*>(x), rows, F, is_row_major, ld, *this, start_row + r0, stream);
    else LaunchBin<double>(static_cast<const double*>(x), rows, F, is_row_major, ld, *this, start_row + r0, stream);
  });
  if (host_rows == 0) return;
  ingest_rows_done_ += host_rows;
  if (ingest_rows_done_ >= num_data) ReleaseIngestStaging();
}

template <typename Fn>
void Dataset::ForEachDeviceBlock(const std::vector<MatPart>& parts, int data_type, int is_row_major, Fn fn) {
  const int F = num_total_features;
  const size_t esz = data_type == 0 ? 4 : 8;
  // host parts: stream row chunks through two device buffers, copy of chunk i+1 overlaps binning of chunk i, also where chunk i is
  // the last of one part and chunk i+1 the first of the next.  The staging buffers, copy stream and events persist across
  // LGBM_DatasetPushRows calls (a cudaMalloc/cudaFree pair per call costs as much as the copy itself) and are released when the
  // last row has arrived.
  const size_t kStageBytes = 256u << 20;
  long long host_max = 0;
  for (const MatPart& p : parts) if (!p.on_device) host_max = std::max(host_max, p.nrow);
  const long long chunk = std::max<long long>(1, std::min<long long>(host_max, static_cast<long long>(kStageBytes) / (static_cast<long long>(F) * esz)));
  if (host_max > 0) {
    const size_t need = static_cast<size_t>(chunk) * F * esz;
    if (!ingest_copy_stream_) {
      B200_CUDA(cudaStreamCreateWithFlags(&ingest_copy_stream_, cudaStreamNonBlocking));
      for (int i = 0; i < 2; ++i) {
        B200_CUDA(cudaEventCreateWithFlags(&ingest_copied_[i], cudaEventDisableTiming));
        B200_CUDA(cudaEventCreateWithFlags(&ingest_binned_[i], cudaEventDisableTiming));
      }
    }
    for (int i = 0; i < 2; ++i) if (ingest_buf_[i].n < need) ingest_buf_[i].Alloc(std::max(need, std::min(kStageBytes, static_cast<size_t>(num_data) * F * esz)));
  }
  cudaStream_t copy_stream = ingest_copy_stream_;
  int it = 0;                 // host chunks so far, over all parts: the buffer of chunk it is it & 1
  long long first = 0;        // first row of the part
  for (const MatPart& p : parts) {
    const long long n = p.nrow;
    if (p.on_device) {
      fn(p.data, n, is_row_major ? F : n, first);
      first += n;
      continue;
    }
    for (long long r0 = 0; r0 < n; r0 += chunk, ++it) {
      const int b = it & 1;
      const long long rows = std::min(chunk, n - r0);
      if (it >= 2) B200_CUDA(cudaStreamWaitEvent(copy_stream, ingest_binned_[b], 0));
      if (is_row_major) {
        B200_CUDA(cudaMemcpyAsync(ingest_buf_[b].p, static_cast<const unsigned char*>(p.data) + static_cast<size_t>(r0) * F * esz, static_cast<size_t>(rows) * F * esz,
                                  cudaMemcpyHostToDevice, copy_stream));
      } else {   // column-major: F column segments of `rows` elements, device chunk keeps ld = rows
        B200_CUDA(cudaMemcpy2DAsync(ingest_buf_[b].p, static_cast<size_t>(rows) * esz, static_cast<const unsigned char*>(p.data) + static_cast<size_t>(r0) * esz,
                                    static_cast<size_t>(n) * esz, static_cast<size_t>(rows) * esz, F, cudaMemcpyHostToDevice, copy_stream));
      }
      B200_CUDA(cudaEventRecord(ingest_copied_[b], copy_stream));
      B200_CUDA(cudaStreamWaitEvent(stream, ingest_copied_[b], 0));
      fn(static_cast<const void*>(ingest_buf_[b].p), rows, is_row_major ? F : rows, first + r0);
      B200_CUDA(cudaEventRecord(ingest_binned_[b], stream));
    }
    first += n;
  }
  B200_CUDA(cudaStreamSynchronize(stream));          // all copies are consumed: the caller may reuse its buffers
}

void Dataset::ReleaseIngestStaging() {
  for (int i = 0; i < 2; ++i) {
    ingest_buf_[i].Free();
    if (ingest_copied_[i]) { cudaEventDestroy(ingest_copied_[i]); ingest_copied_[i] = nullptr; }
    if (ingest_binned_[i]) { cudaEventDestroy(ingest_binned_[i]); ingest_binned_[i] = nullptr; }
  }
  if (ingest_copy_stream_) { cudaStreamDestroy(ingest_copy_stream_); ingest_copy_stream_ = nullptr; }
}

Dataset* Dataset::CreateFromSampledColumn(double** sample_data, int** sample_indices, int ncol, const int* num_per_col, int num_sample_row,
                                          int num_total_row, const char* params) {
  (void)sample_indices;
  EnsureDevice();
  if (num_total_row <= 0 || ncol <= 0) Fatal("Dataset should have at least one row and one column");
  std::unique_ptr<Dataset> d = NewShell(num_total_row, ncol, params);
  d->SetMappers(nullptr, false, [&](std::vector<std::vector<double>>* nz, std::vector<std::vector<int>>*, int, int) {      // the caller sampled the rows and dropped the zeros
    for (int f = 0; f < ncol; ++f) (*nz)[f].assign(sample_data[f], sample_data[f] + num_per_col[f]);
    return num_sample_row;
  });
  d->AllocBins();
  return d.release();
}

void Dataset::PushRows(const void* data, int data_type, int nrow, int ncol, int start_row) {
  EnsureDevice();
  if (ncol != num_total_features) Fatal("PushRows: wrong number of columns");
  if (data_type != 0 && data_type != 1) Fatal("PushRows: unknown data type");
  StreamTimer timer(stream);
  BinBlock({MatPart{data, nrow, IsDevicePointer(data)}}, data_type, 1, start_row);
  ingest_ms += timer.Ms();
}

// the uint8 tile features' bins into out[num_data][num_total_features]; every other column is zero
template <typename T>
void Dataset::UnpackTiles(T* out) const {
  std::vector<uint8_t> h(bins.n);
  B200_CUDA(cudaMemcpy(h.data(), bins.p, bins.n, cudaMemcpyDeviceToHost));
  std::memset(out, 0, static_cast<size_t>(num_data) * num_total_features * sizeof(T));
  for (int u = 0; u < nfn; ++u) {
    const int f = used[u];
    const FeatMeta& m = meta_host[u];
    const int c = m.hist_off >> 8;
    const uint8_t* src = h.data() + (static_cast<size_t>(c >> 5) * rows_stride) * 32 + (c & 31);
    for (int i = 0; i < num_data; ++i)
      out[static_cast<size_t>(i) * num_total_features + f] = static_cast<T>(d_unbundle(src[static_cast<size_t>(i) * 32], bundle_base[u], m.default_bin, m.num_bin));
  }
}
void Dataset::GetBinsRowMajor(uint8_t* out) const {
  if (nw > 0) Fatal("this dataset has features with more than 256 bins: use B200GBM_DatasetGetBins16");
  UnpackTiles(out);
}
void Dataset::GetBinsRowMajor16(uint16_t* out) const {
  UnpackTiles(out);
  if (nw > 0) {
    std::vector<uint16_t> hw(bins16.n);
    B200_CUDA(cudaMemcpy(hw.data(), bins16.p, bins16.n * sizeof(uint16_t), cudaMemcpyDeviceToHost));
    for (int w = 0; w < nw; ++w) {
      const int f = used[nfn + w];
      const uint16_t* src = hw.data() + static_cast<size_t>(w) * rows_stride;
      for (int i = 0; i < num_data; ++i) out[static_cast<size_t>(i) * num_total_features + f] = src[i];
    }
  }
}

__global__ void k_gather_bin_rows(BinView bv, int nf, const FeatMeta* __restrict__ meta, const int* __restrict__ rows, int nrows, int F,
                                  uint16_t* __restrict__ out) {
  for (long long e = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; e < static_cast<long long>(nrows) * nf;
       e += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int i = static_cast<int>(e / nf), u = static_cast<int>(e % nf);
    out[static_cast<size_t>(i) * F + meta[u].real_index] = static_cast<uint16_t>(bv.at(u, static_cast<size_t>(rows[i])));
  }
}
void Dataset::GetBinsOfRows(const int32_t* rows, int nrows, uint16_t* out) const {
  if (nrows <= 0) return;
  for (int i = 0; i < nrows; ++i) if (rows[i] < 0 || rows[i] >= num_data) Fatal("GetBinsOfRows: row index out of range");
  DevBuf<int> dr; dr.Alloc(nrows);
  DevBuf<uint16_t> dout; dout.Alloc(static_cast<size_t>(nrows) * num_total_features);
  dr.Upload(rows, nrows, stream);
  dout.Zero(stream);
  if (nf > 0) k_gather_bin_rows<<<DeviceSMs() * 4, 256, 0, stream>>>(View(), nf, meta.p, dr.p, nrows, num_total_features, dout.p);
  B200_CUDA(cudaGetLastError());
  dout.Download(out, dout.n, stream);
  B200_CUDA(cudaStreamSynchronize(stream));
}

RowBlockBound Dataset::BlockBound() const {
  std::lock_guard<std::mutex> lock(block_bound_mu_);
  if (!block_bound_.p) {
    block_bound_.Alloc(static_cast<size_t>(num_tiles) * (bound_blocks(num_data) + 1));
    launch_block_bound(bins.p, rows_stride, num_data, num_tiles, num_columns, block_bound_.p, stream);
    B200_CUDA(cudaGetLastError());
    B200_CUDA(cudaStreamSynchronize(stream));      // the boosters launch K4 on their own streams
  }
  return RowBlockBound{block_bound_.p, bound_blocks(num_data)};
}

// K4 on this dataset's bins for the given rows through the training path's K3 and launch_k4: quant.bins 0 quantises to the 36-bit
// fixed-point grid, quant.bins = B discretises as use_quantized_grad does (hess null: constant hessians, the count plane).  Returns the
// per-inner-feature int64 histograms [nfn][256][2] (bundle columns expanded, exact as in k_scan); ctrl holds the scales, q the words.
std::vector<long long> Dataset::HistogramInt(const float* grad, const float* hess, const int32_t* idx, int cnt, const QuantSpec& quant,
                                             DevBuf<TreeCtrl>& ctrl, DevBuf<int4>& q) const {
  EnsureDevice();
  B200_CUDA(set_k4_smem_limit());
  const int n = num_data;
  const bool const_hessian = hess == nullptr;
  // K4 bounds an index-list item by the row blocks between its first and last row, so it needs a strictly ascending list; the
  // histogram does not depend on the order.  A list that repeats a row is bounded by row counts instead.
  std::vector<int32_t> rows;
  RowBlockBound bound = BlockBound();
  if (idx) {
    rows.assign(idx, idx + cnt);
    std::sort(rows.begin(), rows.end());
    if (cnt > 0 && (rows.front() < 0 || rows.back() >= n)) Fatal("Histogram: row index out of range");
    if (std::adjacent_find(rows.begin(), rows.end()) != rows.end()) bound.prefix = nullptr;
  }
  DevBuf<float> g, h; g.Alloc(n); h.Alloc(n);
  g.Upload(grad, n, stream);
  if (const_hessian) h.Zero(stream); else h.Upload(hess, n, stream);
  q.Alloc(n);
  ctrl.Alloc(1); ctrl.Zero(stream);
  DevBuf<int> didx; didx.Alloc(std::max(cnt, 1));
  if (idx) didx.Upload(rows.data(), cnt, stream);
  const size_t elems = static_cast<size_t>(num_tiles) * 32 * 512;      // tile features only (wide features are covered by the model-level tests)
  DevBuf<long long> H; H.Alloc(elems); H.Zero(stream);
  const size_t felems = static_cast<size_t>(std::max(nfn, 1)) * 512;     // per feature
  int sms = 0;
  B200_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
  const int ch = const_hessian ? 1 : 0;
  k_absmax<<<sms * 4, 256, 0, stream>>>(g.p, h.p, n, ctrl.p);
  k_set_scale<<<1, 1, 0, stream>>>(ctrl.p, ch, 1.0);
  if (quant.bins > 0) {
    k_set_quant_scale<<<1, 1, 0, stream>>>(ctrl.p, ch, quant.bins);
    k_quantize_discrete<<<sms * 4, 256, 0, stream>>>(g.p, h.p, n, q.p, ctrl.p, ch, nullptr, 0, quant.bins, quant.stochastic ? 1 : 0, quant.seed,
                                                     quant.tree);
  } else {
    k_quantize<<<sms * 4, 256, 0, stream>>>(g.p, h.p, n, q.p, ctrl.p, ch, nullptr, 0);
  }
  HistWork w{0, cnt, idx ? 1 : 0, 0};
  B200_CUDA(cudaMemcpyAsync(&ctrl.p->hist_work, &w, sizeof(w), cudaMemcpyHostToDevice, stream));
  DevBuf<int4> qo; qo.Alloc(std::max(cnt, 1));
  k_gather_q<<<sms * 4, 256, 0, stream>>>(&ctrl.p->hist_work, didx.p, didx.p, q.p, qo.p);
  launch_k4(const_hessian, quant.bins, bins.p, rows_stride, num_tiles, q.p, qo.p, didx.p, didx.p, &ctrl.p->hist_work,
            reinterpret_cast<unsigned long long*>(H.p), bound, sms, stream);
  B200_CUDA(cudaGetLastError());
  // per-feature histograms out of the column histograms, exact int64 as in k_scan: a bundle member's most frequent bin is the column total
  // minus the member's other bins
  std::vector<long long> hc(elems), hf(felems, 0);
  H.Download(hc.data(), elems, stream);
  B200_CUDA(cudaStreamSynchronize(stream));
  for (int u = 0; u < nfn; ++u) {
    const FeatMeta& m = meta_host[u];
    const long long* c = hc.data() + static_cast<size_t>(m.hist_off) * 2;
    long long* o = hf.data() + static_cast<size_t>(u) * 512;
    if (bundle_base[u] < 0) { std::copy(c, c + 512, o); continue; }
    long long tot[2] = {0, 0};
    for (int s = 0; s < 256; ++s) { tot[0] += c[s * 2]; tot[1] += c[s * 2 + 1]; }
    for (int b = 0; b < m.num_bin; ++b) {
      if (b == m.default_bin) continue;
      const unsigned s = d_bundle_slot(static_cast<unsigned>(b), bundle_base[u], m.default_bin);
      for (int j = 0; j < 2; ++j) { o[b * 2 + j] = c[s * 2 + j]; tot[j] -= c[s * 2 + j]; }
    }
    o[m.default_bin * 2] = tot[0]; o[m.default_bin * 2 + 1] = tot[1];
  }
  return hf;
}

void Dataset::Histogram(const float* grad, const float* hess, const int32_t* idx, int cnt, double* out) const {
  DevBuf<TreeCtrl> ctrl;
  DevBuf<int4> q;
  const std::vector<long long> hf = HistogramInt(grad, hess, idx, cnt, QuantSpec{}, ctrl, q);
  const size_t felems = hf.size();
  int sms = 0;
  B200_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
  DevBuf<double> D; D.Alloc(felems);
  DevBuf<long long> HF; HF.Alloc(felems); HF.Upload(hf.data(), felems, stream);
  k_hist_to_double<<<sms * 4, 256, 0, stream>>>(HF.p, D.p, felems, ctrl.p);
  B200_CUDA(cudaGetLastError());
  std::vector<double> hd(felems);
  D.Download(hd.data(), felems, stream);
  B200_CUDA(cudaStreamSynchronize(stream));
  std::memset(out, 0, sizeof(double) * static_cast<size_t>(num_total_features) * 512);
  for (int u = 0; u < nfn; ++u) std::memcpy(out + static_cast<size_t>(used[u]) * 512, hd.data() + static_cast<size_t>(u) * 512, sizeof(double) * 512);
}

void Dataset::QuantizedHistogram(const float* grad, const float* hess, const int32_t* idx, int cnt, const QuantSpec& quant, int32_t* out_q,
                                 double* out_scale2, int64_t* out_hist) const {
  if (quant.bins < 2 || quant.bins > 63) Fatal("num_grad_quant_bins should be in [2, 63], got " + std::to_string(quant.bins));
  DevBuf<TreeCtrl> ctrl;
  DevBuf<int4> q;
  const std::vector<long long> hf = HistogramInt(grad, hess, idx, cnt, quant, ctrl, q);
  TreeCtrl c;
  ctrl.Download(&c, 1, stream);
  std::vector<int4> hq(num_data);
  q.Download(hq.data(), hq.size(), stream);
  B200_CUDA(cudaStreamSynchronize(stream));
  for (int i = 0; i < num_data; ++i) {
    out_q[2 * i] = (hq[i].x << kLoBits) + hq[i].y;
    out_q[2 * i + 1] = hess ? (hq[i].z << kLoBits) + hq[i].w : 1;
  }
  out_scale2[0] = c.inv_g; out_scale2[1] = c.inv_h;
  std::memset(out_hist, 0, sizeof(int64_t) * static_cast<size_t>(num_total_features) * 512);
  for (int u = 0; u < nfn; ++u) std::memcpy(out_hist + static_cast<size_t>(used[u]) * 512, hf.data() + static_cast<size_t>(u) * 512, sizeof(int64_t) * 512);
}

// " (part i)" in the messages of a multi-part create
static std::string PartSuffix(int nparts, int i) { return nparts > 1 ? " (part " + std::to_string(i) + ")" : std::string(); }

Dataset* Dataset::CreateFromMats(int nmat, const void* const* data, int data_type, const int32_t* nrow, int ncol, int is_row_major,
                                 const char* params, const Dataset* reference) {
  EnsureDevice();
  if (data_type != 0 && data_type != 1) Fatal("Unknown data type in CreateFromMat (expect C_API_DTYPE_FLOAT32 or FLOAT64)");
  if (nmat < 1) Fatal("CreateFromMats: nmat must be at least 1");
  if (!data || !nrow) Fatal("CreateFromMats: data and nrow must not be null");
  std::vector<MatPart> parts(nmat);
  std::vector<long long> first(nmat + 1, 0);          // first row of every part, then the total
  for (int i = 0; i < nmat; ++i) {
    if (nrow[i] <= 0 || ncol <= 0) Fatal("Dataset should have at least one row and one column" + PartSuffix(nmat, i));
    if (!data[i]) Fatal("CreateFromMats: the data pointer is null" + PartSuffix(nmat, i));
    parts[i] = MatPart{data[i], nrow[i], IsDevicePointer(data[i])};
    first[i + 1] = first[i] + nrow[i];
  }
  if (first[nmat] > std::numeric_limits<int>::max()) Fatal("CreateFromMats: more than 2^31 - 1 rows in all");
  std::unique_ptr<Dataset> d = NewShell(static_cast<int>(first[nmat]), ncol, params);
  StreamTimer timer(d->stream);
  d->SetMappers(reference, true, [&](std::vector<std::vector<double>>* nz, std::vector<std::vector<int>>* nz_rows, int f0, int f1) {      // the sampled rows, gathered where the data is
    const int F = ncol;
    const std::vector<int> rows = d->SampleRows();      // over the concatenated rows
    const int sample_cnt = static_cast<int>(rows.size());
    std::vector<double> S(static_cast<size_t>(sample_cnt) * F);
    // part and row within the part of every sampled row
    std::vector<int> part_of(sample_cnt), local(sample_cnt);
    for (int s = 0; s < sample_cnt; ++s) {
      part_of[s] = static_cast<int>(std::upper_bound(first.begin() + 1, first.end(), static_cast<long long>(rows[s])) - (first.begin() + 1));
      local[s] = static_cast<int>(rows[s] - first[part_of[s]]);
    }
    for (int i = 0; i < nmat; ++i) {
      if (!parts[i].on_device) continue;
      std::vector<int> pos, lrows;      // sample positions in this part, and their rows in it
      for (int s = 0; s < sample_cnt; ++s) if (part_of[s] == i) { pos.push_back(s); lrows.push_back(local[s]); }
      if (pos.empty()) continue;
      const int cnt = static_cast<int>(pos.size());
      std::vector<double> Sp(static_cast<size_t>(cnt) * F);
      DevBuf<int> d_rows; d_rows.Alloc(cnt);
      DevBuf<double> d_S; d_S.Alloc(Sp.size());
      d_rows.Upload(lrows.data(), cnt, d->stream);
      int grid = static_cast<int>(std::min<size_t>((Sp.size() + 255) / 256, static_cast<size_t>(DeviceSMs()) * 32));
      if (data_type == 0) k_gather_rows<float><<<grid, 256, 0, d->stream>>>(static_cast<const float*>(parts[i].data), nrow[i], F, is_row_major, d_rows.p, cnt, d_S.p);
      else k_gather_rows<double><<<grid, 256, 0, d->stream>>>(static_cast<const double*>(parts[i].data), nrow[i], F, is_row_major, d_rows.p, cnt, d_S.p);
      B200_CUDA(cudaGetLastError());
      d_S.Download(Sp.data(), Sp.size(), d->stream);
      B200_CUDA(cudaStreamSynchronize(d->stream));
      for (int j = 0; j < cnt; ++j) std::memcpy(&S[static_cast<size_t>(pos[j]) * F], &Sp[static_cast<size_t>(j) * F], sizeof(double) * F);
    }
#pragma omp parallel for schedule(static)
    for (int s = 0; s < sample_cnt; ++s) {
      const MatPart& p = parts[part_of[s]];
      if (p.on_device) continue;
      const long long r = local[s], n = p.nrow;
      for (int f = 0; f < F; ++f) {
        double v;
        if (data_type == 0) v = is_row_major ? static_cast<const float*>(p.data)[r * F + f] : static_cast<const float*>(p.data)[static_cast<long long>(f) * n + r];
        else v = is_row_major ? static_cast<const double*>(p.data)[r * F + f] : static_cast<const double*>(p.data)[static_cast<long long>(f) * n + r];
        S[static_cast<size_t>(s) * F + f] = v;
      }
    }
    if (nz_rows) { f0 = 0; f1 = F; }
#pragma omp parallel for schedule(dynamic)
    for (int f = f0; f < f1; ++f) {
      for (int s = 0; s < sample_cnt; ++s) {
        double v = S[static_cast<size_t>(s) * F + f];
        if (std::fabs(v) > kZeroThr || std::isnan(v)) {
          (*nz)[f].push_back(v);
          if (nz_rows) (*nz_rows)[f].push_back(s);
        }
      }
    }
    return sample_cnt;
  });
  d->DissolveConflictingBundles([&](unsigned long long* conflicts) {
    const int nb = static_cast<int>(d->bundles.size()), grid = DeviceSMs() * 8;
    d->ForEachDeviceBlock(parts, data_type, is_row_major, [&](const void* x, long long rows, long long ld, long long) {
      if (data_type == 0) k_bundle_conflicts<float><<<grid, 256, 0, d->stream>>>(static_cast<const float*>(x), rows, is_row_major, ld, d->d_members.p, d->d_bundle_start.p, nb, conflicts);
      else k_bundle_conflicts<double><<<grid, 256, 0, d->stream>>>(static_cast<const double*>(x), rows, is_row_major, ld, d->d_members.p, d->d_bundle_start.p, nb, conflicts);
    });
  });
  d->AllocBins();
  d->BinBlock(parts, data_type, is_row_major, 0);
  d->ReleaseIngestStaging();      // every row is in, also when some parts were on the device
  d->ingest_ms = timer.Ms();
  return d.release();
}

// ---- CSR ingestion without densifying (replaces LGBM_DatasetCreateFromCSR, reference call site DatasetAggregator.scala:438-459).
// Bin finding walks the nonzeros of the sampled rows only; binning fills every row of a tile with the features' zero bins and then
// scatters one thread per stored element.  Memory: O(nnz) + the uint8 bins, never nrow x num_col doubles.
// every wide column's default bin; wmeta = meta + nfn
__global__ void k_fill_default_wide(const FeatMeta* __restrict__ wmeta, int nw, uint16_t* __restrict__ bins16, size_t rows_stride, long long nrow) {
  for (long long e = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; e < nrow * nw; e += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int w = static_cast<int>(e / nrow);
    bins16[static_cast<size_t>(w) * rows_stride + (e - static_cast<long long>(w) * nrow)] = static_cast<uint16_t>(wmeta[w].default_bin);
  }
}
// every column's default: a plain feature's default bin, slot 0 of a bundle column (all members at their default bin), 0 for padding
__global__ void k_fill_default_bins(const FeatMeta* __restrict__ meta, const int* __restrict__ col_feat, uint8_t* __restrict__ bins, size_t rows_stride,
                                    long long nrow, int num_tiles) {
  const long long total = nrow * num_tiles * 32;
  for (long long e = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; e < total; e += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int lane = static_cast<int>(e & 31);
    const long long rt = e >> 5;
    const int tile = static_cast<int>(rt / nrow);
    const long long r = rt - static_cast<long long>(tile) * nrow;
    const int u = col_feat[tile * 32 + lane];
    bins[(static_cast<size_t>(tile) * rows_stride + r) * 32 + lane] = u >= 0 ? static_cast<uint8_t>(meta[u].default_bin) : 0;
  }
}
template <typename TI, typename TV>
__global__ void k_bin_csr(const TI* __restrict__ indptr, const int* __restrict__ indices, const TV* __restrict__ vals, long long nrow, const int* __restrict__ inner_of,
                          const FeatMeta* __restrict__ meta, const double* __restrict__ ub, const uint16_t* __restrict__ catbin, uint8_t* __restrict__ bins,
                          size_t rows_stride, long long elem_base, int nfn, uint16_t* __restrict__ bins16, const int* __restrict__ bundle_base) {
  const int lane = threadIdx.x & 31;
  const long long warp = (blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x) >> 5, nwarps = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  for (long long r = warp; r < nrow; r += nwarps) {
    const long long a = static_cast<long long>(indptr[r]) - elem_base, b = static_cast<long long>(indptr[r + 1]) - elem_base;
    for (long long k = a + lane; k < b; k += 32) {
      const int u = inner_of[indices[k]];
      if (u < 0) continue;
      const FeatMeta m = meta[u];
      unsigned bin = d_value_to_bin(static_cast<double>(vals[k]), m, ub + m.table_off, 1, catbin + m.table_off);
      if (u >= nfn) {           // wide column (categorical with > 256 bins, or numerical with max_bin > 255)
        bins16[static_cast<size_t>(u - nfn) * rows_stride + r] = static_cast<uint16_t>(bin);
        continue;
      }
      const int base = bundle_base[u], c = m.hist_off >> 8;
      if (base >= 0) {      // a bundle member: its default bin is the column's slot 0, already filled
        if (bin == static_cast<unsigned>(m.default_bin)) continue;
        bin = d_bundle_slot(bin, base, m.default_bin);
      }
      bins[(static_cast<size_t>(c >> 5) * rows_stride + r) * 32 + (c & 31)] = static_cast<uint8_t>(bin);
    }
  }
}

Dataset* Dataset::CreateFromCSRs(int nparts, const void* const* indptr, int indptr_type, const int32_t* const* indices, const void* const* data,
                                 int data_type, const int64_t* nindptr, const int64_t* nelem, int64_t num_col, const char* params,
                                 const Dataset* reference) {
  EnsureDevice();
  if (num_col <= 0) Fatal("CreateFromCSR: num_col must be given");
  if (num_col > std::numeric_limits<int>::max()) Fatal("CreateFromCSR: too many columns");
  if (indptr_type != 2 && indptr_type != 3) Fatal("CreateFromCSR: indptr must be int32 or int64");
  if (data_type != 0 && data_type != 1) Fatal("Unknown data type in CreateFromCSR (expect C_API_DTYPE_FLOAT32 or FLOAT64)");
  if (nparts < 1) Fatal("CreateFromCSRs: nparts must be at least 1");
  if (!indptr || !indices || !data || !nindptr || !nelem) Fatal("CreateFromCSRs: the part arrays must not be null");
  // indptr entry r of part i, stored value k of part i
  auto ip = [&](int i, int64_t r) -> int64_t { return indptr_type == 2 ? static_cast<const int32_t*>(indptr[i])[r] : static_cast<const int64_t*>(indptr[i])[r]; };
  auto val = [&](int i, int64_t k) -> double { return data_type == 0 ? static_cast<double>(static_cast<const float*>(data[i])[k]) : static_cast<const double*>(data[i])[k]; };
  std::vector<int64_t> first(nparts + 1, 0);      // first row of every part, then the total
  for (int i = 0; i < nparts; ++i) {
    const std::string where = PartSuffix(nparts, i);
    const int64_t nrow = nindptr[i] - 1;
    if (nrow <= 0) Fatal("Dataset should have at least one row and one column" + where);
    if (!indptr[i] || (nelem[i] > 0 && (!indices[i] || !data[i]))) Fatal("CreateFromCSRs: a pointer is null" + where);
    if (ip(i, 0) < 0 || ip(i, nrow) > nelem[i]) Fatal("CreateFromCSR: indptr does not match the number of elements" + where);
    const int32_t* ix = indices[i];
    int bad = 0;
#pragma omp parallel for schedule(static) reduction(| : bad)
    for (int64_t r = 0; r < nrow; ++r) {
      if (ip(i, r) > ip(i, r + 1)) bad |= 1;
      else for (int64_t k = ip(i, r); k < ip(i, r + 1); ++k) if (ix[k] < 0 || ix[k] >= num_col) bad |= 2;
    }
    if (bad & 1) Fatal("CreateFromCSR: indptr is not non-decreasing" + where);
    if (bad & 2) Fatal("CreateFromCSR: a column index is negative or >= num_col" + where);
    first[i + 1] = first[i] + nrow;
  }
  const int64_t nrow = first[nparts];
  if (nrow > std::numeric_limits<int>::max()) Fatal("CreateFromCSR: too many rows for one partition");
  std::unique_ptr<Dataset> d = NewShell(static_cast<int>(nrow), static_cast<int>(num_col), params);
  StreamTimer timer(d->stream);
  const int F = d->num_total_features;
  d->SetMappers(reference, true, [&](std::vector<std::vector<double>>* nz, std::vector<std::vector<int>>* nz_rows, int, int) {
    const std::vector<int> rows = d->SampleRows();      // over the concatenated rows
    for (int s = 0; s < static_cast<int>(rows.size()); ++s) {
      const int i = static_cast<int>(std::upper_bound(first.begin() + 1, first.end(), static_cast<int64_t>(rows[s])) - (first.begin() + 1));
      const int64_t r = rows[s] - first[i];
      for (int64_t k = ip(i, r); k < ip(i, r + 1); ++k) {
        const double v = val(i, k);
        if (std::fabs(v) > kZeroThr || std::isnan(v)) {
          (*nz)[indices[i][k]].push_back(v);
          if (nz_rows) (*nz_rows)[indices[i][k]].push_back(s);
        }
      }
    }
    return static_cast<int>(rows.size());
  });
  const int sms = DeviceSMs();
  // row blocks of bounded element count, part by part: the stored elements are staged through one device buffer per block; fn(indptr,
  // indices, values, rows, first row over all parts, first element in the part) runs on each.  The block staged last stays on the
  // device: when the whole CSR is one block (up to 64M stored values), the bundle row check and the binning share a single upload.
  const size_t isz = indptr_type == 2 ? 4 : 8, vsz = data_type == 0 ? 4 : 8;
  DevBuf<unsigned char> d_ip, d_ix, d_v;
  int staged_part = -1;
  int64_t staged_r0 = -1, staged_r1 = -1;
  auto for_each_block = [&](auto fn) {
    const int64_t kBlockElems = 64LL << 20;
    for (int i = 0; i < nparts; ++i) {
      const int64_t n = first[i + 1] - first[i];
      int64_t r0 = 0;
      while (r0 < n) {
        int64_t r1 = r0 + 1;
        while (r1 < n && ip(i, r1 + 1) - ip(i, r0) <= kBlockElems) ++r1;
        const int64_t e0k = ip(i, r0), ne = ip(i, r1) - e0k, nr = r1 - r0;
        if (i != staged_part || r0 != staged_r0 || r1 != staged_r1) {
          if (d_ip.n < static_cast<size_t>(nr + 1) * isz) d_ip.Alloc(static_cast<size_t>(nr + 1) * isz);
          if (ne > 0) {
            if (d_ix.n < static_cast<size_t>(ne) * 4) d_ix.Alloc(static_cast<size_t>(ne) * 4);
            if (d_v.n < static_cast<size_t>(ne) * vsz) d_v.Alloc(static_cast<size_t>(ne) * vsz);
            B200_CUDA(cudaMemcpyAsync(d_ix.p, indices[i] + e0k, static_cast<size_t>(ne) * 4, cudaMemcpyHostToDevice, d->stream));
            B200_CUDA(cudaMemcpyAsync(d_v.p, static_cast<const unsigned char*>(data[i]) + static_cast<size_t>(e0k) * vsz, static_cast<size_t>(ne) * vsz, cudaMemcpyHostToDevice, d->stream));
          }
          B200_CUDA(cudaMemcpyAsync(d_ip.p, static_cast<const unsigned char*>(indptr[i]) + static_cast<size_t>(r0) * isz, static_cast<size_t>(nr + 1) * isz, cudaMemcpyHostToDevice, d->stream));
          staged_part = i; staged_r0 = r0; staged_r1 = r1;
        }
        if (ne > 0) {
          const int64_t g0 = first[i] + r0;
          if (indptr_type == 2 && data_type == 0) fn(int32_t{}, float{}, nr, g0, e0k);
          else if (indptr_type == 2) fn(int32_t{}, double{}, nr, g0, e0k);
          else if (data_type == 0) fn(int64_t{}, float{}, nr, g0, e0k);
          else fn(int64_t{}, double{}, nr, g0, e0k);
          B200_CUDA(cudaGetLastError());
        }
        B200_CUDA(cudaStreamSynchronize(d->stream));      // the staging buffers are reused by the next block
        r0 = r1;
      }
    }
  };
  d->DissolveConflictingBundles([&](unsigned long long* conflicts) {
    std::vector<int> member_of(F, -1);
    for (size_t k = 0, i = 0; k < d->bundles.size(); ++k) for (int f : d->bundles[k]) member_of[f] = static_cast<int>(i++);
    DevBuf<int> d_member_of; d_member_of.Alloc(F); d_member_of.Upload(member_of.data(), F, d->stream);
    for_each_block([&](auto index_type, auto value_type, int64_t nr, int64_t, int64_t e0k) {
      using TI = decltype(index_type);
      using TV = decltype(value_type);
      const int grid = static_cast<int>(std::min<int64_t>((nr + 7) / 8, sms * 8));
      k_bundle_conflicts_csr<TI, TV><<<grid, 256, 0, d->stream>>>(reinterpret_cast<const TI*>(d_ip.p), reinterpret_cast<const int*>(d_ix.p),
                                                                 reinterpret_cast<const TV*>(d_v.p), nr, e0k, d_member_of.p, d->d_members.p, conflicts);
    });
  });
  d->AllocBins();
  k_fill_default_bins<<<sms * 8, 256, 0, d->stream>>>(d->meta.p, d->d_col_feat.p, d->bins.p, d->rows_stride, nrow, d->num_tiles);
  if (d->nw > 0) k_fill_default_wide<<<sms * 8, 256, 0, d->stream>>>(d->meta.p + d->nfn, d->nw, d->bins16.p, d->rows_stride, nrow);
  B200_CUDA(cudaGetLastError());
  if (d->nf > 0) {
    DevBuf<int> d_inner; d_inner.Alloc(F); d_inner.Upload(d->inner_of.data(), F, d->stream);
    for_each_block([&](auto index_type, auto value_type, int64_t nr, int64_t r0, int64_t e0k) {
      using TI = decltype(index_type);
      using TV = decltype(value_type);
      const int grid = static_cast<int>(std::min<int64_t>((nr + 7) / 8, sms * 8));
      uint8_t* base = d->bins.p + static_cast<size_t>(r0) * 32;       // row offset inside every tile
      k_bin_csr<TI, TV><<<grid, 256, 0, d->stream>>>(reinterpret_cast<const TI*>(d_ip.p), reinterpret_cast<const int*>(d_ix.p),
                                                    reinterpret_cast<const TV*>(d_v.p), nr, d_inner.p, d->meta.p, d->ub.p, d->catbin.p, base,
                                                    d->rows_stride, e0k, d->nfn, d->bins16.p ? d->bins16.p + r0 : nullptr, d->d_bundle_base.p);
    });
  }
  d->ingest_ms = timer.Ms();
  return d.release();
}

void Dataset::SetField(const char* name, const void* data, int n, int type) {
  EnsureDevice();
  std::string s(name);
  auto to_f32 = [&](std::vector<float>* out) {
    out->resize(n);
    if (type == 0) std::memcpy(out->data(), data, sizeof(float) * n);
    else if (type == 1) for (int i = 0; i < n; ++i) (*out)[i] = static_cast<float>(static_cast<const double*>(data)[i]);
    else Fatal("Input type error for field " + s + " (expect float32)");
  };
  if (s == "label" || s == "target") {
    if (n != num_data) Fatal("Length of label is not same with #data");
    to_f32(&label);
    d_label.Alloc(n); d_label.Upload(label.data(), n, stream);
  } else if (s == "weight" || s == "weights") {
    if (n == 0 || data == nullptr) { weight.clear(); d_weight.Free(); return; }
    if (n != num_data) Fatal("Length of weights is not same with #data");
    to_f32(&weight);
    d_weight.Alloc(n); d_weight.Upload(weight.data(), n, stream);
  } else if (s == "init_score") {
    if (n == 0 || data == nullptr) { init_score.clear(); return; }
    if (n % num_data != 0) Fatal("Initial score size doesn't match data size");
    init_score.resize(n);
    if (type == 1) std::memcpy(init_score.data(), data, sizeof(double) * n);
    else if (type == 0) for (int i = 0; i < n; ++i) init_score[i] = static_cast<const float*>(data)[i];
    else Fatal("Input type error for init_score (expect float64)");
  } else if (s == "group" || s == "query") {
    if (type != 2) Fatal("Input type error for group (expect int32)");
    const int32_t* g = static_cast<const int32_t*>(data);
    group_sizes.assign(g, g + n);
    query_boundaries.assign(1, 0);
    for (int i = 0; i < n; ++i) query_boundaries.push_back(query_boundaries.back() + g[i]);
    if (query_boundaries.back() != num_data) Fatal("Sum of query counts is not same with #data");
    d_qb.Alloc(query_boundaries.size()); d_qb.Upload(query_boundaries.data(), query_boundaries.size(), stream);
  } else if (s == "position") {
    if (n == 0 || data == nullptr) { position.clear(); d_position.Free(); return; }
    if (type != 2) Fatal("Input type error for position (expect int32)");
    if (n != num_data) Fatal("Length of position (" + std::to_string(n) + ") is not same with #data (" + std::to_string(num_data) + ")");
    const int32_t* p = static_cast<const int32_t*>(data);
    position.assign(p, p + n);
    d_position.Alloc(n); d_position.Upload(position.data(), n, stream);
  } else {
    Fatal("Unknown field name: " + s);
  }
  B200_CUDA(cudaStreamSynchronize(stream));
}

void Dataset::GetField(const char* name, int* out_len, const void** out_ptr, int* out_type) const {
  std::string s(name);
  if (s == "label" || s == "target") { *out_len = static_cast<int>(label.size()); *out_ptr = label.data(); *out_type = 0; }
  else if (s == "weight" || s == "weights") { *out_len = static_cast<int>(weight.size()); *out_ptr = weight.empty() ? nullptr : weight.data(); *out_type = 0; }
  else if (s == "init_score") { *out_len = static_cast<int>(init_score.size()); *out_ptr = init_score.empty() ? nullptr : init_score.data(); *out_type = 1; }
  else if (s == "group" || s == "query") { *out_len = static_cast<int>(query_boundaries.size()); *out_ptr = query_boundaries.empty() ? nullptr : query_boundaries.data(); *out_type = 2; }
  else if (s == "position") { *out_len = static_cast<int>(position.size()); *out_ptr = position.empty() ? nullptr : position.data(); *out_type = 2; }
  else Fatal("Unknown field name: " + s);
}

void Dataset::GetBundles(int* out_num_columns, int* out_column_of) const {
  *out_num_columns = num_columns + nw;
  for (int f = 0; f < num_total_features; ++f) {
    const int u = inner_of[f];
    out_column_of[f] = u < 0 ? -1 : (u < nfn ? meta_host[u].hist_off >> 8 : num_columns + (u - nfn));
  }
}

void Dataset::SetFeatureNames(const char** names, int n) {
  if (n != num_total_features) Fatal("Size of feature_names error, should equal with total number of features");
  feature_names.assign(n, "");
  for (int i = 0; i < n; ++i) {
    feature_names[i] = names[i];
    for (auto& c : feature_names[i]) if (c == ' ') c = '_';
  }
}

// =============================================================================== booster
}  // namespace b200gbm
#include "tree_learner.cu"      // the booster's tree learner, in this translation unit
#include "forced_splits.h"
namespace b200gbm {

// the voting learner's local and global scans would each need their own draw order of the extra_trees streams; not restated
static const char* const kVotingExtraTrees = "tree_learner=voting does not support extra_trees with more than one machine; "
                                             "use tree_learner=data_parallel or extra_trees=false";
// the voting learner's local scan and vote would need the leaf bounds of every rank's candidates; not restated
static const char* const kVotingMonotone = "tree_learner=voting does not support monotone_constraints with more than one machine; "
                                           "use tree_learner=data_parallel or no monotone_constraints";

// monotone constraints (basic method only): the same checks at LGBM_BoosterCreate and ResetParameter, identical on every rank
static void CheckMonotone(const Config& cfg, const Dataset& train, bool voting_parallel) {
  if (!(cfg.monotone_penalty >= 0.0)) Fatal("monotone_penalty should be >= 0, got " + Config::Num(cfg.monotone_penalty));
  const std::vector<int>& mc = cfg.monotone_constraints;
  if (mc.empty()) return;
  if (cfg.monotone_constraints_method != "basic")
    Fatal("monotone_constraints_method=" + cfg.monotone_constraints_method + " is not supported; use monotone_constraints_method=basic");
  if (static_cast<int>(mc.size()) != train.num_total_features)
    Fatal("monotone_constraints has " + std::to_string(mc.size()) + " entries, but the dataset has " + std::to_string(train.num_total_features) +
          " features");
  for (int f = 0; f < train.num_total_features; ++f) {
    if (mc[f] < -1 || mc[f] > 1) Fatal("monotone_constraints entries should be -1, 0 or 1, got " + std::to_string(mc[f]) + " for feature " + std::to_string(f));
    if (mc[f] != 0 && train.mappers[f].categorical)
      Fatal("monotone_constraints: feature " + std::to_string(f) + " is categorical and cannot carry a monotone constraint");
  }
  if (voting_parallel) Fatal(kVotingMonotone);
}

// the voting learner's local top-k and vote would need every rank's candidates filtered by the leaves' set masks; not restated
static const char* const kVotingInteraction = "tree_learner=voting does not support interaction_constraints with more than one machine; "
                                              "use tree_learner=data_parallel or no interaction_constraints";
constexpr size_t kMaxInteractionSets = 64;      // one 64-bit set mask per leaf (kernels.cuh LeafState::inter_mask)

// interaction constraints: the same checks at LGBM_BoosterCreate and ResetParameter, identical on every rank
static void CheckInteraction(const Config& cfg, const Dataset& train, bool voting_parallel) {
  if (!cfg.interaction_constraints_malformed.empty())
    Fatal("interaction_constraints should be bracketed lists of feature indices like [0,1,2],[2,3], got '" +
          cfg.interaction_constraints_malformed + "'");
  const std::vector<std::vector<int>>& ic = cfg.interaction_constraints;
  if (ic.empty()) return;
  if (ic.size() > kMaxInteractionSets)
    Fatal("interaction_constraints supports at most " + std::to_string(kMaxInteractionSets) + " sets (one 64-bit mask per leaf), got " +
          std::to_string(ic.size()));
  for (size_t s = 0; s < ic.size(); ++s)
    for (int f : ic[s])
      if (f < 0 || f >= train.num_total_features)
        Fatal("interaction_constraints: feature index " + std::to_string(f) + " in set " + std::to_string(s) + " is outside [0, " +
              std::to_string(train.num_total_features) + ")");
  if (voting_parallel) Fatal(kVotingInteraction);
}

// the voting learner's local top-k would need every rank's candidates restricted to the leaves' samples; not restated
static const char* const kVotingByNode = "tree_learner=voting does not support feature_fraction_bynode < 1 with more than one machine; "
                                         "use tree_learner=data_parallel or feature_fraction_bynode=1";

// per-node feature sampling: the same checks at LGBM_BoosterCreate and ResetParameter, identical on every rank
static void CheckByNode(const Config& cfg, bool voting_parallel) {
  const double f = cfg.feature_fraction_bynode;
  if (!(f > 0.0 && f <= 1.0)) Fatal("feature_fraction_bynode should be in (0, 1], got " + Config::Num(f));
  if (f < 1.0 && voting_parallel) Fatal(kVotingByNode);
}

// the voting learner's local scans and vote would need every leaf's output on every rank to smooth toward; not restated
static const char* const kVotingPathSmooth = "tree_learner=voting does not support path_smooth with more than one machine; "
                                             "use tree_learner=data_parallel or path_smooth=0";

// path smoothing: the same checks at LGBM_BoosterCreate and ResetParameter, identical on every rank
static void CheckPathSmooth(const Config& cfg, bool voting_parallel) {
  if (!(cfg.path_smooth >= 0.0)) Fatal("path_smooth should be >= 0, got " + Config::Num(cfg.path_smooth));
  if (cfg.path_smooth > kPathSmoothEps && voting_parallel) Fatal(kVotingPathSmooth);
}

// quantised training: the same checks at LGBM_BoosterCreate and ResetParameter, identical on every rank
// [UPSTREAM 4.1, from knowledge] the position factors' L2 regularisation
static void CheckPositionBias(const Config& cfg) {
  if (!(cfg.lambdarank_position_bias_regularization >= 0.0))
    Fatal("lambdarank_position_bias_regularization should be >= 0, got " + Config::Num(cfg.lambdarank_position_bias_regularization));
}

static void CheckQuantized(const Config& cfg) {
  if (!cfg.use_quantized_grad) return;
  // K4's packed plane flushes a cell after at most floor(32767 / B) additions, and its row chunks are whole 512-row stages
  if (cfg.num_grad_quant_bins < 2 || cfg.num_grad_quant_bins > 63)
    Fatal("num_grad_quant_bins should be in [2, 63] with use_quantized_grad, got " + std::to_string(cfg.num_grad_quant_bins));
  // the renewed leaf outputs would need the bounds and the parent outputs of the scans; not restated
  if (cfg.quant_train_renew_leaf && !cfg.monotone_constraints.empty())
    Fatal("quant_train_renew_leaf does not support monotone_constraints; use quant_train_renew_leaf=false or no monotone_constraints");
  if (cfg.quant_train_renew_leaf && cfg.path_smooth > kPathSmoothEps)
    Fatal("quant_train_renew_leaf does not support path_smooth > 0; use quant_train_renew_leaf=false or path_smooth=0");
}

// the voting learner's local scans and vote would need every rank to evaluate the plan on the global histograms; not restated
static const char* const kVotingForced = "tree_learner=voting does not support forcedsplits_filename with more than one machine; "
                                         "use tree_learner=data_parallel or no forcedsplits_filename";
// upstream tightens the children's bounds after a forced split with the same update as after any split; not restated and tested here
static const char* const kForcedMonotone = "forcedsplits_filename does not support monotone_constraints; "
                                           "use no monotone_constraints or no forcedsplits_filename";

// forced splits: the same checks at LGBM_BoosterCreate and ResetParameter.  Reads and flattens the plan (forced_splits.h).  With several
// ranks every rank then takes part in one all-reduce of (failed, digest, -digest), whatever happened before it, so that all of them fail
// together when any rank could not load its plan or the plans differ, and none is left waiting in a collective.
static std::vector<ForcedNode> CheckForcedSplits(const Config& cfg, const Dataset& train, bool voting_parallel, bool parallel) {
  std::vector<ForcedNode> plan;
  std::string err;
  try {
    plan = LoadForcedPlan(cfg.forcedsplits_filename, train);
  } catch (const std::exception& e) {
    err = "forcedsplits_filename=" + cfg.forcedsplits_filename + ": " + e.what();
  }
  if (err.empty() && !plan.empty() && voting_parallel) err = kVotingForced;
  if (err.empty() && !plan.empty() && !cfg.monotone_constraints.empty()) err = kForcedMonotone;
  if (parallel) {
    const double d = ForcedPlanDigest(plan);
    double v[3] = {err.empty() ? 0.0 : 1.0, d, -d};
    cudaStream_t ts = AcquireStream();
    try { AllReduceHost(v, 3, ncclMax, ts); } catch (...) { ReleaseStream(ts); throw; }
    ReleaseStream(ts);
    if (err.empty() && v[0] > 0.0) err = "forcedsplits_filename: another rank could not load its forced split plan";
    if (err.empty() && v[1] != -v[2]) err = "forcedsplits_filename: the ranks were given different forced split plans";
  }
  if (!err.empty()) Fatal(err);
  return plan;
}

Booster::Booster(const std::string& model_text) : predictor(new Predictor(model, stream_)) {
  std::unique_ptr<HostModel> m = HostModel::FromString(model_text);
  model = std::move(*m);
  K = model.num_tree_per_iteration;
  num_init_iteration = model.NumIterations();
}

Booster::Booster(const Dataset* tr, const char* params) : train(tr), predictor(new Predictor(model, stream_)) {
  EnsureDevice();
  device_ = CurrentDevice();
  cfg.Parse(params);
  if (cfg.boosting != "gbdt" && cfg.boosting != "rf" && cfg.boosting != "goss" && cfg.boosting != "dart")
    Fatal("Unknown boosting type " + cfg.boosting);
  is_rf_ = cfg.boosting == "rf"; is_goss_ = cfg.boosting == "goss"; is_dart_ = cfg.boosting == "dart";
  drop_rand_ = LcgRandom(cfg.drop_seed);
  obj_.reset(new Objective(cfg, *train));
  balanced_bagging_ = cfg.bagging_freq > 0 && (cfg.pos_bagging_fraction < 1.0 || cfg.neg_bagging_fraction < 1.0) && obj_->kind() == ObjectiveKind::kBinary;
  bagging_ = cfg.bagging_freq > 0 && (cfg.bagging_fraction < 1.0 || balanced_bagging_);
  if (bagging_ && !(cfg.bagging_fraction > 0.0)) Fatal("bagging_fraction should be in (0, 1]");
  if (is_goss_) {      // [LightGBM goss.hpp ResetGoss]
    if (!(cfg.top_rate + cfg.other_rate <= 1.0)) Fatal("Check failed: (config_->top_rate + config_->other_rate) <= (1.0f)");
    if (!(cfg.top_rate > 0.0 && cfg.other_rate > 0.0)) Fatal("Check failed: config_->top_rate > 0.0f && config_->other_rate > 0.0f");
    if (bagging_) Fatal("Cannot use bagging in GOSS");
  }
  if (is_rf_) {        // [LightGBM rf.hpp RF::Init]
    const bool ff = cfg.feature_fraction < 1.0 && cfg.feature_fraction > 0.0;
    if (!(bagging_ || ff)) Fatal("Check failed: (config->bagging_freq > 0 && config->bagging_fraction < 1.0f && config->bagging_fraction > 0.0f) || (config->feature_fraction < 1.0f && config->feature_fraction > 0.0f)");
  }
  if (cfg.num_leaves < 2) Fatal("num_leaves should be >= 2");
  metrics_.reset(new Metrics(cfg, *obj_, *train));      // an unknown metric must fail LGBM_BoosterCreate, not the first GetEval in training
  if (train->label.empty()) Fatal("label should not be empty for training");
  K = obj_->NumTreePerIteration();
  parallel_ = Net().active && Net().world > 1;
  same_device_ = parallel_ && Net().same_device != nullptr;
  cfg.num_machines = parallel_ ? Net().world : 1;
  voting_ = parallel_ && cfg.tree_learner == "voting";
  if (voting_) {      // identical on every rank: they all fail here, before any collective of training
    if (cfg.top_k <= 0) Fatal("tree_learner=voting needs top_k > 0, got top_k=" + std::to_string(cfg.top_k));
    if (train->nw > 0)
      Fatal("tree_learner=voting does not support features with more than 256 bins (" + std::to_string(train->nw) +
            " such features); use tree_learner=data_parallel or a max_bin of at most 255");
    if (static_cast<long long>(Net().world) * std::min(cfg.top_k, std::max(train->nf, 1)) > kVoteMaxRecords)
      Fatal("tree_learner=voting supports num_machines * top_k <= " + std::to_string(kVoteMaxRecords) + ", got " + std::to_string(Net().world) +
            " * " + std::to_string(std::min(cfg.top_k, train->nf)));
    if (cfg.extra_trees) Fatal(kVotingExtraTrees);
  }
  CheckMonotone(cfg, *train, voting_);
  CheckInteraction(cfg, *train, voting_);
  CheckByNode(cfg, voting_);
  CheckPathSmooth(cfg, voting_);
  CheckQuantized(cfg);
  CheckPositionBias(cfg);
  const std::vector<ForcedNode> forced_plan = CheckForcedSplits(cfg, *train, voting_, parallel_);
  if (balanced_bagging_) {      // [LightGBM GBDT::ResetBaggingConfig] needs (globally) at least one positive row
    double npos = static_cast<double>(std::count_if(train->label.begin(), train->label.end(), [](float v) { return v > 0; }));
    if (parallel_) {
      cudaStream_t ts = AcquireStream();
      try { AllReduceHost(&npos, 1, ncclSum, ts); } catch (...) { ReleaseStream(ts); throw; }
      ReleaseStream(ts);
    }
    if (!(npos > 0)) { balanced_bagging_ = false; bagging_ = cfg.bagging_freq > 0 && cfg.bagging_fraction < 1.0; }
  }
  shrinkage_ = is_rf_ ? 1.0 : cfg.learning_rate;      // "no shrinkage rate for the RF"
  model.average_output = is_rf_;
  model.num_class = K;
  model.num_tree_per_iteration = K;
  model.label_index = 0;
  model.max_feature_idx = train->num_total_features - 1;
  model.feature_names = train->feature_names;
  for (int f = 0; f < train->num_total_features; ++f) model.feature_infos.push_back(train->mappers[f].InfoString());
  model.monotone_constraints = cfg.monotone_constraints;
  InitTraining();
  learner_->SetForcedPlan(forced_plan);
  model.objective_str = obj_->ToString();
}

Booster::~Booster() {
  learner_.reset();
  for (auto* v : valids_) delete v;
  if (ev_a_) cudaEventDestroy(ev_a_);
  if (ev_b_) cudaEventDestroy(ev_b_);
  ReleaseStream(stream_);
}

void Booster::InitTraining() {
  const int n = train->num_data;
  cudaDeviceProp prop;
  B200_CUDA(cudaGetDeviceProperties(&prop, device_));
  num_sms_ = prop.multiProcessorCount;
  stream_ = AcquireStream();
  B200_CUDA(cudaEventCreate(&ev_a_)); B200_CUDA(cudaEventCreate(&ev_b_));
  score_.Alloc(static_cast<size_t>(K) * n); score_.Zero(stream_);
  grad_.Alloc(static_cast<size_t>(K) * n); hess_.Alloc(static_cast<size_t>(K) * n);
  // init score from the dataset
  if (!train->init_score.empty()) {
    if (train->init_score.size() != static_cast<size_t>(K) * n) Fatal("Initial score size doesn't match data size");
    has_init_score_ = true;
    score_.Upload(train->init_score.data(), train->init_score.size(), stream_);
  }
  obj_->Init(stream_);
  const_hessian_ = obj_->ConstHessian() && !is_goss_;      // GOSS amplifies hessians [LightGBM goss.hpp GetIsConstHessian -> false]
  learner_.reset(new TreeLearner(*train, cfg, *obj_, parallel_, same_device_, num_sms_, stream_, timing));      // after Init: renewal weights
  if (bagging_ || is_goss_) {
    bag_blocks_ = (n + kBagBlock - 1) / kBagBlock;
    std::vector<unsigned> st(bag_blocks_);
    for (int i = 0; i < bag_blocks_; ++i) st[i] = static_cast<unsigned>(cfg.bagging_seed + i);     // bagging_rands_[i] = Random(bagging_seed + i)
    bag_lcg_.Alloc(bag_blocks_); bag_lcg_.Upload(st.data(), st.size(), stream_);
    std::unique_ptr<LcgJump> jt(new LcgJump());
    unsigned a = 1, c = 0;
    for (int j = 0; j < kBagBlock; ++j) { a = a * 214013u; c = c * 214013u + 2531011u; jt->mul[j] = a; jt->add[j] = c; }
    bag_jump_.Alloc(1); bag_jump_.Upload(jt.get(), 1, stream_);
    in_bag_.Alloc(n); bag_block_cnt_.Alloc(bag_blocks_); bag_idx_.Alloc(n); bag_total_.Alloc(1);
    need_re_bagging_ = bagging_;
    B200_CUDA(cudaStreamSynchronize(stream_));
  }
  if (is_rf_) {        // [LightGBM rf.hpp RF::Boosting] gradients are taken once, at the constant init score
    if (!train->init_score.empty()) Fatal("Check failed: train_data->metadata().init_score() == nullptr");
    rf_init_scores_.assign(K, 0.0);
    DevBuf<double> tmp;
    tmp.Alloc(static_cast<size_t>(K) * n); tmp.Zero(stream_);
    for (int k = 0; k < K; ++k) {
      double init = (cfg.boost_from_average && !has_init_score_) ? obj_->BoostFromScore(k) : 0.0;
      if (!(std::fabs(init) > kEps)) init = 0.0;
      rf_init_scores_[k] = init;
      if (init != 0.0) k_add_const<<<num_sms_ * 4, 256, 0, stream_>>>(tmp.p + static_cast<size_t>(k) * n, n, init);
    }
    ComputeGradientsAt(tmp.p);
    B200_CUDA(cudaStreamSynchronize(stream_));
  }
  B200_CUDA(cudaStreamSynchronize(stream_));
}

// ---- DART [LightGBM src/boosting/dart.hpp]
// ScoreUpdater::AddScore(models_[tree], class): the tree's CURRENT host leaf values (after the Shrinkage calls) are pushed into
// its stored device blob and every row walks the tree on its bins.
void Booster::AddStoredTree(int iter_index, int k, bool to_train, bool to_valid) {
  const size_t ti = static_cast<size_t>(num_init_iteration + iter_index) * K + k;
  const HostTree& ht = *model.trees[ti];
  cudaStream_t s = stream_;
  const int n = train->num_data;
  if (ht.num_leaves <= 1) {
    const double v = ht.leaf_value[0];
    if (v != 0.0) {
      if (to_train) k_add_const<<<num_sms_ * 4, 256, 0, s>>>(score_.p + static_cast<size_t>(k) * n, n, v);
      if (to_valid) for (auto* vs : valids_) k_add_const<<<num_sms_ * 4, 256, 0, s>>>(vs->score.p + static_cast<size_t>(k) * vs->ds->num_data, vs->ds->num_data, v);
    }
    return;
  }
  DevBuf<unsigned char>& blob = *tree_store_.at(static_cast<size_t>(iter_index) * K + k);
  TreeDev td = learner_->TreeAt(blob.p);
  B200_CUDA(cudaMemcpyAsync(td.leaf_value, ht.leaf_value.data(), sizeof(double) * ht.num_leaves, cudaMemcpyHostToDevice, s));
  const int egrid = num_sms_ * 8;
  if (to_train) k_add_tree_binned<<<egrid, 256, 0, s>>>(td, train->meta.p, train->View(), n, score_.p + static_cast<size_t>(k) * n, 1.0);
  if (to_valid)
    for (auto* vs : valids_)
      k_add_tree_binned<<<egrid, 256, 0, s>>>(td, vs->ds->meta.p, vs->ds->View(), vs->ds->num_data,
                                              vs->score.p + static_cast<size_t>(k) * vs->ds->num_data, 1.0);
  B200_CUDA(cudaGetLastError());
  B200_CUDA(cudaStreamSynchronize(s));        // the pageable host leaf values must stay put until the copy is done
  timing.launches += (to_train ? 1 : 0) + (to_valid ? static_cast<long long>(valids_.size()) : 0);
}
void Booster::DroppingTrees() {
  drop_index_.clear();
  const bool is_skip = drop_rand_.NextFloat() < cfg.skip_drop;
  if (!is_skip) {
    double drop_rate = cfg.drop_rate;
    if (!cfg.uniform_drop) {
      const double inv_average_weight = static_cast<double>(tree_weight_.size()) / sum_weight_;
      if (cfg.max_drop > 0) drop_rate = std::min(drop_rate, cfg.max_drop * inv_average_weight / sum_weight_);
      for (int i = 0; i < iter; ++i)
        if (drop_rand_.NextFloat() < drop_rate * tree_weight_[i] * inv_average_weight) {
          drop_index_.push_back(i);
          if (drop_index_.size() >= static_cast<size_t>(cfg.max_drop)) break;
        }
    } else {
      if (cfg.max_drop > 0) drop_rate = std::min(drop_rate, cfg.max_drop / static_cast<double>(iter));
      for (int i = 0; i < iter; ++i)
        if (drop_rand_.NextFloat() < drop_rate) {
          drop_index_.push_back(i);
          if (drop_index_.size() >= static_cast<size_t>(cfg.max_drop)) break;
        }
    }
  }
  for (int i : drop_index_)
    for (int k = 0; k < K; ++k) {
      model.trees[static_cast<size_t>(num_init_iteration + i) * K + k]->Shrink(-1.0);
      AddStoredTree(i, k, true, false);
    }
  if (!cfg.xgboost_dart_mode) shrinkage_ = cfg.learning_rate / (1.0f + static_cast<double>(drop_index_.size()));
  else if (drop_index_.empty()) shrinkage_ = cfg.learning_rate;
  else shrinkage_ = cfg.learning_rate / (cfg.learning_rate + static_cast<double>(drop_index_.size()));
  if (!drop_index_.empty()) predictor->Invalidate();
  dart_dropped_this_iter_ = true;
}
void Booster::DartNormalize() {
  const double k = static_cast<double>(drop_index_.size());
  for (int i : drop_index_) {
    for (int c = 0; c < K; ++c) {
      HostTree& t = *model.trees[static_cast<size_t>(num_init_iteration + i) * K + c];
      if (!cfg.xgboost_dart_mode) {
        t.Shrink(1.0f / (k + 1.0f)); AddStoredTree(i, c, false, true);
        t.Shrink(-k); AddStoredTree(i, c, true, false);
      } else {
        t.Shrink(shrinkage_); AddStoredTree(i, c, false, true);
        t.Shrink(-k / cfg.learning_rate); AddStoredTree(i, c, true, false);
      }
    }
    if (!cfg.uniform_drop) {
      if (!cfg.xgboost_dart_mode) { sum_weight_ -= tree_weight_[i] * (1.0f / (k + 1.0f)); tree_weight_[i] *= (k / (k + 1.0f)); }
      else { sum_weight_ -= tree_weight_[i] * (1.0f / (k + cfg.learning_rate)); tree_weight_[i] *= (k / (k + cfg.learning_rate)); }
    }
  }
  if (!drop_index_.empty()) predictor->Invalidate();        // leaf values of earlier trees changed: the device forest for predict is stale
}

// [LightGBM gbdt.cpp GBDT::Bagging / goss.hpp GOSS::Bagging] draws the in-bag flags on the device, compacts the in-bag rows
// (ascending) into bag_idx_; the tree's root leaf is that list.  One small D2H (the bag size) per re-bagging.
void Booster::Bagging(int it) {
  const int n = train->num_data;
  cudaStream_t s = stream_;
  if (is_goss_) {
    use_bag_ = false;
    if (it < static_cast<int>(1.0f / cfg.learning_rate)) return;
    k_goss_draw<<<bag_blocks_, 256, 0, s>>>(bag_lcg_.p, n, K, cfg.top_rate, cfg.other_rate, grad_.p, hess_.p, in_bag_.p, bag_block_cnt_.p);
  } else {
    if (!bagging_) return;
    if (!((use_bag_ && it % cfg.bagging_freq == 0) || need_re_bagging_)) return;
    need_re_bagging_ = false;
    k_bag_draw<<<bag_blocks_, 256, 0, s>>>(bag_lcg_.p, bag_jump_.p, n, cfg.bagging_fraction, in_bag_.p, bag_block_cnt_.p,
                                           balanced_bagging_ ? train->d_label.p : nullptr, cfg.pos_bagging_fraction, cfg.neg_bagging_fraction);
  }
  k_bag_scan<<<1, 1024, 0, s>>>(bag_block_cnt_.p, bag_blocks_, bag_total_.p);
  k_bag_compact<<<bag_blocks_, 256, 0, s>>>(in_bag_.p, bag_block_cnt_.p, n, bag_idx_.p);
  B200_CUDA(cudaGetLastError());
  B200_CUDA(cudaMemcpyAsync(&bag_count_, bag_total_.p, sizeof(int), cudaMemcpyDeviceToHost, s));
  B200_CUDA(cudaStreamSynchronize(s));
  timing.launches += 3;
  use_bag_ = true;
}

double Booster::BoostFromAverage(int k) {
  if (model.trees.empty() && !has_init_score_ && cfg.boost_from_average) {
    double init = obj_->BoostFromScore(k);
    if (std::fabs(init) > kEps) {
      const int n = train->num_data;
      k_add_const<<<num_sms_ * 4, 256, 0, stream_>>>(score_.p + static_cast<size_t>(k) * n, n, init);
      for (auto* v : valids_) k_add_const<<<num_sms_ * 4, 256, 0, stream_>>>(v->score.p + static_cast<size_t>(k) * v->ds->num_data, v->ds->num_data, init);
      B200_CUDA(cudaGetLastError());
      return init;
    }
  }
  return 0.0;
}

void Booster::ComputeGradientsAt(const double* score_p) {
  NvtxRange nvtx("b200gbm:K1/K2 gradients");
  obj_->LaunchGradients(score_p, grad_.p, hess_.p, num_sms_, true);
  B200_CUDA(cudaGetLastError());
  timing.launches += 1;
}

void Booster::SetProfile(bool profile_hist) {
  if (learner_) learner_->profile_hist = profile_hist;
}

void Booster::GetMemoryInfo(int64_t* out2) {
  EnsureDevice();
  size_t free_b = 0, total_b = 0;
  if (cudaMemGetInfo(&free_b, &total_b) != cudaSuccess) { cudaGetLastError(); free_b = 0; }
  out2[0] = learner_ ? static_cast<int64_t>(learner_->ColumnCopyBytes()) : 0;
  out2[1] = static_cast<int64_t>(free_b);
}

void Booster::GetCommInfo(int64_t* out3) const {
  out3[0] = out3[1] = out3[2] = 0;
  if (learner_) learner_->GetCommInfo(out3);
}

void Booster::GetColumnCacheInfo(int64_t* out4) const {
  if (learner_) learner_->GetColumnCacheInfo(out4);
  else std::fill(out4, out4 + 4, 0);
}

// One tree: the learner grows it on class k's (g, h) and renews its leaves; the tree is applied to the training and validation scores
// on the device, then read back.
void Booster::TrainOneTree(int k, HostTree* out) {
  NvtxRange nvtx_tree("b200gbm:tree");
  const Dataset& d = *train;
  const int n = d.num_data;
  double* score_k = score_.p + static_cast<size_t>(k) * n;
  cudaStream_t s = stream_;
  const int egrid = num_sms_ * 8;
  const TreeLearner::Bag bag{in_bag_.p, bag_idx_.p, bag_count_};
  const float* g = grad_.p + static_cast<size_t>(k) * n;
  const float* h = hess_.p + static_cast<size_t>(k) * n;
  learner_->Grow(g, h, const_hessian_, use_bag_ ? &bag : nullptr, iter * K + k);
  if (cfg.use_quantized_grad && cfg.quant_train_renew_leaf) learner_->RenewQuantized(g, h, const_hessian_);
  if (obj_->RenewsLeaves()) learner_->Renew(*obj_, is_rf_ ? nullptr : score_k, is_rf_ ? rf_init_scores_[k] : 0.0);
  // rf keeps scores as the running average of (tree + init score) over the iterations [LightGBM rf.hpp MultiplyScore / UpdateScore]
  const double bias = is_rf_ ? rf_init_scores_[k] : 0.0, pre = is_rf_ ? static_cast<double>(iter + num_init_iteration) : 1.0;
  const double post = is_rf_ ? 1.0 / (iter + num_init_iteration + 1) : 1.0;
  const TreeDev& tree = learner_->Tree();
  if (use_bag_ || is_rf_)      // out-of-bag rows are scored by walking the tree on the binned data, so walk it for every row
    k_add_tree_binned<<<egrid, 256, 0, s>>>(tree, d.meta.p, d.View(), n, score_k, shrinkage_, bias, pre, post);
  else
    learner_->AddScore(score_k, shrinkage_);
  for (auto* v : valids_)
    k_add_tree_binned<<<egrid, 256, 0, s>>>(tree, v->ds->meta.p, v->ds->View(), v->ds->num_data,
                                            v->score.p + static_cast<size_t>(k) * v->ds->num_data, shrinkage_, bias, pre, post);
  timing.launches += 2 + static_cast<long long>(valids_.size());
  B200_CUDA(cudaGetLastError());
  learner_->ReadTree(out);
}

bool Booster::TrainTrees(const float* custom_g, const float* custom_h) {
  NvtxRange nvtx("b200gbm:iteration (LGBM_BoosterUpdateOneIter)");
  if (!train) Fatal("this booster was loaded from a model string and cannot be trained");
  EnsureDevice();
  cudaStream_t s = stream_;
  const int n = train->num_data;
  B200_CUDA(cudaEventRecord(ev_a_, s));
  std::vector<double> init_scores(K, 0.0);
  bool saved_const = const_hessian_;
  if (is_rf_) {
    if (custom_g) Fatal("RF mode do not support custom objective function, please use built-in objectives.");
    init_scores = rf_init_scores_;
  } else if (!custom_g) {
    for (int k = 0; k < K; ++k) init_scores[k] = BoostFromAverage(k);
    if (is_dart_ && !dart_dropped_this_iter_) DroppingTrees();      // GetTrainingScore() in GBDT::Boosting: "only drop one time in one iteration"
    ComputeGradientsAt(score_.p);
  } else {
    grad_.Upload(custom_g, static_cast<size_t>(K) * n, s);
    hess_.Upload(custom_h, static_cast<size_t>(K) * n, s);
    const_hessian_ = false;
    custom_grad_ = true;
  }
  Bagging(iter);
  bool should_continue = is_rf_;        // a random forest never stops early
  for (int k = 0; k < K; ++k) {
    std::unique_ptr<HostTree> t(new HostTree());
    t->Resize(1);
    t->leaf_value[0] = 0;
    if (obj_->NeedTrain(k) && train->nf > 0) TrainOneTree(k, t.get());
    if (t->num_leaves > 1) {
      should_continue = true;
      t->Shrink(shrinkage_);
      if (std::fabs(init_scores[k]) > kEps) t->AddBias(init_scores[k]);
    } else if (static_cast<int>(model.trees.size()) < K) {
      double output = obj_->NeedTrain(k) ? init_scores[k] : obj_->BoostFromScore(k);
      t->MakeConstant(output);
      const double pre = is_rf_ ? static_cast<double>(iter + num_init_iteration) : 1.0, post = is_rf_ ? 1.0 / (iter + num_init_iteration + 1) : 1.0;
      k_scale_add<<<num_sms_ * 4, 256, 0, s>>>(score_.p + static_cast<size_t>(k) * n, n, pre, output, post);
      for (auto* v : valids_) k_scale_add<<<num_sms_ * 4, 256, 0, s>>>(v->score.p + static_cast<size_t>(k) * v->ds->num_data, v->ds->num_data, pre, output, post);
    } else {
      t->MakeConstant(0.0);
    }
    model.trees.push_back(std::move(t));
    if (is_dart_) {       // keep the device form of the tree (bin thresholds, inner bitsets) for later drops
      tree_store_.emplace_back(new DevBuf<unsigned char>());
      const DevBuf<unsigned char>& blob = learner_->Blob();
      tree_store_.back()->Alloc(blob.n);
      B200_CUDA(cudaMemcpyAsync(tree_store_.back()->p, blob.p, blob.n, cudaMemcpyDeviceToDevice, s));
    }
  }
  const_hessian_ = saved_const;
  B200_CUDA(cudaEventRecord(ev_b_, s));
  B200_CUDA(cudaEventSynchronize(ev_b_));
  float ms = 0;
  B200_CUDA(cudaEventElapsedTime(&ms, ev_a_, ev_b_));
  timing.total_ms += ms;
  dart_dropped_this_iter_ = false;
  if (!should_continue) {
    if (static_cast<int>(model.trees.size()) > K) for (int k = 0; k < K; ++k) { model.trees.pop_back(); if (is_dart_) tree_store_.pop_back(); }
    return true;
  }
  ++iter;
  if (is_dart_) {
    DartNormalize();
    if (!cfg.uniform_drop) { tree_weight_.push_back(shrinkage_); sum_weight_ += shrinkage_; }
  }
  return false;
}

bool Booster::UpdateOneIter() { return TrainTrees(nullptr, nullptr); }
bool Booster::UpdateOneIterCustom(const float* grad, const float* hess) { return TrainTrees(grad, hess); }

void Booster::ResetParameter(const char* params) {
  Config nc;
  nc.Parse(params);
  const Config before = cfg;
  for (auto& kv : nc.raw) cfg.raw[kv.first] = kv.second;
  int keep_machines = cfg.num_machines;
  cfg.Refresh();
  cfg.num_machines = keep_machines;
  std::vector<ForcedNode> forced_plan;
  bool reload_plan = false;
  if (train) {      // metrics named by the reset meet the checks of LGBM_BoosterCreate / AddValidData; a rejected reset changes nothing
    try {
      // the voting checks follow the learner built at create: a reset's tree_learner does not change it
      if (voting_ && cfg.extra_trees) Fatal(kVotingExtraTrees);
      CheckMonotone(cfg, *train, voting_);
      CheckInteraction(cfg, *train, voting_);
      CheckByNode(cfg, voting_);
      CheckPathSmooth(cfg, voting_);
      CheckQuantized(cfg);
      CheckPositionBias(cfg);
      // a reset that gives the key (set, changed or cleared) reloads the plan on every rank
      if (nc.raw.count("forcedsplits_filename")) { forced_plan = CheckForcedSplits(cfg, *train, voting_, parallel_); reload_plan = true; }
      else if (learner_ && learner_->HasForcedPlan() && !cfg.monotone_constraints.empty()) Fatal(kForcedMonotone);
      metrics_->Reset(cfg, valids_);      // last: it takes the new metrics only when they pass every check
    } catch (...) {
      cfg = before;
      throw;
    }
  }
  shrinkage_ = is_rf_ ? 1.0 : cfg.learning_rate;
  if (is_dart_) { drop_rand_ = LcgRandom(cfg.drop_seed); sum_weight_ = 0.0; }      // [LightGBM dart.hpp DART::ResetConfig]
  if (train) model.monotone_constraints = cfg.monotone_constraints;
  if (learner_) learner_->ResetConfig(cfg);
  if (learner_ && reload_plan) learner_->SetForcedPlan(forced_plan);
}

void Booster::AddValidData(const Dataset* valid) {
  EnsureDevice();
  if (!train) Fatal("cannot add validation data to a prediction-only booster");
  if (valid->nf != train->nf) Fatal("validation data must be created with reference=train");
  metrics_->CheckData(*valid);
  ValidSet* v = new ValidSet();
  v->ds = valid;
  v->score.Alloc(static_cast<size_t>(K) * valid->num_data);
  v->score.Zero(stream_);
  if (!valid->init_score.empty() && valid->init_score.size() == static_cast<size_t>(K) * valid->num_data)
    v->score.Upload(valid->init_score.data(), valid->init_score.size(), stream_);
  B200_CUDA(cudaStreamSynchronize(stream_));
  valids_.push_back(v);
}

void Booster::MergeFrom(const Booster* other) {
  // [UPSTREAM GBDT::MergeFrom] other's trees first, then ours; scores are NOT replayed
  std::vector<std::unique_ptr<HostTree>> mine = std::move(model.trees);
  model.trees.clear();
  for (auto& t : other->model.trees) model.trees.emplace_back(new HostTree(*t));
  num_init_iteration = static_cast<int>(model.trees.size()) / std::max(K, 1);
  for (auto& t : mine) model.trees.push_back(std::move(t));
}

std::string Booster::SaveModelToString(int start_iteration, int num_iteration, int importance_type) const {
  std::string pb = train ? cfg.ToString() : std::string();
  return model.ToString(start_iteration, num_iteration, importance_type, pb);
}

std::string Booster::DumpModelJson(int start_iteration, int num_iteration) const {
  std::ostringstream s;
  int t0, t1;
  model.IterRange(start_iteration, num_iteration, &t0, &t1);
  s << "{\"name\":\"tree\",\"version\":\"v3\",\"num_class\":" << model.num_class << ",\"num_tree_per_iteration\":" << model.num_tree_per_iteration
    << ",\"label_index\":" << model.label_index << ",\"max_feature_idx\":" << model.max_feature_idx << ",\"objective\":\"" << model.objective_str
    << "\",\"average_output\":" << (model.average_output ? "true" : "false") << ",\"feature_names\":[";
  for (size_t i = 0; i < model.feature_names.size(); ++i) s << (i ? "," : "") << '"' << model.feature_names[i] << '"';
  s << "],\"tree_info\":[";
  char buf[64];
  auto num = [&](double v) { snprintf(buf, sizeof(buf), "%.17g", v); return std::string(buf); };
  for (int t = t0; t < t1; ++t) {
    const HostTree& tr = *model.trees[t];
    s << (t > t0 ? "," : "") << "{\"tree_index\":" << (t - t0) << ",\"num_leaves\":" << tr.num_leaves << ",\"num_cat\":" << (tr.cat_boundaries.empty() ? 0 : static_cast<int>(tr.cat_boundaries.size()) - 1)
      << ",\"shrinkage\":" << num(tr.shrinkage)
      << ",\"tree_structure\":";
    struct Rec { static void node(std::ostringstream& o, const HostTree& tr, int idx, const std::function<std::string(double)>& num) {
      if (idx >= 0) {
        int mt = (tr.decision_type[idx] >> 2) & 3;
        const bool is_cat = (tr.decision_type[idx] & 1) != 0;
        std::string thr = num(tr.threshold[idx]);
        if (is_cat) {       // [UPSTREAM Tree::NodeToJSON]: the categories that go left, joined by "||"
          const int ci = static_cast<int>(tr.threshold[idx]);
          thr = "\"";
          bool first = true;
          for (int wd = tr.cat_boundaries[ci]; wd < tr.cat_boundaries[ci + 1]; ++wd)
            for (int bit = 0; bit < 32; ++bit)
              if ((tr.cat_threshold[wd] >> bit) & 1u) { thr += (first ? "" : "||") + std::to_string((wd - tr.cat_boundaries[ci]) * 32 + bit); first = false; }
          thr += "\"";
        }
        o << "{\"split_index\":" << idx << ",\"split_feature\":" << tr.split_feature[idx] << ",\"split_gain\":" << num(tr.split_gain[idx])
          << ",\"threshold\":" << thr << ",\"decision_type\":\"" << (is_cat ? "==" : "<=") << "\",\"default_left\":" << ((tr.decision_type[idx] & 2) ? "true" : "false")
          << ",\"missing_type\":\"" << (mt == 0 ? "None" : mt == 1 ? "Zero" : "NaN") << "\",\"internal_value\":" << num(tr.internal_value[idx])
          << ",\"internal_weight\":" << num(tr.internal_weight[idx]) << ",\"internal_count\":" << tr.internal_count[idx] << ",\"left_child\":";
        node(o, tr, tr.left_child[idx], num);
        o << ",\"right_child\":";
        node(o, tr, tr.right_child[idx], num);
        o << "}";
      } else {
        int l = ~idx;
        o << "{\"leaf_index\":" << l << ",\"leaf_value\":" << num(tr.leaf_value[l]) << ",\"leaf_weight\":" << num(tr.leaf_weight[l]) << ",\"leaf_count\":" << tr.leaf_count[l] << "}";
      }
    } };
    if (tr.num_leaves <= 1) s << "{\"leaf_value\":" << num(tr.leaf_value[0]) << "}";
    else Rec::node(s, tr, 0, num);
    s << "}";
  }
  s << "],\"feature_importances\":{";
  std::vector<double> imp = model.FeatureImportance(num_iteration, 0);
  bool first = true;
  for (size_t i = 0; i < imp.size() && i < model.feature_names.size(); ++i)
    if (imp[i] > 0) { s << (first ? "" : ",") << '"' << model.feature_names[i] << "\":" << static_cast<long long>(imp[i]); first = false; }
  s << "}}";
  return s.str();
}

// ---- the scores of the training / validation data, and their evaluation ------------------------
std::pair<const Dataset*, const DevBuf<double>*> Booster::ScoredData(int data_idx) const {
  if (data_idx < 0 || data_idx > static_cast<int>(valids_.size())) Fatal("data_idx out of range");
  if (data_idx == 0) return {train, &score_};
  return {valids_[data_idx - 1]->ds, &valids_[data_idx - 1]->score};
}
int64_t Booster::NumPredict(int data_idx) const {
  if (!train) Fatal("this booster was loaded from a model string: it holds no training/validation data (use the predict entry points)");
  return static_cast<int64_t>(K) * ScoredData(data_idx).first->num_data;
}
void Booster::GetPredict(int data_idx, int64_t* out_len, double* out) {
  if (!train) Fatal("this booster was loaded from a model string: it holds no training/validation data (use the predict entry points)");
  EnsureDevice();
  if (is_dart_ && data_idx == 0 && !dart_dropped_this_iter_) DroppingTrees();      // DART::GetTrainingScore
  const int n = ScoredData(data_idx).first->num_data;
  GetRawScores(data_idx, out);
  model.ConvertScores(out, n, 1, n, 0, false);
  *out_len = static_cast<int64_t>(K) * n;
}
void Booster::GetRawScores(int data_idx, double* out) {
  if (!train) Fatal("this booster was loaded from a model string: it holds no training/validation data");
  EnsureDevice();
  const auto [ds, sc] = ScoredData(data_idx);
  sc->Download(out, static_cast<size_t>(K) * ds->num_data, stream_);
  B200_CUDA(cudaStreamSynchronize(stream_));
}
std::vector<std::string> Booster::EvalNames() const { return metrics_ ? metrics_->Names() : std::vector<std::string>(); }
std::vector<double> Booster::GetEval(int data_idx) {
  NvtxRange nvtx("b200gbm:eval metrics (LGBM_BoosterGetEval)");
  if (!train) Fatal("this booster was loaded from a model string: it holds no training/validation data to evaluate");
  EnsureDevice();
  if (is_dart_ && data_idx == 0 && !dart_dropped_this_iter_) DroppingTrees();      // DART::GetTrainingScore
  const auto [ds, sc] = ScoredData(data_idx);
  return metrics_->Eval(sc->p, *ds, stream_);
}

void Booster::GetGradients(float* grad, float* hess) {
  if (!train) Fatal("this booster was loaded from a model string: it holds no training data to take gradients on");
  EnsureDevice();
  const size_t m = static_cast<size_t>(K) * train->num_data;
  DevBuf<float> g, h;      // zero-filled: classes the objective does not train (NeedTrain) read back as 0
  g.Alloc(m); h.Alloc(m); g.Zero(stream_); h.Zero(stream_);
  obj_->LaunchGradients(score_.p, g.p, h.p, num_sms_, false);      // training state (rank_xendcg's random states) unchanged
  B200_CUDA(cudaGetLastError());
  g.Download(grad, m, stream_); h.Download(hess, m, stream_);
  B200_CUDA(cudaStreamSynchronize(stream_));
}

void Booster::GetPositionBias(std::vector<int32_t>* values, std::vector<double>* factors) const {
  values->clear(); factors->clear();
  if (!obj_) return;
  EnsureDevice();
  obj_->PositionBias(values, factors);
}

}  // namespace b200gbm
#include "metrics.cu"      // the booster's metrics, in this translation unit
#include "predictor.cu"    // the booster's batched predictor, in this translation unit
#include "refit.cu"       // the booster's refit, in this translation unit
