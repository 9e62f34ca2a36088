// Row-band communication for the multi-GPU drivers (one process per GPU): a tiny interface -- exchange a row with the
// band above / below, all-reduce a buffer -- with two backends:
//   * NCCL over NVLink (the product path).  libnccl.so.2 is opened at run time, so the library itself has no link-time
//     dependency and loads on a box without NCCL; inside a process that already uses torch.distributed the loader hands
//     back the copy torch brought along.  All calls are stream-ordered on the library's stream.
//   * caller-supplied callbacks (host-synchronous).  Used by the CPU tests to drive the very same C++ band drivers over
//     torch.distributed/gloo with the kernels of the CPU model; never by the product.
// The reference's distributed design is an MPI tile farm with a master rank (programs/parallel_priority_flood/main.cpp);
// here every rank runs the same band driver and only seam rows / small flags / the coarse raster travel.
#include "common.cuh"

#include <dlfcn.h>
#include <memory>

namespace rdb {

namespace {

// the handful of NCCL declarations needed (stable since NCCL 2.7; values from nccl.h)
struct NcclUniqueId {
  char internal[128];
};
typedef void *NcclComm;
enum { kNcclInt32 = 2, kNcclFloat32 = 7, kNcclSum = 0, kNcclMax = 2, kNcclMin = 3 };

struct NcclApi {
  int (*GetUniqueId)(NcclUniqueId *);
  int (*CommInitRank)(NcclComm *, int, NcclUniqueId, int);
  int (*CommDestroy)(NcclComm);
  const char *(*GetErrorString)(int);
  int (*AllReduce)(const void *, void *, size_t, int, int, NcclComm, cudaStream_t);
  int (*Send)(const void *, size_t, int, int, NcclComm, cudaStream_t);
  int (*Recv)(void *, size_t, int, int, NcclComm, cudaStream_t);
  int (*GroupStart)();
  int (*GroupEnd)();
};

NcclApi &nccl() {
  static NcclApi api;
  static bool loaded = false;
  if (loaded) return api;
  void *h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD | RTLD_GLOBAL);  // the copy already in the process (torch's)
  if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
  if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
  if (!h) fail("multi-GPU: libnccl.so.2 not found (%s)", dlerror());
  auto sym = [&](const char *name) {
    void *p = dlsym(h, name);
    if (!p) fail("multi-GPU: %s missing from libnccl", name);
    return p;
  };
  api.GetUniqueId = (decltype(api.GetUniqueId))sym("ncclGetUniqueId");
  api.CommInitRank = (decltype(api.CommInitRank))sym("ncclCommInitRank");
  api.CommDestroy = (decltype(api.CommDestroy))sym("ncclCommDestroy");
  api.GetErrorString = (decltype(api.GetErrorString))sym("ncclGetErrorString");
  api.AllReduce = (decltype(api.AllReduce))sym("ncclAllReduce");
  api.Send = (decltype(api.Send))sym("ncclSend");
  api.Recv = (decltype(api.Recv))sym("ncclRecv");
  api.GroupStart = (decltype(api.GroupStart))sym("ncclGroupStart");
  api.GroupEnd = (decltype(api.GroupEnd))sym("ncclGroupEnd");
  loaded = true;
  return api;
}

void nccl_ck(int rc, const char *what) {
  if (rc != 0) fail("NCCL %s failed: %s", what, nccl().GetErrorString(rc));
}

}  // namespace

}  // namespace rdb

struct rdb200_comm {
  int rank = 0, world = 1;
  rdb::NcclComm nccl = nullptr;
  void *user = nullptr;
  rdb200_exchange_fn exchange = nullptr;
  rdb200_allreduce_fn allreduce = nullptr;
};

namespace rdb {

int comm_rank(const rdb200_comm *c) { return c ? c->rank : 0; }
int comm_world(const rdb200_comm *c) { return c ? c->world : 1; }

// Send `bytes` from send_up to rank-1 and from send_dn to rank+1, receive theirs into recv_up / recv_dn (device
// pointers; the sides without a neighbour are skipped).  Ordered after everything queued on the library's stream.
void comm_exchange(const rdb200_comm *c, const void *send_up, void *recv_up, const void *send_dn, void *recv_dn, size_t bytes) {
  if (!c || c->world == 1) return;
  Ctx &x = ctx();
  const bool up = c->rank > 0, dn = c->rank < c->world - 1;
  if (c->nccl) {
    NcclApi &n = nccl();
    nccl_ck(n.GroupStart(), "group start");
    if (up) {
      nccl_ck(n.Send(send_up, bytes, 0 /* ncclInt8 */, c->rank - 1, c->nccl, x.stream), "send");
      nccl_ck(n.Recv(recv_up, bytes, 0, c->rank - 1, c->nccl, x.stream), "recv");
    }
    if (dn) {
      nccl_ck(n.Send(send_dn, bytes, 0, c->rank + 1, c->nccl, x.stream), "send");
      nccl_ck(n.Recv(recv_dn, bytes, 0, c->rank + 1, c->nccl, x.stream), "recv");
    }
    nccl_ck(n.GroupEnd(), "group end");
    return;
  }
  RDB_CK(cudaStreamSynchronize(x.stream));
  if (c->exchange(c->user, up ? send_up : nullptr, up ? recv_up : nullptr, dn ? send_dn : nullptr, dn ? recv_dn : nullptr, bytes) != 0)
    fail("multi-GPU: the caller's exchange callback failed");
}

// in-place all-reduce; op: RDB200_MAX_F32 / RDB200_MIN_F32 / RDB200_MAX_I32 / RDB200_SUM_I32
void comm_allreduce(const rdb200_comm *c, void *buf, size_t count, int op) {
  if (!c || c->world == 1) return;
  Ctx &x = ctx();
  if (c->nccl) {
    int dt = kNcclFloat32, o = kNcclMax;
    switch (op) {
      case RDB200_MAX_F32: dt = kNcclFloat32; o = kNcclMax; break;
      case RDB200_MIN_F32: dt = kNcclFloat32; o = kNcclMin; break;
      case RDB200_MAX_I32: dt = kNcclInt32; o = kNcclMax; break;
      case RDB200_SUM_I32: dt = kNcclInt32; o = kNcclSum; break;
      default: fail("multi-GPU: unknown reduction %d", op);
    }
    nccl_ck(nccl().AllReduce(buf, buf, count, dt, o, c->nccl, x.stream), "all-reduce");
    return;
  }
  RDB_CK(cudaStreamSynchronize(x.stream));
  if (c->allreduce(c->user, buf, count, op) != 0) fail("multi-GPU: the caller's all-reduce callback failed");
}

// Arguments of a collective band driver.  Every driver calls this before its first collective: a rank that fails here
// must not leave its peers waiting.
void check_band_args(const char *what, const rdb200_comm *comm, const void *d_band, int w, int hloc, int gt, int gb) {
  const int rank = comm_rank(comm), world = comm_world(comm);
  if (!comm || !d_band) fail("%s: null pointer", what);
  if (w < 1 || hloc - (gt ? 1 : 0) - (gb ? 1 : 0) < 1) fail("%s: band has no owned rows (%d x %d)", what, w, hloc);
  if ((gt != 0) != (rank > 0) || (gb != 0) != (rank < world - 1))
    fail("%s: rank %d of %d needs ghost_top = %d and ghost_bottom = %d (got %d, %d)", what, rank, world, rank > 0 ? 1 : 0,
         rank < world - 1 ? 1 : 0, gt, gb);
}

// one edge row of a band array (elem bytes per cell) to each neighbour's ghost row, in place
void exchange_band_rows(const rdb200_comm *comm, void *d_band, size_t elem, int w, int hloc, int gt, int gb) {
  uint8_t *b = static_cast<uint8_t *>(d_band);
  const size_t row = (size_t)w * elem;
  comm_exchange(comm, b + (size_t)gt * row, b, b + (size_t)(hloc - 1 - gb) * row, b + (size_t)(hloc - 1) * row, row);
}

}  // namespace rdb

extern "C" {

int rdb200_nccl_unique_id(uint8_t *out128) {
  return rdb::capi_call([&] {
    if (!out128) rdb::fail("nccl_unique_id: null pointer");
    rdb::NcclUniqueId id;
    rdb::nccl_ck(rdb::nccl().GetUniqueId(&id), "get unique id");
    memcpy(out128, id.internal, 128);
  });
}

int rdb200_comm_create_nccl(rdb200_comm **out, int32_t rank, int32_t world, const uint8_t *id128) {
  return rdb::capi_call([&] {
    rdb::ensure_init();  // the communicator binds to this process's device
    if (!out || !id128 || world < 1 || rank < 0 || rank >= world) rdb::fail("comm_create_nccl: bad arguments");
    auto c = std::make_unique<rdb200_comm>();
    c->rank = rank;
    c->world = world;
    if (world > 1) {
      rdb::NcclUniqueId id;
      memcpy(id.internal, id128, 128);
      rdb::nccl_ck(rdb::nccl().CommInitRank(&c->nccl, world, id, rank), "communicator init");
    }
    *out = c.release();
  });
}

int rdb200_comm_create_callbacks(rdb200_comm **out, int32_t rank, int32_t world, void *user, rdb200_exchange_fn exchange,
                                 rdb200_allreduce_fn allreduce) {
  return rdb::capi_call([&] {
    if (!out || world < 1 || rank < 0 || rank >= world || (world > 1 && (!exchange || !allreduce)))
      rdb::fail("comm_create_callbacks: bad arguments");
    auto *c = new rdb200_comm();
    c->rank = rank;
    c->world = world;
    c->user = user;
    c->exchange = exchange;
    c->allreduce = allreduce;
    *out = c;
  });
}

int rdb200_comm_destroy(rdb200_comm *c) {
  return rdb::capi_call([&] {
    if (c) {
      if (c->nccl) rdb::nccl().CommDestroy(c->nccl);
      delete c;
    }
  });
}

}  // extern "C"
