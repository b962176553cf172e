#ifndef _GNU_SOURCE
#define _GNU_SOURCE
#endif
// Symmetric-memory runtime for one NVSwitch domain (<= 8 GPUs, one process per GPU).
//
// Replaces the Horovod C++ core pieces that own communication memory (fusion buffer
// manager, NCCL communicator bootstrap; SURVEY.md §2.2 N1/N2/N5).  H100-first: memory that
// peers touch is allocated with the CUDA VMM API (cuMemCreate) as POSIX-fd shareable
// handles, the fds are passed between the ranks' processes with SCM_RIGHTS over abstract
// unix sockets, every rank maps every peer's allocation into its own VA space (P2P over
// NVLink) and, when the fabric supports it, all ranks bind the same physical pages to one
// multicast object (NVLS: multimem.ld_reduce / multimem.st execute in the NVSwitch).
//
// Pure C ABI, called from Python through ctypes (runtime/symm.py).  No torch headers.
// Driver entry points are resolved at run time through cudaGetDriverEntryPoint, so the
// library links against the CUDA runtime only and builds on a machine without a driver.
#include <cuda.h>
#include <cuda_runtime.h>

#include <errno.h>
#include <poll.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <sys/socket.h>
#include <sys/un.h>
#include <unistd.h>

#include <mutex>
#include <string>

namespace {

thread_local std::string g_err;
std::mutex g_mu;

int fail(const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_err = buf;
  return -1;
}

#define DRV_FN(name) decltype(&name) p_##name = nullptr
struct Driver {
  bool loaded = false;
  DRV_FN(cuGetErrorString);
  DRV_FN(cuDeviceGet);
  DRV_FN(cuDeviceGetAttribute);
  DRV_FN(cuMemGetAllocationGranularity);
  DRV_FN(cuMemCreate);
  DRV_FN(cuMemRelease);
  DRV_FN(cuMemExportToShareableHandle);
  DRV_FN(cuMemImportFromShareableHandle);
  DRV_FN(cuMemAddressReserve);
  DRV_FN(cuMemAddressFree);
  DRV_FN(cuMemMap);
  DRV_FN(cuMemUnmap);
  DRV_FN(cuMemSetAccess);
  DRV_FN(cuMulticastCreate);
  DRV_FN(cuMulticastAddDevice);
  DRV_FN(cuMulticastBindMem);
  DRV_FN(cuMulticastUnbind);
  DRV_FN(cuMulticastGetGranularity);
} drv;

template <typename T>
bool resolve(const char* name, T* out, bool required) {
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult st;
  cudaError_t e = cudaGetDriverEntryPoint(name, &fn, cudaEnableDefault, &st);
  if (e != cudaSuccess || st != cudaDriverEntryPointSuccess || fn == nullptr) {
    cudaGetLastError();
    *out = nullptr;
    if (required) fail("driver entry point %s not available (%s)", name, cudaGetErrorString(e));
    return false;
  }
  *out = reinterpret_cast<T>(fn);
  return true;
}

int drv_check(CUresult r, const char* what) {
  if (r == CUDA_SUCCESS) return 0;
  const char* s = "?";
  if (drv.p_cuGetErrorString) drv.p_cuGetErrorString(r, &s);
  return fail("%s failed: CUresult %d (%s)", what, (int)r, s ? s : "?");
}
#define DRV(call, what) do { if (drv_check((call), what)) return -1; } while (0)

CUmemAllocationProp alloc_prop(int device) {
  CUmemAllocationProp p;
  memset(&p, 0, sizeof(p));
  p.type = CU_MEM_ALLOCATION_TYPE_PINNED;
  p.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
  p.location.id = device;
  p.requestedHandleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
  return p;
}

}  // namespace

extern "C" {

const char* b200dp_last_error() { return g_err.c_str(); }

// Resolve driver entry points and make sure the primary context of `device` exists.
int b200dp_rt_init(int device) {
  std::lock_guard<std::mutex> lk(g_mu);
  cudaError_t e = cudaSetDevice(device);
  if (e != cudaSuccess) return fail("cudaSetDevice(%d): %s", device, cudaGetErrorString(e));
  e = cudaFree(0);
  if (e != cudaSuccess) return fail("cudaFree(0): %s", cudaGetErrorString(e));
  if (drv.loaded) return 0;
  bool ok = true;
  ok &= resolve("cuGetErrorString", &drv.p_cuGetErrorString, true);
  ok &= resolve("cuDeviceGet", &drv.p_cuDeviceGet, true);
  ok &= resolve("cuDeviceGetAttribute", &drv.p_cuDeviceGetAttribute, true);
  ok &= resolve("cuMemGetAllocationGranularity", &drv.p_cuMemGetAllocationGranularity, true);
  ok &= resolve("cuMemCreate", &drv.p_cuMemCreate, true);
  ok &= resolve("cuMemRelease", &drv.p_cuMemRelease, true);
  ok &= resolve("cuMemExportToShareableHandle", &drv.p_cuMemExportToShareableHandle, true);
  ok &= resolve("cuMemImportFromShareableHandle", &drv.p_cuMemImportFromShareableHandle, true);
  ok &= resolve("cuMemAddressReserve", &drv.p_cuMemAddressReserve, true);
  ok &= resolve("cuMemAddressFree", &drv.p_cuMemAddressFree, true);
  ok &= resolve("cuMemMap", &drv.p_cuMemMap, true);
  ok &= resolve("cuMemUnmap", &drv.p_cuMemUnmap, true);
  ok &= resolve("cuMemSetAccess", &drv.p_cuMemSetAccess, true);
  if (!ok) return -1;
  // multicast is optional (absent on pre-12.1 drivers / non-NVSwitch fabrics)
  resolve("cuMulticastCreate", &drv.p_cuMulticastCreate, false);
  resolve("cuMulticastAddDevice", &drv.p_cuMulticastAddDevice, false);
  resolve("cuMulticastBindMem", &drv.p_cuMulticastBindMem, false);
  resolve("cuMulticastUnbind", &drv.p_cuMulticastUnbind, false);
  resolve("cuMulticastGetGranularity", &drv.p_cuMulticastGetGranularity, false);
  drv.loaded = true;
  return 0;
}

// caps[0]=VMM supported, [1]=posix-fd handles, [2]=multicast, [3]=SM count, [4]=cc major, [5]=cc minor
int b200dp_rt_caps(int device, int* caps, size_t* gran, size_t* mc_gran, int ndev_for_mc) {
  if (!drv.loaded) return fail("runtime not initialised");
  CUdevice dev;
  DRV(drv.p_cuDeviceGet(&dev, device), "cuDeviceGet");
  int v = 0;
  DRV(drv.p_cuDeviceGetAttribute(&v, CU_DEVICE_ATTRIBUTE_VIRTUAL_MEMORY_MANAGEMENT_SUPPORTED, dev),
      "attr VMM");
  caps[0] = v;
  DRV(drv.p_cuDeviceGetAttribute(&v, CU_DEVICE_ATTRIBUTE_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR_SUPPORTED,
                                 dev), "attr posix fd");
  caps[1] = v;
  v = 0;
  if (drv.p_cuMulticastCreate != nullptr) {
    if (drv.p_cuDeviceGetAttribute(&v, CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED, dev) != CUDA_SUCCESS)
      v = 0;
  }
  caps[2] = v;
  DRV(drv.p_cuDeviceGetAttribute(&v, CU_DEVICE_ATTRIBUTE_MULTIPROCESSOR_COUNT, dev), "attr SMs");
  caps[3] = v;
  DRV(drv.p_cuDeviceGetAttribute(&v, CU_DEVICE_ATTRIBUTE_COMPUTE_CAPABILITY_MAJOR, dev), "attr cc");
  caps[4] = v;
  DRV(drv.p_cuDeviceGetAttribute(&v, CU_DEVICE_ATTRIBUTE_COMPUTE_CAPABILITY_MINOR, dev), "attr cc");
  caps[5] = v;
  CUmemAllocationProp p = alloc_prop(device);
  DRV(drv.p_cuMemGetAllocationGranularity(gran, &p, CU_MEM_ALLOC_GRANULARITY_RECOMMENDED),
      "cuMemGetAllocationGranularity");
  *mc_gran = 0;
  if (caps[2] && ndev_for_mc > 1) {
    CUmulticastObjectProp mp;
    memset(&mp, 0, sizeof(mp));
    mp.numDevices = ndev_for_mc;
    mp.size = *gran;
    mp.handleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
    size_t g = 0;
    if (drv.p_cuMulticastGetGranularity(&g, &mp, CU_MULTICAST_GRANULARITY_MINIMUM) ==
        CUDA_SUCCESS)
      *mc_gran = g;
    else
      caps[2] = 0;
  }
  return 0;
}

// ---- physical allocation -------------------------------------------------------------
int b200dp_mem_create(int device, size_t bytes, uint64_t* handle_out, int* fd_out) {
  if (!drv.loaded) return fail("runtime not initialised");
  CUmemAllocationProp p = alloc_prop(device);
  CUmemGenericAllocationHandle h;
  DRV(drv.p_cuMemCreate(&h, bytes, &p, 0), "cuMemCreate");
  int fd = -1;
  CUresult r = drv.p_cuMemExportToShareableHandle(&fd, h, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0);
  if (r != CUDA_SUCCESS) {
    drv.p_cuMemRelease(h);
    return drv_check(r, "cuMemExportToShareableHandle");
  }
  *handle_out = (uint64_t)h;
  *fd_out = fd;
  return 0;
}

int b200dp_mem_import(int fd, uint64_t* handle_out) {
  if (!drv.loaded) return fail("runtime not initialised");
  CUmemGenericAllocationHandle h;
  DRV(drv.p_cuMemImportFromShareableHandle(&h, (void*)(uintptr_t)fd,
                                           CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR),
      "cuMemImportFromShareableHandle");
  *handle_out = (uint64_t)h;
  return 0;
}

// Reserve a VA range, map `handle` (unicast allocation or multicast object) and grant RW.
int b200dp_mem_map(int device, uint64_t handle, size_t bytes, size_t align, uint64_t* va_out) {
  if (!drv.loaded) return fail("runtime not initialised");
  CUdeviceptr va = 0;
  DRV(drv.p_cuMemAddressReserve(&va, bytes, align, 0, 0), "cuMemAddressReserve");
  CUresult r = drv.p_cuMemMap(va, bytes, 0, (CUmemGenericAllocationHandle)handle, 0);
  if (r != CUDA_SUCCESS) {
    drv.p_cuMemAddressFree(va, bytes);
    return drv_check(r, "cuMemMap");
  }
  CUmemAccessDesc acc;
  memset(&acc, 0, sizeof(acc));
  acc.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
  acc.location.id = device;
  acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
  r = drv.p_cuMemSetAccess(va, bytes, &acc, 1);
  if (r != CUDA_SUCCESS) {
    drv.p_cuMemUnmap(va, bytes);
    drv.p_cuMemAddressFree(va, bytes);
    return drv_check(r, "cuMemSetAccess");
  }
  *va_out = (uint64_t)va;
  return 0;
}

int b200dp_mem_unmap(uint64_t va, size_t bytes) {
  if (!drv.loaded) return fail("runtime not initialised");
  DRV(drv.p_cuMemUnmap((CUdeviceptr)va, bytes), "cuMemUnmap");
  DRV(drv.p_cuMemAddressFree((CUdeviceptr)va, bytes), "cuMemAddressFree");
  return 0;
}

int b200dp_mem_release(uint64_t handle) {
  if (!drv.loaded) return fail("runtime not initialised");
  DRV(drv.p_cuMemRelease((CUmemGenericAllocationHandle)handle), "cuMemRelease");
  return 0;
}

// ---- multicast (NVLS) ------------------------------------------------------------------
int b200dp_mc_create(int ndev, size_t bytes, uint64_t* handle_out, int* fd_out) {
  if (!drv.loaded || !drv.p_cuMulticastCreate) return fail("multicast not available");
  CUmulticastObjectProp mp;
  memset(&mp, 0, sizeof(mp));
  mp.numDevices = ndev;
  mp.size = bytes;
  mp.handleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
  CUmemGenericAllocationHandle h;
  DRV(drv.p_cuMulticastCreate(&h, &mp), "cuMulticastCreate");
  int fd = -1;
  CUresult r = drv.p_cuMemExportToShareableHandle(&fd, h, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0);
  if (r != CUDA_SUCCESS) {
    drv.p_cuMemRelease(h);
    return drv_check(r, "cuMemExportToShareableHandle(multicast)");
  }
  *handle_out = (uint64_t)h;
  *fd_out = fd;
  return 0;
}

int b200dp_mc_add_device(uint64_t mc, int device) {
  if (!drv.loaded || !drv.p_cuMulticastAddDevice) return fail("multicast not available");
  CUdevice dev;
  DRV(drv.p_cuDeviceGet(&dev, device), "cuDeviceGet");
  DRV(drv.p_cuMulticastAddDevice((CUmemGenericAllocationHandle)mc, dev), "cuMulticastAddDevice");
  return 0;
}

int b200dp_mc_bind(uint64_t mc, size_t mc_off, uint64_t mem, size_t mem_off, size_t bytes) {
  if (!drv.loaded || !drv.p_cuMulticastBindMem) return fail("multicast not available");
  DRV(drv.p_cuMulticastBindMem((CUmemGenericAllocationHandle)mc, mc_off,
                               (CUmemGenericAllocationHandle)mem, mem_off, bytes, 0),
      "cuMulticastBindMem");
  return 0;
}

int b200dp_mc_unbind(uint64_t mc, int device, size_t mc_off, size_t bytes) {
  if (!drv.loaded || !drv.p_cuMulticastUnbind) return fail("multicast not available");
  CUdevice dev;
  DRV(drv.p_cuDeviceGet(&dev, device), "cuDeviceGet");
  DRV(drv.p_cuMulticastUnbind((CUmemGenericAllocationHandle)mc, dev, mc_off, bytes),
      "cuMulticastUnbind");
  return 0;
}

// ---- fd passing over abstract unix sockets (SCM_RIGHTS) --------------------------------
static int make_addr(const char* name, sockaddr_un* addr, socklen_t* len) {
  memset(addr, 0, sizeof(*addr));
  addr->sun_family = AF_UNIX;
  size_t n = strlen(name);
  if (n + 2 > sizeof(addr->sun_path)) return fail("socket name too long: %s", name);
  addr->sun_path[0] = '\0';  // abstract namespace: no filesystem entry, dies with the process
  memcpy(addr->sun_path + 1, name, n);
  *len = (socklen_t)(offsetof(sockaddr_un, sun_path) + 1 + n);
  return 0;
}

int b200dp_fd_listen(const char* name) {
  sockaddr_un addr;
  socklen_t len;
  if (make_addr(name, &addr, &len)) return -1;
  int s = socket(AF_UNIX, SOCK_STREAM | SOCK_CLOEXEC, 0);
  if (s < 0) return fail("socket(): %s", strerror(errno));
  if (bind(s, (sockaddr*)&addr, len) < 0) {
    int e = errno;
    close(s);
    return fail("bind(@%s): %s", name, strerror(e));
  }
  if (listen(s, 64) < 0) {
    int e = errno;
    close(s);
    return fail("listen(@%s): %s", name, strerror(e));
  }
  return s;
}

// Connect (retrying until timeout_ms) to `peer_name` and send `fd` tagged with (src, tag).
int b200dp_fd_send(const char* peer_name, int fd, int src, int tag, int timeout_ms) {
  sockaddr_un addr;
  socklen_t len;
  if (make_addr(peer_name, &addr, &len)) return -1;
  int s = -1;
  int waited = 0;
  for (;;) {
    s = socket(AF_UNIX, SOCK_STREAM | SOCK_CLOEXEC, 0);
    if (s < 0) return fail("socket(): %s", strerror(errno));
    if (connect(s, (sockaddr*)&addr, len) == 0) break;
    int e = errno;
    close(s);
    if (waited >= timeout_ms) return fail("connect(@%s): %s", peer_name, strerror(e));
    usleep(20 * 1000);
    waited += 20;
  }
  int hdr[2] = {src, tag};
  struct iovec iov;
  iov.iov_base = hdr;
  iov.iov_len = sizeof(hdr);
  char ctrl[CMSG_SPACE(sizeof(int))];
  memset(ctrl, 0, sizeof(ctrl));
  struct msghdr msg;
  memset(&msg, 0, sizeof(msg));
  msg.msg_iov = &iov;
  msg.msg_iovlen = 1;
  msg.msg_control = ctrl;
  msg.msg_controllen = sizeof(ctrl);
  struct cmsghdr* c = CMSG_FIRSTHDR(&msg);
  c->cmsg_level = SOL_SOCKET;
  c->cmsg_type = SCM_RIGHTS;
  c->cmsg_len = CMSG_LEN(sizeof(int));
  memcpy(CMSG_DATA(c), &fd, sizeof(int));
  ssize_t n = sendmsg(s, &msg, 0);
  int e = errno;
  // Once sendmsg returns the kernel holds its own reference to the file in the socket
  // buffer, so the caller may close `fd` immediately; no ack round-trip is needed (and not
  // having one lets every rank send first and receive afterwards without deadlock).
  close(s);
  if (n != (ssize_t)sizeof(hdr)) return fail("sendmsg(@%s): %s", peer_name, strerror(e));
  return 0;
}

// Accept one connection on `listen_fd`; returns the received fd (>= 0) and fills src/tag.
int b200dp_fd_recv(int listen_fd, int* src, int* tag, int timeout_ms) {
  struct pollfd pfd = {listen_fd, POLLIN, 0};
  int pr = poll(&pfd, 1, timeout_ms);
  if (pr <= 0) return fail("timed out waiting for a peer fd (%d ms)", timeout_ms);
  int s = accept4(listen_fd, nullptr, nullptr, SOCK_CLOEXEC);
  if (s < 0) return fail("accept(): %s", strerror(errno));
  {  // abstract socket names are visible to every local user: only accept handles from our own uid
    struct ucred cred;
    socklen_t clen = sizeof(cred);
    if (getsockopt(s, SOL_SOCKET, SO_PEERCRED, &cred, &clen) != 0 || cred.uid != geteuid()) {
      close(s);
      return fail("fd_recv: rejected a connection from uid %d (expected %d)", (int)cred.uid, (int)geteuid());
    }
  }
  int hdr[2] = {-1, -1};
  struct iovec iov;
  iov.iov_base = hdr;
  iov.iov_len = sizeof(hdr);
  char ctrl[CMSG_SPACE(sizeof(int))];
  memset(ctrl, 0, sizeof(ctrl));
  struct msghdr msg;
  memset(&msg, 0, sizeof(msg));
  msg.msg_iov = &iov;
  msg.msg_iovlen = 1;
  msg.msg_control = ctrl;
  msg.msg_controllen = sizeof(ctrl);
  ssize_t n = recvmsg(s, &msg, MSG_CMSG_CLOEXEC);
  int fd = -1;
  if (n == (ssize_t)sizeof(hdr)) {
    for (struct cmsghdr* c = CMSG_FIRSTHDR(&msg); c; c = CMSG_NXTHDR(&msg, c)) {
      if (c->cmsg_level == SOL_SOCKET && c->cmsg_type == SCM_RIGHTS) {
        memcpy(&fd, CMSG_DATA(c), sizeof(int));
        break;
      }
    }
  }
  close(s);
  if (fd < 0) return fail("recvmsg(): no fd received (n=%zd, %s)", n, strerror(errno));
  *src = hdr[0];
  *tag = hdr[1];
  return fd;
}

int b200dp_fd_close(int fd) { return close(fd); }

// ---- misc helpers ----------------------------------------------------------------------
// Host-pinned, device-mapped word(s) used as the kernels' error/watchdog mailbox.
int b200dp_host_mailbox(size_t bytes, uint64_t* host_ptr, uint64_t* dev_ptr) {
  void* h = nullptr;
  cudaError_t e = cudaHostAlloc(&h, bytes, cudaHostAllocMapped | cudaHostAllocPortable);
  if (e != cudaSuccess) return fail("cudaHostAlloc: %s", cudaGetErrorString(e));
  memset(h, 0, bytes);
  void* d = nullptr;
  e = cudaHostGetDevicePointer(&d, h, 0);
  if (e != cudaSuccess) return fail("cudaHostGetDevicePointer: %s", cudaGetErrorString(e));
  *host_ptr = (uint64_t)(uintptr_t)h;
  *dev_ptr = (uint64_t)(uintptr_t)d;
  return 0;
}

int b200dp_memset_async(uint64_t ptr, int value, size_t bytes, uint64_t stream) {
  cudaError_t e = cudaMemsetAsync((void*)(uintptr_t)ptr, value, bytes, (cudaStream_t)(uintptr_t)stream);
  if (e != cudaSuccess) return fail("cudaMemsetAsync: %s", cudaGetErrorString(e));
  return 0;
}

int b200dp_can_access_peer(int dev, int peer) {
  int ok = 0;
  cudaError_t e = cudaDeviceCanAccessPeer(&ok, dev, peer);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return ok;
}

}  // extern "C"
