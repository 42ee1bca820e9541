// infer.cu — the inference-time twin of the Categorify / FillMissing transforms for HOST
// arrays (dict-of-numpy in, dict-of-numpy out), replacing the reference's pybind11 module
// nvtabular_cpp.inference (cpp/nvtabular/inference/categorify.cc:31-347, fill.cc:32-124;
// entry points nvtabular/ops/categorify.py:602-609, ops/fill.py:59-65).
//
// Serving batches are tens to thousands of rows: a PCIe round trip plus a kernel launch costs
// more than probing a host table, so — like the reference — this path stays on the CPU: an
// open-addressing table of the kept keys (built once from the device vocabulary), probed by a
// few host threads.  Labels are bit-identical to the device encode (same label space, same
// pandas value hash for the OOV buckets).  Large batches belong on the device path
// (nvtb_encode_apply) — the Python wrapper picks by where the arrays live.
#include <cstdint>
#include <cstring>
#include <new>
#include <thread>
#include <vector>

#include "common.cuh"


struct nvtb_infer_vocab {
  std::vector<int64_t> slots;      // key, position pairs; key == kEmptyKey: free
  int64_t capacity;                // power of two
  int64_t n;
  int64_t min_key_pos;             // position of the key equal to the sentinel, or -1
};

namespace {

inline int64_t host_find(const nvtb_infer_vocab* v, int64_t key) {
  if (key == nvtb::kEmptyKey) return v->min_key_pos;
  const int64_t mask = v->capacity - 1;
  int64_t s = (int64_t)(nvtb::table_mix64((uint64_t)key) & (uint64_t)mask);
  for (;;) {
    const int64_t k = v->slots[2 * s];
    if (k == key) return v->slots[2 * s + 1];
    if (k == nvtb::kEmptyKey) return -1;
    s = (s + 1) & mask;
  }
}

template <typename KeyT, typename OutT>
void encode_range(const nvtb_infer_vocab* v, const KeyT* keys, const uint8_t* validity, int64_t lo, int64_t hi,
                  int64_t null_label, int64_t oov_label, int64_t first_label, uint64_t num_buckets, OutT* out) {
  for (int64_t i = lo; i < hi; ++i) {
    if (validity != nullptr && !((validity[i >> 3] >> (i & 7)) & 1)) { out[i] = (OutT)null_label; continue; }
    const KeyT x = keys[i];
    const int64_t pos = host_find(v, (int64_t)x);
    if (pos >= 0) { out[i] = (OutT)(first_label + pos); continue; }
    int64_t lab = oov_label;
    if (num_buckets > 1) lab += (int64_t)(nvtb::pandas_mix64(nvtb::value_bits<KeyT>(x)) % num_buckets);
    out[i] = (OutT)lab;
  }
}

template <typename F>
void run_threads(int64_t n, int n_threads, F f) {
  const int64_t kMinPerThread = 1 << 14;
  int t = n_threads > 0 ? n_threads : (int)std::thread::hardware_concurrency();
  if (t < 1) t = 1;
  if ((int64_t)t > (n + kMinPerThread - 1) / kMinPerThread) t = (int)((n + kMinPerThread - 1) / kMinPerThread);
  if (t <= 1) { f(0, n); return; }
  std::vector<std::thread> th;
  const int64_t chunk = (n + t - 1) / t;
  for (int j = 0; j < t; ++j) {
    const int64_t lo = j * chunk, hi = lo + chunk < n ? lo + chunk : n;
    if (lo < hi) th.emplace_back(f, lo, hi);
  }
  for (auto& x : th) x.join();
}

}  // namespace

extern "C" {

int nvtb_infer_vocab_create(nvtb_infer_vocab_t** out, const int64_t* keys_host, int64_t n) {
  NVTB_REQUIRE(out != nullptr && n >= 0 && (n == 0 || keys_host != nullptr), "bad arguments");
  nvtb_infer_vocab* v = new (std::nothrow) nvtb_infer_vocab();
  NVTB_REQUIRE(v != nullptr, "host allocation failed");
  int64_t cap = 16;
  while (cap < 2 * n) cap <<= 1;
  v->capacity = cap;
  v->n = n;
  v->min_key_pos = -1;
  try {
    v->slots.assign((size_t)(2 * cap), nvtb::kEmptyKey);
  } catch (...) {
    delete v;
    nvtb::set_error("nvtb_infer_vocab_create: host allocation failed");
    return NVTB_ENOMEM;
  }
  const int64_t mask = cap - 1;
  for (int64_t i = 0; i < n; ++i) {
    const int64_t key = keys_host[i];
    if (key == nvtb::kEmptyKey) {                      // first wins here too
      if (v->min_key_pos < 0) v->min_key_pos = i;
      continue;
    }
    int64_t s = (int64_t)(nvtb::table_mix64((uint64_t)key) & (uint64_t)mask);
    while (v->slots[2 * s] != nvtb::kEmptyKey && v->slots[2 * s] != key) s = (s + 1) & mask;
    if (v->slots[2 * s] == nvtb::kEmptyKey) { v->slots[2 * s] = key; v->slots[2 * s + 1] = i; }   // first wins
  }
  *out = v;
  return NVTB_OK;
}

int nvtb_infer_vocab_from_device(nvtb_infer_vocab_t** out, const nvtb_vocab_t* dv, void* stream) {
  NVTB_REQUIRE(out != nullptr && dv != nullptr, "NULL argument");
  nvtb_vocab_info_t info;
  int rc = nvtb_vocab_info(dv, &info);
  if (rc) return rc;
  const int64_t n = info.n_kept;
  std::vector<int64_t> host((size_t)(n > 0 ? n : 1));
  if (n > 0) {
    int64_t* d = nullptr;
    cudaStream_t st = (cudaStream_t)stream;
    NVTB_CUDA_OK(cudaMallocAsync(&d, sizeof(int64_t) * (size_t)n, st));
    rc = nvtb_vocab_export(dv, d, nullptr, stream);
    if (rc) { cudaFreeAsync(d, st); return rc; }
    NVTB_CUDA_OK(cudaMemcpyAsync(host.data(), d, sizeof(int64_t) * (size_t)n, cudaMemcpyDeviceToHost, st));
    NVTB_CUDA_OK(cudaFreeAsync(d, st));
    NVTB_CUDA_OK(cudaStreamSynchronize(st));
  }
  return nvtb_infer_vocab_create(out, host.data(), n);
}

int nvtb_infer_vocab_destroy(nvtb_infer_vocab_t* v) {
  delete v;
  return NVTB_OK;
}

int nvtb_infer_categorify_host(const nvtb_infer_vocab_t* v, const void* keys_host, int key_dtype,
                               const uint8_t* validity_host, int64_t n, int64_t null_label, int64_t oov_label,
                               int64_t first_label, uint64_t num_buckets, void* labels_out_host, int out_dtype,
                               int n_threads) {
  NVTB_REQUIRE(v != nullptr && n >= 0, "NULL vocabulary or n < 0");
  NVTB_REQUIRE(key_dtype == NVTB_I32 || key_dtype == NVTB_I64, "key dtype must be int32 or int64");
  NVTB_REQUIRE(out_dtype == NVTB_I32 || out_dtype == NVTB_I64, "out dtype must be int32 or int64");
  if (n == 0) return NVTB_OK;
  NVTB_REQUIRE(keys_host != nullptr && labels_out_host != nullptr, "NULL keys / labels");
  auto body = [&](int64_t lo, int64_t hi) {
    if (key_dtype == NVTB_I32) {
      if (out_dtype == NVTB_I32) encode_range<int32_t, int32_t>(v, (const int32_t*)keys_host, validity_host, lo, hi, null_label, oov_label, first_label, num_buckets, (int32_t*)labels_out_host);
      else                       encode_range<int32_t, int64_t>(v, (const int32_t*)keys_host, validity_host, lo, hi, null_label, oov_label, first_label, num_buckets, (int64_t*)labels_out_host);
    } else {
      if (out_dtype == NVTB_I32) encode_range<int64_t, int32_t>(v, (const int64_t*)keys_host, validity_host, lo, hi, null_label, oov_label, first_label, num_buckets, (int32_t*)labels_out_host);
      else                       encode_range<int64_t, int64_t>(v, (const int64_t*)keys_host, validity_host, lo, hi, null_label, oov_label, first_label, num_buckets, (int64_t*)labels_out_host);
    }
  };
  run_threads(n, n_threads, body);
  return NVTB_OK;
}

// FillMissing on a host array, in place (fill.cc:32-106): NaN -> fill for float32 / float64;
// integer arrays carry no nulls in a dict-of-arrays request and are left alone
int nvtb_infer_fill_host(void* data_host, int dtype, int64_t n, double fill) {
  NVTB_REQUIRE(n >= 0 && (n == 0 || data_host != nullptr), "bad arguments");
  if (dtype == NVTB_F32) {
    float* p = (float*)data_host;
    const float f = (float)fill;
    for (int64_t i = 0; i < n; ++i) if (p[i] != p[i]) p[i] = f;
  } else if (dtype == NVTB_F64) {
    double* p = (double*)data_host;
    for (int64_t i = 0; i < n; ++i) if (p[i] != p[i]) p[i] = fill;
  } else {
    NVTB_REQUIRE(dtype == NVTB_I32 || dtype == NVTB_I64 || dtype == NVTB_U8, "unsupported dtype");
  }
  return NVTB_OK;
}

}  // extern "C"
