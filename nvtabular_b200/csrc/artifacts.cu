// artifacts.cu — the Categorify artefact files meta.<col>.parquet and unique.<col>.parquet
// (reference nvtabular/ops/categorify.py:731-822), written by library threads.  Host code only.
//
// A Criteo fit writes 26 meta files and about 20 small vocabulary files.  Their bytes are few
// (about 1e6 keys in all); through pandas / pyarrow each file costs a frame, a table, the
// pandas metadata and a writer set-up, all under the GIL, and that per-file work used to bound
// the step.  Here a submit only queues a job: a writer thread waits for that vocabulary's own
// build, copies its kept rows to the host and writes both files, while the Python thread goes
// on queueing device work.
//
// The writer emits the subset of Parquet that DataFrame.to_parquet(compression=None) output
// needs to read back identically: one row group, PLAIN-encoded, uncompressed v1 data pages of
// about 1 MiB per OPTIONAL column (definition levels: one RLE run of 1s per page; a page's sizes
// are int32), a Thrift-compact FileMetaData, and
// the `pandas` key-value metadata that carries the RangeIndex of the labels.  No dictionary
// pages, no statistics, no compression.
#include <algorithm>
#include <cerrno>
#include <chrono>
#include <condition_variable>
#include <cstdint>
#include <cstring>
#include <deque>
#include <memory>
#include <mutex>
#include <new>
#include <string>
#include <thread>
#include <vector>

#include "common.cuh"

namespace nvtb {
cudaEvent_t vocab_build_event(const nvtb_vocab_t* v);   // vocab.cu
}

namespace {

using nvtb::set_error;

// ------------------------------------------------------------------ Thrift compact protocol
// Only what the page headers and the footer use: i32 / i64 / binary fields, nested structs,
// lists of structs, i32 and binary.
class Compact {
 public:
  static constexpr int kI32 = 5, kI64 = 6, kBinary = 8, kList = 9, kStruct = 12;
  std::string out;

  void i32(int id, int32_t v) { field(id, kI32); varint(zigzag(v)); }
  void i64(int id, int64_t v) { field(id, kI64); varint(zigzag(v)); }
  void str(int id, const std::string& s) { field(id, kBinary); bytes(s); }
  void begin(int id) { field(id, kStruct); last_.push_back(0); }   // a struct-valued field
  void elem_begin() { last_.push_back(0); }                        // a struct element of a list
  void end() { out.push_back('\0'); last_.pop_back(); }            // stop byte of either
  void list(int id, int elem_type, size_t n) {
    field(id, kList);
    if (n < 15) {
      out.push_back((char)((n << 4) | elem_type));
    } else {
      out.push_back((char)(0xF0 | elem_type));
      varint(n);
    }
  }
  void elem_i32(int32_t v) { varint(zigzag(v)); }
  void elem_str(const std::string& s) { bytes(s); }
  void stop() { out.push_back('\0'); }                             // end of the message

 private:
  std::vector<int> last_{0};   // last field id per open struct

  static uint64_t zigzag(int64_t v) { return ((uint64_t)v << 1) ^ (uint64_t)(v >> 63); }
  void varint(uint64_t v) {
    while (v >= 0x80) {
      out.push_back((char)((v & 0x7F) | 0x80));
      v >>= 7;
    }
    out.push_back((char)v);
  }
  void bytes(const std::string& s) {
    varint(s.size());
    out += s;
  }
  void field(int id, int type) {
    const int d = id - last_.back();
    if (d > 0 && d <= 15) {
      out.push_back((char)((d << 4) | type));
    } else {
      out.push_back((char)type);
      varint(zigzag(id));
    }
    last_.back() = id;
  }
};

// ------------------------------------------------------------------ the Parquet subset
enum { kPqInt32 = 1, kPqInt64 = 2, kPqFloat = 4, kPqDouble = 5, kPqByteArray = 6 };
enum { kPlain = 0, kRle = 3 };

struct PqColumn {
  std::string name;
  int type;              // physical type
  bool utf8;             // BYTE_ARRAY annotated UTF8 / STRING
  const void* data;      // PLAIN-encoded values
  size_t bytes;
  size_t width;          // bytes per value; 0: variable (BYTE_ARRAY), written as one page
};

// A page's sizes are int32 in its header, so a column is cut into pages of about this many bytes
// (pyarrow's default page size).
constexpr int64_t kPageBytes = (int64_t)1 << 20;

// definition levels of n present values (max level 1): a 4-byte length, then one RLE run
static std::string all_defined(int64_t n) {
  std::string s(4, '\0');
  if (n > 0) {
    uint64_t h = (uint64_t)n << 1;   // run header: count << 1 | 0 (an RLE run)
    while (h >= 0x80) {
      s.push_back((char)((h & 0x7F) | 0x80));
      h >>= 7;
    }
    s.push_back((char)h);
    s.push_back('\1');               // the repeated level, in one byte (bit width 1)
  }
  const uint32_t len = (uint32_t)(s.size() - 4);
  memcpy(&s[0], &len, 4);
  return s;
}

class File {
 public:
  explicit File(const std::string& path) : path_(path), f_(fopen(path.c_str(), "wb")), errno_(f_ ? 0 : errno) {}
  ~File() {
    if (f_) fclose(f_);
  }
  void put(const void* p, size_t n) {
    if (f_ && n && fwrite(p, 1, n, f_) != n && !errno_) errno_ = errno ? errno : EIO;
    pos_ += (int64_t)n;
  }
  void put(const std::string& s) { put(s.data(), s.size()); }
  int64_t pos() const { return pos_; }
  int close() {
    if (f_ && fclose(f_) != 0 && !errno_) errno_ = errno ? errno : EIO;
    f_ = nullptr;
    if (errno_) {
      set_error("cannot write %s: %s", path_.c_str(), strerror(errno_));
      return NVTB_EIO;
    }
    return NVTB_OK;
  }

 private:
  std::string path_;
  FILE* f_;
  int errno_;
  int64_t pos_ = 0;
};

// page_rows: values per page of a fixed-width column (0: pages of about kPageBytes)
static int write_parquet(const std::string& path, const std::vector<PqColumn>& cols, int64_t n,
                         const std::string* pandas_meta, int64_t page_rows = 0) {
  const int64_t kMaxPageBytes = INT32_MAX - 64;      // room for the definition levels
  for (const PqColumn& col : cols) {
    if (col.width == 0 && (int64_t)col.bytes > kMaxPageBytes) {
      set_error("cannot write %s: column %s holds %zu bytes, more than one page can", path.c_str(),
                col.name.c_str(), col.bytes);
      return NVTB_EINVAL;
    }
  }
  File f(path);
  f.put("PAR1", 4);
  std::vector<int64_t> offset(cols.size()), total(cols.size());
  int64_t all_bytes = 0;
  for (size_t c = 0; c < cols.size(); ++c) {
    const PqColumn& col = cols[c];
    int64_t per_page = n;                              // a variable-width column: one page
    if (col.width > 0) {
      per_page = page_rows > 0 ? page_rows : kPageBytes / (int64_t)col.width;
      per_page = std::max<int64_t>(1, std::min<int64_t>(per_page, kMaxPageBytes / (int64_t)col.width));
    }
    offset[c] = f.pos();
    int64_t r = 0;
    do {                                               // an empty column still gets one page
      const int64_t m = std::min(per_page, n - r);
      const std::string defs = all_defined(m);
      const size_t vbytes = col.width > 0 ? (size_t)m * col.width : col.bytes;
      const int64_t page = (int64_t)(defs.size() + vbytes);
      Compact ph;                                     // PageHeader
      ph.i32(1, 0);                                   // type DATA_PAGE
      ph.i32(2, (int32_t)page);                       // uncompressed_page_size
      ph.i32(3, (int32_t)page);                       // compressed_page_size
      ph.begin(5);                                    // data_page_header
      ph.i32(1, (int32_t)m);                          //   num_values
      ph.i32(2, kPlain);                              //   encoding
      ph.i32(3, kRle);                                //   definition_level_encoding
      ph.i32(4, kRle);                                //   repetition_level_encoding
      ph.end();
      ph.stop();
      f.put(ph.out);
      f.put(defs);
      f.put((const char*)col.data + (size_t)r * col.width, vbytes);
      r += m;
    } while (r < n);
    total[c] = f.pos() - offset[c];
    all_bytes += total[c];
  }
  Compact m;                                          // FileMetaData
  m.i32(1, 1);                                        // version
  m.list(2, Compact::kStruct, cols.size() + 1);       // schema: root, then one leaf per column
  m.elem_begin();
  m.str(4, "schema");
  m.i32(5, (int32_t)cols.size());                     // num_children
  m.end();
  for (const PqColumn& col : cols) {
    m.elem_begin();
    m.i32(1, col.type);
    m.i32(3, 1);                                      // repetition_type OPTIONAL
    m.str(4, col.name);
    if (col.utf8) {
      m.i32(6, 0);                                    // converted_type UTF8
      m.begin(10);                                    // logicalType: STRING
      m.begin(1);
      m.end();
      m.end();
    }
    m.end();
  }
  m.i64(3, n);                                        // num_rows
  m.list(4, Compact::kStruct, 1);                     // row_groups
  m.elem_begin();
  m.list(1, Compact::kStruct, cols.size());           // columns
  for (size_t c = 0; c < cols.size(); ++c) {
    m.elem_begin();
    m.i64(2, offset[c]);                              // file_offset
    m.begin(3);                                       // meta_data
    m.i32(1, cols[c].type);
    m.list(2, Compact::kI32, 2);                      // encodings
    m.elem_i32(kPlain);
    m.elem_i32(kRle);
    m.list(3, Compact::kBinary, 1);                   // path_in_schema
    m.elem_str(cols[c].name);
    m.i32(4, 0);                                      // codec UNCOMPRESSED
    m.i64(5, n);                                      // num_values
    m.i64(6, total[c]);                               // total_uncompressed_size
    m.i64(7, total[c]);                               // total_compressed_size
    m.i64(9, offset[c]);                              // data_page_offset
    m.end();
    m.end();
  }
  m.i64(2, all_bytes);                                // total_byte_size
  m.i64(3, n);                                        // num_rows
  m.end();
  if (pandas_meta != nullptr) {
    m.list(5, Compact::kStruct, 1);                   // key_value_metadata
    m.elem_begin();
    m.str(1, "pandas");
    m.str(2, *pandas_meta);
    m.end();
  }
  m.str(6, "nvtabular_b200");                         // created_by
  m.stop();
  f.put(m.out);
  const uint32_t len = (uint32_t)m.out.size();
  f.put(&len, 4);
  f.put("PAR1", 4);
  return f.close();
}

static int pq_type(int dtype) {
  switch (dtype) {
    case NVTB_I32: return kPqInt32;
    case NVTB_I64: return kPqInt64;
    case NVTB_F32: return kPqFloat;
    case NVTB_F64: return kPqDouble;
    default: return -1;
  }
}

// ------------------------------------------------------------------ vocabulary jobs
struct Job {
  const nvtb_vocab_t* v;
  cudaEvent_t ev = nullptr;  // recorded at submit for a handle without a build event
  std::string meta_path, meta_pandas, unique_path, key_name, size_name, head, tail;
  bool has_unique, has_sizes;
  int64_t unique_max_rows, index_start, oov_count;
  int key_dtype;
  int rc = NVTB_OK;
  std::string err;

  ~Job() {
    if (ev) cudaEventDestroy(ev);
  }
  // the event after which the vocabulary's kept rows are final
  cudaEvent_t done() const { return ev ? ev : nvtb::vocab_build_event(v); }
  // true once that event has fired (or failed: the job then reports the error)
  bool ready() const {
    const cudaEvent_t e = done();
    return e == nullptr || cudaEventQuery(e) != cudaErrorNotReady;
  }
};

// Pinned staging buffer + copy stream of a writer thread.  Pooled for the life of the process:
// a fit runs one batch of jobs, and cudaMallocHost / cudaFreeHost each time would cost more
// than the copies.
struct Stage {
  void* pin;
  cudaStream_t st;
};
constexpr size_t kStageBytes = (size_t)4 << 20;
static std::mutex g_stage_mu;
static std::vector<Stage*> g_stage_free;

static int stage_acquire(Stage** out) {
  {
    std::lock_guard<std::mutex> lk(g_stage_mu);
    if (!g_stage_free.empty()) {
      *out = g_stage_free.back();
      g_stage_free.pop_back();
      return NVTB_OK;
    }
  }
  Stage* s = new (std::nothrow) Stage{nullptr, nullptr};
  NVTB_REQUIRE(s != nullptr, "host allocation failed");
  cudaError_t e = cudaMallocHost(&s->pin, kStageBytes);
  if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&s->st, cudaStreamNonBlocking);
  if (e != cudaSuccess) {
    if (s->pin) cudaFreeHost(s->pin);
    delete s;
    set_error("artefact writer staging: %s", cudaGetErrorString(e));
    return e == cudaErrorMemoryAllocation ? NVTB_ENOMEM : NVTB_ECUDA;
  }
  *out = s;
  return NVTB_OK;
}

static void stage_release(Stage* s) {
  if (s == nullptr) return;
  std::lock_guard<std::mutex> lk(g_stage_mu);
  g_stage_free.push_back(s);
}

// n int64 values from the device to the host, through the pinned stage
static int copy_to_host(Stage* s, const int64_t* src, int64_t n, int64_t* dst) {
  const int64_t per = (int64_t)(kStageBytes / sizeof(int64_t));
  for (int64_t off = 0; off < n; off += per) {
    const size_t bytes = sizeof(int64_t) * (size_t)std::min(per, n - off);
    NVTB_CUDA_OK(cudaMemcpyAsync(s->pin, src + off, bytes, cudaMemcpyDeviceToHost, s->st));
    NVTB_CUDA_OK(cudaStreamSynchronize(s->st));
    memcpy(dst + off, s->pin, bytes);
  }
  return NVTB_OK;
}

// the kept keys / sizes of a built vocabulary, in label order, on the host
static int kept_rows(const nvtb_vocab_t* v, int64_t n, bool with_sizes, Stage* s, std::vector<int64_t>* keys,
                     std::vector<int64_t>* sizes) {
  keys->resize((size_t)n);
  if (with_sizes) sizes->resize((size_t)n);
  if (n == 0) return NVTB_OK;
  int64_t* d = nullptr;
  NVTB_CUDA_OK(cudaMallocAsync(&d, sizeof(int64_t) * (size_t)n * (with_sizes ? 2 : 1), s->st));
  int rc = nvtb_vocab_export(v, d, with_sizes ? d + n : nullptr, s->st);
  if (rc == NVTB_OK) rc = copy_to_host(s, d, n, keys->data());
  if (rc == NVTB_OK && with_sizes) rc = copy_to_host(s, d + n, n, sizes->data());
  cudaFreeAsync(d, s->st);
  return rc;
}

static int write_meta(const std::string& path, int64_t oov_count, const nvtb_vocab_info_t& info, bool observed,
                      const std::string& pandas_meta) {
  static const char* kinds[4] = {"pad", "null", "oov", "unique"};
  std::string kind;
  for (const char* k : kinds) {
    const uint32_t len = (uint32_t)strlen(k);
    kind.append((const char*)&len, 4);
    kind.append(k, len);
  }
  const int64_t offset[4] = {0, 1, 2, 2 + oov_count};   // PAD_OFFSET, NULL_OFFSET, OOV_OFFSET, first label
  const int64_t num_indices[4] = {1, 1, oov_count, info.n_kept};
  const int64_t num_observed[4] = {0, info.null_size, info.oov_size, info.unique_size};
  std::vector<PqColumn> cols = {{"kind", kPqByteArray, true, kind.data(), kind.size(), 0},
                                {"offset", kPqInt64, false, offset, sizeof(offset), 8},
                                {"num_indices", kPqInt64, false, num_indices, sizeof(num_indices), 8}};
  if (observed) cols.push_back({"num_observed", kPqInt64, false, num_observed, sizeof(num_observed), 8});
  return write_parquet(path, cols, 4, &pandas_meta);
}

// int64 keys -> the written key values (KeySpace.decode: int keys are the values; float keys are
// the order-preserving image of a float64)
static void decode_keys(const std::vector<int64_t>& k, int dtype, std::vector<uint8_t>* out) {
  const size_t n = k.size();
  out->resize(n * nvtb::dtype_size(dtype));
  for (size_t i = 0; i < n; ++i) {
    if (dtype == NVTB_I32) {
      const int32_t x = (int32_t)k[i];
      memcpy(out->data() + 4 * i, &x, 4);
    } else {
      const int64_t b = k[i] >= 0 ? k[i] : (k[i] ^ INT64_MAX);
      double x;
      memcpy(&x, &b, 8);
      if (dtype == NVTB_F32) {
        const float y = (float)x;
        memcpy(out->data() + 4 * i, &y, 4);
      } else {
        memcpy(out->data() + 8 * i, &x, 8);
      }
    }
  }
}

static int run_job(Job& j, Stage** stage) {
  if (j.ev) NVTB_CUDA_OK(cudaEventSynchronize(j.ev));
  nvtb_vocab_info_t info;
  int rc = nvtb_vocab_info(j.v, &info);        // waits for the build's scalars
  if (rc) return rc;
  rc = write_meta(j.meta_path, j.oov_count, info, j.has_sizes, j.meta_pandas);
  if (rc) return rc;
  if (!j.has_unique || info.n_total == 0 || (j.unique_max_rows >= 0 && info.n_kept > j.unique_max_rows))
    return NVTB_OK;   // a lazily written vocabulary, or an empty input's null row (written by the caller)
  if (*stage == nullptr) {
    rc = stage_acquire(stage);
    if (rc) return rc;
  }
  std::vector<int64_t> keys, sizes;
  rc = kept_rows(j.v, info.n_kept, j.has_sizes, *stage, &keys, &sizes);
  if (rc) return rc;
  std::vector<uint8_t> decoded;
  const void* kdata = keys.data();
  if (j.key_dtype != NVTB_I64) {
    decode_keys(keys, j.key_dtype, &decoded);
    kdata = decoded.data();
  }
  const size_t kw = nvtb::dtype_size(j.key_dtype);
  std::vector<PqColumn> cols = {{j.key_name, pq_type(j.key_dtype), false, kdata, (size_t)info.n_kept * kw, kw}};
  if (j.has_sizes)
    cols.push_back({j.size_name, kPqInt64, false, sizes.data(), sizeof(int64_t) * (size_t)info.n_kept, 8});
  const std::string pandas = j.head + std::to_string(j.index_start + info.n_kept) + j.tail;
  return write_parquet(j.unique_path, cols, info.n_kept, &pandas);
}

}  // namespace

struct nvtb_artifacts {
  std::mutex mu;
  std::condition_variable cv;
  std::deque<Job*> queue;
  std::vector<std::unique_ptr<Job>> jobs;   // submission order
  bool closing = false;
  bool polling = false;                     // a thread is polling the build events
  int device = 0;
  std::vector<std::thread> threads;
};

// The next job to run: the first queued one whose vocabulary is built, so that a job waiting
// for a large build never holds a thread while small vocabularies are ready behind it.  Nothing
// signals the host when a build finishes, so while no queued job is ready ONE thread polls the
// events (every 500 us) and the others sleep until it hands over.
static Job* next_job(nvtb_artifacts* h) {
  std::unique_lock<std::mutex> lk(h->mu);
  bool poller = false;
  for (;;) {
    if (h->queue.empty()) {
      if (poller) h->polling = false;
      if (h->closing) {
        h->cv.notify_all();
        return nullptr;
      }
      h->cv.wait(lk);
      poller = false;
      continue;
    }
    for (auto it = h->queue.begin(); it != h->queue.end(); ++it) {
      if ((*it)->ready()) {
        Job* j = *it;
        h->queue.erase(it);
        if (poller) h->polling = false;
        h->cv.notify_all();      // another thread takes over the polling, or the next ready job
        return j;
      }
    }
    if (h->polling && !poller) {
      h->cv.wait(lk);
      continue;
    }
    h->polling = poller = true;
    h->cv.wait_for(lk, std::chrono::microseconds(500));
  }
}

static void writer_thread(nvtb_artifacts* h) {
  cudaSetDevice(h->device);
  Stage* stage = nullptr;
  for (;;) {
    Job* j = next_job(h);
    if (j == nullptr) break;
    try {
      j->rc = run_job(*j, &stage);
    } catch (const std::bad_alloc&) {
      set_error("host allocation failed");
      j->rc = NVTB_ENOMEM;
    }
    if (j->rc) {
      const std::string msg = nvtb_last_error();
      // a file error names its path already; anything else is told with the job's files
      j->err = msg.find(j->meta_path) != std::string::npos || (j->has_unique && msg.find(j->unique_path) != std::string::npos)
                   ? msg
                   : "writing " + j->meta_path + (j->has_unique ? " / " + j->unique_path : "") + ": " + msg;
    }
  }
  stage_release(stage);
}

extern "C" {

int nvtb_parquet_write(const char* path, const nvtb_pq_col_t* cols_host, int ncols, int64_t n,
                       const char* pandas_meta, int64_t page_rows) {
  NVTB_REQUIRE(path != nullptr && ncols >= 0 && n >= 0 && page_rows >= 0 && (ncols == 0 || cols_host != nullptr),
               "nvtb_parquet_write: bad arguments");
  try {
    std::vector<PqColumn> cols;
    for (int c = 0; c < ncols; ++c) {
      const int t = pq_type(cols_host[c].dtype);
      NVTB_REQUIRE(t >= 0, "nvtb_parquet_write: dtype must be I32, I64, F32 or F64");
      NVTB_REQUIRE(cols_host[c].name != nullptr && (n == 0 || cols_host[c].data != nullptr),
                   "nvtb_parquet_write: NULL column name or data");
      const size_t w = nvtb::dtype_size(cols_host[c].dtype);
      cols.push_back({cols_host[c].name, t, false, cols_host[c].data, (size_t)n * w, w});
    }
    const std::string meta = pandas_meta ? pandas_meta : "";
    return write_parquet(path, cols, n, pandas_meta ? &meta : nullptr, page_rows);
  } catch (const std::bad_alloc&) {
    set_error("nvtb_parquet_write %s: host allocation failed", path);
    return NVTB_ENOMEM;
  }
}

int nvtb_parquet_write_meta(const char* path, int64_t oov_count, const nvtb_vocab_info_t* info_host,
                            int with_observed, const char* pandas_meta) {
  NVTB_REQUIRE(path != nullptr && info_host != nullptr && pandas_meta != nullptr && oov_count >= 1,
               "nvtb_parquet_write_meta: bad arguments");
  try {
    return write_meta(path, oov_count, *info_host, with_observed != 0, pandas_meta);
  } catch (const std::bad_alloc&) {
    set_error("nvtb_parquet_write_meta %s: host allocation failed", path);
    return NVTB_ENOMEM;
  }
}

int nvtb_artifacts_begin(nvtb_artifacts_t** out, int threads) {
  NVTB_REQUIRE(out != nullptr && threads >= 1 && threads <= 64, "nvtb_artifacts_begin: threads must be in [1, 64]");
  nvtb_artifacts* h = new (std::nothrow) nvtb_artifacts();
  NVTB_REQUIRE(h != nullptr, "host allocation failed");
  cudaError_t e = cudaGetDevice(&h->device);
  if (e != cudaSuccess) {
    delete h;
    set_error("nvtb_artifacts_begin: %s", cudaGetErrorString(e));
    return NVTB_ECUDA;
  }
  try {
    for (int t = 0; t < threads; ++t) h->threads.emplace_back(writer_thread, h);
  } catch (...) {
    nvtb_artifacts_join(h);
    set_error("nvtb_artifacts_begin: cannot start writer threads");
    return NVTB_ENOMEM;
  }
  *out = h;
  return NVTB_OK;
}

int nvtb_artifacts_submit_vocab(nvtb_artifacts_t* h, const nvtb_vocab_t* v, const char* meta_path,
                                const char* meta_pandas, const char* unique_path, int64_t unique_max_rows,
                                const char* key_name, int key_dtype, const char* size_name, int64_t index_start,
                                int64_t oov_count, const char* unique_pandas_head, const char* unique_pandas_tail,
                                void* stream) {
  NVTB_REQUIRE(h != nullptr && v != nullptr && meta_path != nullptr && meta_pandas != nullptr && key_name != nullptr,
               "nvtb_artifacts_submit_vocab: NULL argument");
  NVTB_REQUIRE(pq_type(key_dtype) >= 0, "nvtb_artifacts_submit_vocab: key_dtype must be I32, I64, F32 or F64");
  NVTB_REQUIRE(unique_path == nullptr || (unique_pandas_head != nullptr && unique_pandas_tail != nullptr),
               "nvtb_artifacts_submit_vocab: a unique file needs its pandas metadata");
  NVTB_REQUIRE(oov_count >= 1, "nvtb_artifacts_submit_vocab: oov_count < 1");
  std::unique_ptr<Job> j;
  try {
    j.reset(new Job());
    j->v = v;
    j->meta_path = meta_path;
    j->meta_pandas = meta_pandas;
    j->has_unique = unique_path != nullptr;
    j->unique_path = unique_path ? unique_path : "";
    j->head = unique_pandas_head ? unique_pandas_head : "";
    j->tail = unique_pandas_tail ? unique_pandas_tail : "";
    j->key_name = key_name;
    j->has_sizes = size_name != nullptr;
    j->size_name = size_name ? size_name : "";
    j->unique_max_rows = unique_max_rows;
    j->index_start = index_start;
    j->oov_count = oov_count;
    j->key_dtype = key_dtype;
  } catch (const std::bad_alloc&) {
    set_error("host allocation failed");
    return NVTB_ENOMEM;
  }
  if (nvtb::vocab_build_event(v) == nullptr) {
    // no enqueued build to wait for (from_arrays): order the copy after what `stream` holds now.
    // On an early return the Job, and with it the event, is destroyed.
    NVTB_CUDA_OK(cudaEventCreateWithFlags(&j->ev, cudaEventDisableTiming));
    NVTB_CUDA_OK(cudaEventRecord(j->ev, (cudaStream_t)stream));
  }
  {
    std::lock_guard<std::mutex> lk(h->mu);
    NVTB_REQUIRE(!h->closing, "nvtb_artifacts_submit_vocab: the batch is joined");
    h->queue.push_back(j.get());
    h->jobs.push_back(std::move(j));
  }
  h->cv.notify_one();
  return NVTB_OK;
}

int nvtb_artifacts_join(nvtb_artifacts_t* h) {
  if (h == nullptr) return NVTB_OK;
  {
    std::lock_guard<std::mutex> lk(h->mu);
    h->closing = true;
  }
  h->cv.notify_all();
  for (std::thread& t : h->threads) t.join();
  int rc = NVTB_OK;
  std::string err;
  for (const std::unique_ptr<Job>& j : h->jobs) {
    if (rc == NVTB_OK && j->rc != NVTB_OK) {
      rc = j->rc;
      err = j->err;
    }
  }
  delete h;
  if (rc) set_error("%s", err.c_str());
  return rc;
}

}  // extern "C"
