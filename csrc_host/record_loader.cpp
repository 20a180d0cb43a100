// Native host runtime: record-database reader + multi-threaded batch assembler.
//
// The reference's data path is C++ end to end: a LevelDB/LMDB cursor, Datum::ParseFromString and the
// DataTransformer run on one prefetch thread per data layer (src/caffe/layers/data_layer.cpp:143-259,
// src/caffe/layers/base_data_layer.cpp:57-104).  One H100 trains AlexNet at ~47 k ImageNet-sized records per second, i.e.
// ~7 GB/s of record payload, which a single thread (let alone Python) cannot decode, so this module
//   * memory-maps the PDB record file (b"PDB1" | u64 n | n x (u32 klen, u32 vlen, key, value)) and indexes it once,
//   * parses the Datum wire format in place (no protobuf library, no copies other than the payload memcpy),
//   * fills caller-owned batch buffers (page-locked memory handed in from PyTorch) with a pool of worker threads, and
//   * runs a producer thread that keeps a ring of such batches filled ahead of the consumer.
// The GPU-side transform (crop / mirror / mean / scale / layout) is a CUDA kernel, so the host only ever moves raw
// uint8 pixels; float_data records are supported as fp32.
//
// Pure C++17 + pybind11 (no CUDA, no torch headers): builds and is unit-tested on a CPU-only box.
#include <pybind11/pybind11.h>
#include <pybind11/stl.h>

#include "leveldb_reader.h"

#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

#include <atomic>
#include <condition_variable>
#include <cstdint>
#include <cstring>
#include <deque>
#include <algorithm>
#include <functional>
#include <memory>
#include <mutex>
#include <stdexcept>
#include <string>
#include <thread>
#include <vector>

namespace py = pybind11;

namespace psd_host {

// ----------------------------------------------------------------------------- record file
struct Record {
  const uint8_t* key;
  uint32_t klen;
  const uint8_t* val;
  uint32_t vlen;
};

class RecordFile {
 public:
  explicit RecordFile(const std::string& path_in) {
    // a directory is a LevelDB (CURRENT + MANIFEST), an LMDB environment (data.mdb) or a PDB store (data.pdb)
    std::string path = path_in;
    struct stat dst;
    if (::stat(path.c_str(), &dst) == 0 && S_ISDIR(dst.st_mode)) {
      auto exists = [](const std::string& p) { struct stat s; return ::stat(p.c_str(), &s) == 0; };
      if (exists(path + "/data.pdb")) path += "/data.pdb";
      else if (exists(path + "/data.mdb")) path += "/data.mdb";
      else if (exists(path + "/CURRENT")) {
        ldb_.reset(new LevelDBIndex(path));
        for (const LdbRecord& r : ldb_->records()) recs_.push_back(Record{r.key, r.klen, r.val, r.vlen});
        return;
      } else {
        throw std::runtime_error(path + ": no data.pdb, data.mdb or LevelDB CURRENT file in this directory");
      }
    }
    fd_ = ::open(path.c_str(), O_RDONLY);
    if (fd_ < 0) throw std::runtime_error("cannot open " + path);
    struct stat st;
    if (fstat(fd_, &st) != 0 || st.st_size < 12) { ::close(fd_); throw std::runtime_error(path + ": not a record database"); }
    size_ = static_cast<size_t>(st.st_size);
    base_ = static_cast<const uint8_t*>(mmap(nullptr, size_, PROT_READ, MAP_SHARED, fd_, 0));
    if (base_ == MAP_FAILED) { ::close(fd_); throw std::runtime_error("mmap failed for " + path); }
    if (std::memcmp(base_, "PDB1", 4) == 0) {
      uint64_t n;
      std::memcpy(&n, base_ + 4, 8);
      size_t off = 12;
      recs_.reserve(n);
      while (off + 8 <= size_ && recs_.size() < n) {
        uint32_t kl, vl;
        std::memcpy(&kl, base_ + off, 4);
        std::memcpy(&vl, base_ + off + 4, 4);
        if (off + 8 + kl + static_cast<size_t>(vl) > size_) break;       // truncated tail: ignore
        recs_.push_back(Record{base_ + off + 8, kl, base_ + off + 8 + kl, vl});
        off += 8 + kl + static_cast<size_t>(vl);
      }
    } else if (is_lmdb()) {
      try {
        index_lmdb(path);
      } catch (...) {
        close();
        throw;
      }
    } else {
      close();
      throw std::runtime_error(path + ": neither a PDB record file nor an LMDB data.mdb");
    }
    madvise(const_cast<uint8_t*>(base_), size_, MADV_SEQUENTIAL);
  }
  ~RecordFile() { close(); }
  RecordFile(const RecordFile&) = delete;
  RecordFile& operator=(const RecordFile&) = delete;

  size_t size() const { return recs_.size(); }
  const Record& at(size_t i) const { return recs_[i]; }

 private:
  // ---- LMDB 0.9 data.mdb (read-only; same definition as poseidon_b200/data/lmdb_reader.py) ---------------------------
  //   page header 16 B: pgno u64 | pad u16 | flags u16 | lower u16 upper u16 ; node: lo u16 hi u16 flags u16 ksize u16 key data
  template <class T>
  T rd(size_t off) const {
    if (off + sizeof(T) > size_) throw std::runtime_error("LMDB: read past end of file");
    T v;
    std::memcpy(&v, base_ + off, sizeof(T));
    return v;
  }
  bool is_lmdb() const {
    return size_ >= 1024 && (rd<uint16_t>(10) & 0x08) && rd<uint32_t>(16) == 0xBEEFC0DEu;
  }
  struct LmdbMeta { uint32_t psize; uint16_t flags; uint64_t entries, root, txnid; };
  LmdbMeta lmdb_meta(size_t off) const {
    if (!(rd<uint16_t>(off + 10) & 0x08) || rd<uint32_t>(off + 16) != 0xBEEFC0DEu) throw std::runtime_error("LMDB: bad meta page");
    if (rd<uint32_t>(off + 20) != 1) throw std::runtime_error("LMDB: unsupported data version");
    const size_t dbs = off + 16 + 24;
    LmdbMeta m;
    m.psize = rd<uint32_t>(dbs);
    m.flags = rd<uint16_t>(dbs + 48 + 4);
    m.entries = rd<uint64_t>(dbs + 48 + 32);
    m.root = rd<uint64_t>(dbs + 48 + 40);
    m.txnid = rd<uint64_t>(dbs + 96 + 8);
    return m;
  }
  void lmdb_walk(uint64_t pgno, uint32_t psize, int depth) {
    if (depth > 64) throw std::runtime_error("LMDB: tree too deep");
    const size_t off = static_cast<size_t>(pgno) * psize;
    const uint16_t flags = rd<uint16_t>(off + 10), lower = rd<uint16_t>(off + 12);
    const int n = (lower - 16) >> 1;
    for (int i = 0; i < n; ++i) {
      const size_t node = off + rd<uint16_t>(off + 16 + 2 * static_cast<size_t>(i));
      const uint32_t lo = rd<uint16_t>(node), hi = rd<uint16_t>(node + 2);
      const uint16_t nflags = rd<uint16_t>(node + 4), ksize = rd<uint16_t>(node + 6);
      if (flags & 0x01) {                                                     // branch
        lmdb_walk(lo | (static_cast<uint64_t>(hi) << 16) | (static_cast<uint64_t>(nflags) << 32), psize, depth + 1);
      } else if (flags & 0x02) {                                              // leaf
        if ((flags & 0x20) || (nflags & 0x06)) throw std::runtime_error("LMDB: DUPSORT / sub-databases are not supported");
        const uint32_t dsize = lo | (hi << 16);
        const uint8_t* key = base_ + node + 8;
        const uint8_t* val = key + ksize;
        if (nflags & 0x01) {                                                  // F_BIGDATA: overflow run
          const uint64_t opg = rd<uint64_t>(node + 8 + ksize);
          const size_t ooff = static_cast<size_t>(opg) * psize;
          if (!(rd<uint16_t>(ooff + 10) & 0x04)) throw std::runtime_error("LMDB: expected an overflow page");
          val = base_ + ooff + 16;
        }
        if (static_cast<size_t>(val - base_) + dsize > size_) throw std::runtime_error("LMDB: value past end of file");
        recs_.push_back(Record{key, ksize, val, dsize});
      } else {
        throw std::runtime_error("LMDB: unexpected page type");
      }
    }
  }
  void index_lmdb(const std::string& path) {
    const LmdbMeta m0 = lmdb_meta(0);
    if (m0.psize < 512 || m0.psize > 65536 || (m0.psize & (m0.psize - 1))) throw std::runtime_error(path + ": implausible LMDB page size");
    const LmdbMeta m1 = lmdb_meta(m0.psize);
    const LmdbMeta& m = m1.txnid > m0.txnid ? m1 : m0;
    if (m.flags & 0x04) throw std::runtime_error(path + ": DUPSORT LMDB databases are not supported");
    recs_.reserve(m.entries);
    if (m.root != ~0ull) lmdb_walk(m.root, m0.psize, 0);
    if (m.entries && recs_.size() != m.entries) throw std::runtime_error(path + ": LMDB record count does not match its meta page");
  }

  void close() {
    if (base_ != nullptr && base_ != MAP_FAILED) munmap(const_cast<uint8_t*>(base_), size_);
    base_ = nullptr;
    if (fd_ >= 0) ::close(fd_);
    fd_ = -1;
  }
  int fd_ = -1;
  size_t size_ = 0;
  const uint8_t* base_ = nullptr;
  std::vector<Record> recs_;
  std::unique_ptr<LevelDBIndex> ldb_;      // LevelDB directories: owns the table mappings the records point into
};

// ----------------------------------------------------------------------------- Datum wire format
// message Datum { int32 channels=1; int32 height=2; int32 width=3; bytes data=4; int32 label=5;
//                 repeated float float_data=6; }   (reference: src/caffe/proto/caffe.proto, message Datum)
struct DatumView {
  int channels = 0, height = 0, width = 0, label = 0;
  const uint8_t* data = nullptr;
  size_t data_len = 0;
  // float_data: either one packed run or many 5-byte unpacked entries; collected lazily by copy_floats
  const uint8_t* buf = nullptr;
  size_t len = 0;
  size_t n_float = 0;
};

static inline bool read_varint(const uint8_t*& p, const uint8_t* end, uint64_t& v) {
  v = 0;
  for (int shift = 0; shift < 64 && p < end; shift += 7) {
    const uint8_t b = *p++;
    v |= static_cast<uint64_t>(b & 0x7f) << shift;
    if (!(b & 0x80)) return true;
  }
  return false;
}

static bool parse_datum(const uint8_t* buf, size_t len, DatumView& d) {
  const uint8_t* p = buf;
  const uint8_t* end = buf + len;
  d.buf = buf;
  d.len = len;
  while (p < end) {
    uint64_t tag;
    if (!read_varint(p, end, tag)) return false;
    const uint32_t field = static_cast<uint32_t>(tag >> 3), wt = static_cast<uint32_t>(tag & 7);
    if (wt == 0) {
      uint64_t v;
      if (!read_varint(p, end, v)) return false;
      if (field == 1) d.channels = static_cast<int>(v);
      else if (field == 2) d.height = static_cast<int>(v);
      else if (field == 3) d.width = static_cast<int>(v);
      else if (field == 5) d.label = static_cast<int>(static_cast<int64_t>(v));
    } else if (wt == 2) {
      uint64_t l;
      if (!read_varint(p, end, l) || l > static_cast<uint64_t>(end - p)) return false;
      if (field == 4) { d.data = p; d.data_len = static_cast<size_t>(l); }
      else if (field == 6) d.n_float += static_cast<size_t>(l) / 4;
      p += l;
    } else if (wt == 5) {
      if (end - p < 4) return false;
      if (field == 6) d.n_float += 1;
      p += 4;
    } else if (wt == 1) {
      if (end - p < 8) return false;
      p += 8;
    } else {
      return false;
    }
  }
  return true;
}

// second pass over the message copying float_data (packed or not) in order
static void copy_floats(const DatumView& d, float* dst, size_t max_n) {
  const uint8_t* p = d.buf;
  const uint8_t* end = d.buf + d.len;
  size_t n = 0;
  while (p < end && n < max_n) {
    uint64_t tag;
    if (!read_varint(p, end, tag)) return;
    const uint32_t field = static_cast<uint32_t>(tag >> 3), wt = static_cast<uint32_t>(tag & 7);
    if (wt == 0) { uint64_t v; if (!read_varint(p, end, v)) return; }
    else if (wt == 2) {
      uint64_t l;
      if (!read_varint(p, end, l)) return;
      if (field == 6) {
        const size_t k = std::min(static_cast<size_t>(l) / 4, max_n - n);
        std::memcpy(dst + n, p, k * 4);
        n += k;
      }
      p += l;
    } else if (wt == 5) {
      if (field == 6) { std::memcpy(dst + n, p, 4); ++n; }
      p += 4;
    } else if (wt == 1) p += 8;
    else return;
  }
}

// ----------------------------------------------------------------------------- worker pool
class Pool {
 public:
  explicit Pool(int n) {
    for (int i = 0; i < std::max(1, n); ++i) threads_.emplace_back([this] { run(); });
  }
  ~Pool() {
    { std::lock_guard<std::mutex> l(m_); stop_ = true; }
    cv_.notify_all();
    for (auto& t : threads_) t.join();
  }
  // runs fn(i) for i in [0, n) on the pool and the calling thread; returns when all are done
  void parallel_for(size_t n, const std::function<void(size_t)>& fn) {
    if (n == 0) return;
    auto job = std::make_shared<Job>();
    job->n = n;
    job->fn = &fn;
    { std::lock_guard<std::mutex> l(m_); jobs_.push_back(job); }
    cv_.notify_all();
    work(*job);
    std::unique_lock<std::mutex> l(job->m);
    job->cv.wait(l, [&] { return job->done.load() == n; });
    { std::lock_guard<std::mutex> g(m_);
      for (auto it = jobs_.begin(); it != jobs_.end(); ++it) if (it->get() == job.get()) { jobs_.erase(it); break; } }
  }
  int size() const { return static_cast<int>(threads_.size()); }

 private:
  struct Job {
    size_t n = 0;
    const std::function<void(size_t)>* fn = nullptr;
    std::atomic<size_t> next{0}, done{0};
    std::mutex m;
    std::condition_variable cv;
  };
  static void work(Job& j) {
    for (;;) {
      const size_t i = j.next.fetch_add(1);
      if (i >= j.n) return;
      (*j.fn)(i);
      if (j.done.fetch_add(1) + 1 == j.n) { std::lock_guard<std::mutex> l(j.m); j.cv.notify_all(); }
    }
  }
  void run() {
    for (;;) {
      std::shared_ptr<Job> job;
      {
        std::unique_lock<std::mutex> l(m_);
        cv_.wait(l, [&] {
          if (stop_) return true;
          for (auto& j : jobs_) if (j->next.load() < j->n) return true;
          return false;
        });
        if (stop_) return;
        for (auto& j : jobs_) if (j->next.load() < j->n) { job = j; break; }
      }
      if (job) work(*job);
    }
  }
  std::vector<std::thread> threads_;
  std::deque<std::shared_ptr<Job>> jobs_;
  std::mutex m_;
  std::condition_variable cv_;
  bool stop_ = false;
};

// ----------------------------------------------------------------------------- batch loader
struct Slot {
  uint8_t* data;     // [batch, C, H, W] uint8 or float32
  float* label;      // [batch]
};

class BatchLoader {
 public:
  // cursor semantics of the reference data layer: start at `offset`, advance `stride` records per item, wrap.
  BatchLoader(const std::string& path, int batch, long offset, long stride, int threads)
      : file_(path), batch_(batch), stride_(std::max<long>(1, stride)), pool_(threads) {
    if (file_.size() == 0) throw std::runtime_error(path + ": empty database");
    pos_ = static_cast<size_t>(offset) % file_.size();
    DatumView d;
    const Record& r = file_.at(pos_);
    if (!parse_datum(r.val, r.vlen, d)) throw std::runtime_error("malformed Datum in " + path);
    c_ = d.channels; h_ = d.height; w_ = d.width;
    is_bytes_ = d.data_len > 0;
    item_ = static_cast<size_t>(c_) * h_ * w_;
    if (item_ == 0) throw std::runtime_error("Datum without shape in " + path);
  }
  ~BatchLoader() { stop(); }

  py::tuple shape() const { return py::make_tuple(c_, h_, w_); }
  bool is_bytes() const { return is_bytes_; }
  size_t num_records() const { return file_.size(); }
  size_t position() const { return pos_; }
  void seek(size_t pos) { pos_ = pos % file_.size(); }
  size_t bytes_per_batch() const { return static_cast<size_t>(batch_) * item_ * (is_bytes_ ? 1 : 4); }

  // synchronous: fill one caller-owned batch (pointers as integers; the buffers must outlive the call)
  void fill(uintptr_t data_ptr, uintptr_t label_ptr) {
    py::gil_scoped_release nogil;
    fill_impl(reinterpret_cast<uint8_t*>(data_ptr), reinterpret_cast<float*>(label_ptr));
  }

  // asynchronous ring: the producer thread keeps `slots` filled ahead; acquire() blocks for the next ready slot
  // (returned in submission order), release(i) hands it back to the producer.
  void start(const std::vector<std::pair<uintptr_t, uintptr_t>>& slots) {
    stop();
    slots_.clear();
    for (auto& s : slots) slots_.push_back(Slot{reinterpret_cast<uint8_t*>(s.first), reinterpret_cast<float*>(s.second)});
    free_.clear();
    ready_.clear();
    for (size_t i = 0; i < slots_.size(); ++i) free_.push_back(static_cast<int>(i));
    stopping_ = false;
    producer_ = std::thread([this] { produce(); });
  }
  int acquire() {
    py::gil_scoped_release nogil;
    std::unique_lock<std::mutex> l(m_);
    cv_.wait(l, [&] { return !ready_.empty() || !error_.empty() || stopping_; });
    if (!error_.empty()) throw std::runtime_error(error_);
    if (ready_.empty()) throw std::runtime_error("loader stopped");
    const int s = ready_.front();
    ready_.pop_front();
    return s;
  }
  void release(int slot) {
    { std::lock_guard<std::mutex> l(m_); free_.push_back(slot); }
    cv_.notify_all();
  }
  void stop() {
    { std::lock_guard<std::mutex> l(m_); stopping_ = true; }
    cv_.notify_all();
    if (producer_.joinable()) {
      py::gil_scoped_release nogil;
      producer_.join();
    }
  }
  uint64_t batches_produced() const { return produced_.load(); }

 private:
  void fill_impl(uint8_t* data, float* label) {
    const size_t n = file_.size();
    const size_t start = pos_;
    const size_t esz = is_bytes_ ? 1 : 4;
    std::atomic<int> bad{0};
    const std::function<void(size_t)> fn = [&](size_t i) {
      const Record& r = file_.at((start + i * static_cast<size_t>(stride_)) % n);
      DatumView d;
      uint8_t* dst = data + i * item_ * esz;
      if (!parse_datum(r.val, r.vlen, d) || static_cast<size_t>(d.channels) * d.height * d.width != item_) {
        bad.fetch_add(1);
        std::memset(dst, 0, item_ * esz);
        label[i] = 0.f;
        return;
      }
      if (is_bytes_) {
        const size_t k = std::min(d.data_len, item_);
        std::memcpy(dst, d.data, k);
        if (k < item_) std::memset(dst + k, 0, item_ - k);
      } else {
        if (d.n_float < item_) std::memset(dst, 0, item_ * 4);
        copy_floats(d, reinterpret_cast<float*>(dst), item_);
      }
      label[i] = static_cast<float>(d.label);
    };
    pool_.parallel_for(static_cast<size_t>(batch_), fn);
    pos_ = (start + static_cast<size_t>(batch_) * static_cast<size_t>(stride_)) % n;
    if (bad.load() > 0) throw std::runtime_error("malformed or mis-shaped Datum records in batch");
  }
  void produce() {
    for (;;) {
      int s;
      {
        std::unique_lock<std::mutex> l(m_);
        cv_.wait(l, [&] { return stopping_ || !free_.empty(); });
        if (stopping_) return;
        s = free_.front();
        free_.pop_front();
      }
      try {
        fill_impl(slots_[s].data, slots_[s].label);
      } catch (const std::exception& e) {
        std::lock_guard<std::mutex> l(m_);
        error_ = e.what();
        cv_.notify_all();
        return;
      }
      produced_.fetch_add(1);
      { std::lock_guard<std::mutex> l(m_); ready_.push_back(s); }
      cv_.notify_all();
    }
  }

  RecordFile file_;
  int batch_;
  long stride_;
  Pool pool_;
  size_t pos_ = 0;
  int c_ = 0, h_ = 0, w_ = 0;
  bool is_bytes_ = true;
  size_t item_ = 0;
  std::vector<Slot> slots_;
  std::deque<int> free_, ready_;
  std::mutex m_;
  std::condition_variable cv_;
  std::thread producer_;
  bool stopping_ = true;
  std::string error_;
  std::atomic<uint64_t> produced_{0};
};

// ----------------------------------------------------------------------------- bf16 wire compression
// The reference can ship parameter updates as fp16 on the wire (dense-float16 row oplog,
// ps/src/petuum_ps_common/util/float16_compressor.hpp).  The CPU/gloo SSP backend uses these for the same purpose with
// bf16 (round-to-nearest-even), which keeps fp32's exponent range for gradient sums.
static void f32_to_bf16(uintptr_t src, uintptr_t dst, size_t n) {
  const uint32_t* s = reinterpret_cast<const uint32_t*>(src);
  uint16_t* d = reinterpret_cast<uint16_t*>(dst);
  for (size_t i = 0; i < n; ++i) {
    const uint32_t x = s[i];
    if ((x & 0x7fffffffu) > 0x7f800000u) { d[i] = static_cast<uint16_t>((x >> 16) | 0x40); continue; }   // NaN
    d[i] = static_cast<uint16_t>((x + 0x7fffu + ((x >> 16) & 1u)) >> 16);
  }
}
static void bf16_to_f32(uintptr_t src, uintptr_t dst, size_t n) {
  const uint16_t* s = reinterpret_cast<const uint16_t*>(src);
  uint32_t* d = reinterpret_cast<uint32_t*>(dst);
  for (size_t i = 0; i < n; ++i) d[i] = static_cast<uint32_t>(s[i]) << 16;
}

}  // namespace psd_host

namespace psd_host {
void bind_ml(py::module_& m);      // libsvm_parser.cpp
}

PYBIND11_MODULE(poseidon_b200_host, m) {
  using namespace psd_host;
  m.doc() = "poseidon-b200 native host runtime (record reader, batch loader, wire compression)";
  py::class_<BatchLoader>(m, "BatchLoader")
      .def(py::init<const std::string&, int, long, long, int>(), py::arg("path"), py::arg("batch"), py::arg("offset") = 0,
           py::arg("stride") = 1, py::arg("threads") = 4)
      .def("shape", &BatchLoader::shape)
      .def("is_bytes", &BatchLoader::is_bytes)
      .def("num_records", &BatchLoader::num_records)
      .def("position", &BatchLoader::position)
      .def("seek", &BatchLoader::seek)
      .def("bytes_per_batch", &BatchLoader::bytes_per_batch)
      .def("fill", &BatchLoader::fill)
      .def("start", &BatchLoader::start)
      .def("acquire", &BatchLoader::acquire)
      .def("release", &BatchLoader::release)
      .def("stop", &BatchLoader::stop)
      .def("batches_produced", &BatchLoader::batches_produced);
  // random access to the records of any supported database (PDB / LMDB / LevelDB), e.g. for the Python DBSource
  py::class_<RecordFile>(m, "RecordDB")
      .def(py::init<const std::string&>())
      .def("size", &RecordFile::size)
      .def("key", [](const RecordFile& f, size_t i) {
        if (i >= f.size()) throw py::index_error();
        const Record& r = f.at(i);
        return py::bytes(reinterpret_cast<const char*>(r.key), r.klen);
      })
      .def("value", [](const RecordFile& f, size_t i) {
        if (i >= f.size()) throw py::index_error();
        const Record& r = f.at(i);
        return py::bytes(reinterpret_cast<const char*>(r.val), r.vlen);
      });
  m.def("snappy_uncompress", [](py::bytes b) {
    const std::string s = b;
    const std::vector<uint8_t> out = snappy_uncompress(reinterpret_cast<const uint8_t*>(s.data()), s.size());
    return py::bytes(reinterpret_cast<const char*>(out.data()), out.size());
  });
  m.def("f32_to_bf16", &f32_to_bf16);
  m.def("bf16_to_f32", &bf16_to_f32);
  bind_ml(m);
}
