// nvb_map_io.cu -- map files and voxel-layer point export.
//
// A map file is the reference's .nvblx layer cake: an SQLite database with a metadata table and a data table per layer
// (map_saving/serializer.cpp, map_saving/internal/impl/block_serialization_impl.h). SQLite is opened at run time from
// libsqlite3.so.0, so building the library needs no SQLite headers; the handful of entry points used here are SQLite's
// stable C ABI. Without the library, saving and loading fail with NVB_ERR_IO.
//
// The kernels: the ESDF clear pass's parent boxes of loaded blocks, and the per-layer point export
// (io/pointcloud_io.cpp:23-73), counted per block, scanned and written in canonical order.
#include <dlfcn.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <string>

#include "nvb_esdf_block.cuh"

namespace nvb {

namespace {

// ---- SQLite, resolved with dlopen
struct sqlite3;
struct sqlite3_stmt;
constexpr int kSqliteOk = 0, kSqliteRow = 100, kSqliteDone = 101, kSqliteNull = 5;
constexpr int kOpenReadOnly = 0x1, kOpenReadWrite = 0x2, kOpenCreate = 0x4;

struct SqliteApi {
  int (*open_v2)(const char*, sqlite3**, int, const char*);
  int (*close_v2)(sqlite3*);
  const char* (*errmsg)(sqlite3*);
  int (*exec)(sqlite3*, const char*, int (*)(void*, int, char**, char**), void*, char**);
  int (*prepare_v2)(sqlite3*, const char*, int, sqlite3_stmt**, const char**);
  int (*step)(sqlite3_stmt*);
  int (*reset)(sqlite3_stmt*);
  int (*finalize)(sqlite3_stmt*);
  int (*bind_int)(sqlite3_stmt*, int, int);
  int (*bind_text)(sqlite3_stmt*, int, const char*, int, void (*)(void*));
  int (*bind_null)(sqlite3_stmt*, int);
  int (*bind_blob)(sqlite3_stmt*, int, const void*, int, void (*)(void*));
  long long (*column_int64)(sqlite3_stmt*, int);
  double (*column_double)(sqlite3_stmt*, int);
  int (*column_type)(sqlite3_stmt*, int);
  const void* (*column_blob)(sqlite3_stmt*, int);
  int (*column_bytes)(sqlite3_stmt*, int);
};

// Null when libsqlite3.so.0 or one of its entry points is missing. Resolved once, on the first save or load.
const SqliteApi* sqliteApi() {
  static const SqliteApi* api = []() -> const SqliteApi* {
    void* h = dlopen("libsqlite3.so.0", RTLD_NOW | RTLD_LOCAL);
    if (!h) return nullptr;
    static SqliteApi a;
    bool ok = true;
    auto get = [&](auto& fn, const char* name) {
      void* p = dlsym(h, name);
      ok = ok && p != nullptr;
      fn = reinterpret_cast<std::remove_reference_t<decltype(fn)>>(p);
    };
    get(a.open_v2, "sqlite3_open_v2"), get(a.close_v2, "sqlite3_close_v2"), get(a.errmsg, "sqlite3_errmsg");
    get(a.exec, "sqlite3_exec"), get(a.prepare_v2, "sqlite3_prepare_v2"), get(a.step, "sqlite3_step");
    get(a.reset, "sqlite3_reset"), get(a.finalize, "sqlite3_finalize"), get(a.bind_int, "sqlite3_bind_int");
    get(a.bind_text, "sqlite3_bind_text"), get(a.bind_null, "sqlite3_bind_null"), get(a.bind_blob, "sqlite3_bind_blob");
    get(a.column_int64, "sqlite3_column_int64"), get(a.column_double, "sqlite3_column_double");
    get(a.column_type, "sqlite3_column_type"), get(a.column_blob, "sqlite3_column_blob");
    get(a.column_bytes, "sqlite3_column_bytes");
    return ok ? &a : nullptr;
  }();
  return api;
}

// One open database and the statements prepared on it, all released by the destructor.
class Db {
 public:
  explicit Db(const SqliteApi* api) : api_(api) {}
  ~Db() {
    for (sqlite3_stmt* s : stmts_) api_->finalize(s);
    if (db_) api_->close_v2(db_);
  }
  bool open(const char* path, int flags, std::string* err) {
    if (api_->open_v2(path, &db_, flags, nullptr) == kSqliteOk) return true;
    return error(std::string("cannot open ") + path, err);
  }
  bool exec(const std::string& sql, std::string* err) {
    return api_->exec(db_, sql.c_str(), nullptr, nullptr, nullptr) == kSqliteOk || error(sql, err);
  }
  sqlite3_stmt* prepare(const std::string& sql, std::string* err) {
    sqlite3_stmt* s = nullptr;
    if (api_->prepare_v2(db_, sql.c_str(), -1, &s, nullptr) != kSqliteOk) {
      error(sql, err);
      return nullptr;
    }
    stmts_.push_back(s);
    return s;
  }
  bool error(const std::string& what, std::string* err) {
    *err = what + ": " + (db_ ? api_->errmsg(db_) : "out of memory");
    return false;
  }

 private:
  const SqliteApi* api_;
  sqlite3* db_ = nullptr;
  std::vector<sqlite3_stmt*> stmts_;
};

const char* const kTableNames[kMapFileLayers] = {"tsdf_layer", "esdf_layer", "occupancy_layer", "freespace_layer", "color_layer",
                                                 "feature_layer"};

}  // namespace

const char* mapFileTableName(int k) { return kTableNames[k]; }

int writeMapFile(const char* path, const MapFileLayerOut layers[kMapFileLayers], float block_size, std::string* err) {
  const SqliteApi* api = sqliteApi();
  if (!api) return *err = "libsqlite3.so.0 could not be loaded", NVB_ERR_IO;
  // the reference opens with std::ios::trunc, which removes an existing file first (sqlite_database.cpp)
  if (FILE* f = fopen(path, "rb")) {
    fclose(f);
    std::remove(path);
  }
  Db db(api);
  if (!db.open(path, kOpenReadWrite | kOpenCreate, err)) return NVB_ERR_IO;
  for (int k = 0; k < kMapFileLayers; k++) {
    const std::string L = kTableNames[k];
    const MapFileLayerOut& o = layers[k];
    // the reference's DDL, verbatim (serializer.cpp, createLayerTables)
    const std::string meta_ddl = "CREATE TABLE " + L + "_metadata" +
                                 "(param_name TEXT PRIMARY KEY UNIQUE NOT NULL,value_string TEXT,value_int INT,value_float FLOAT);";
    const std::string data_ddl = "CREATE TABLE " + L + "_data" +
                                 "(index_x INT NOT NULL,index_y INT NOT NULL,index_z INT NOT NULL,data BLOB,"
                                 "PRIMARY KEY(index_x, index_y, index_z));";
    if (!db.exec("BEGIN TRANSACTION;", err) || !db.exec(meta_ddl, err) || !db.exec(data_ddl, err)) return NVB_ERR_IO;
    sqlite3_stmt* meta = db.prepare("INSERT INTO " + L + "_metadata (param_name, value_string, value_float) VALUES (?1, ?2, ?3);", err);
    if (!meta) return NVB_ERR_IO;
    // ('type', value_string = L) and ('block_size', value_float): the float as std::to_string's six-decimal text, which the
    // FLOAT column stores as a REAL, like the reference's string-built statement
    const std::string bs = std::to_string(block_size);
    bool ok = api->bind_text(meta, 1, "type", -1, nullptr) == kSqliteOk && api->bind_text(meta, 2, L.c_str(), -1, nullptr) == kSqliteOk &&
              api->bind_null(meta, 3) == kSqliteOk && api->step(meta) == kSqliteDone && api->reset(meta) == kSqliteOk;
    ok = ok && api->bind_text(meta, 1, "block_size", -1, nullptr) == kSqliteOk && api->bind_null(meta, 2) == kSqliteOk &&
         api->bind_text(meta, 3, bs.c_str(), -1, nullptr) == kSqliteOk && api->step(meta) == kSqliteDone;
    if (!ok) return db.error("metadata of " + L, err), NVB_ERR_IO;
    if (o.n > 0) {
      sqlite3_stmt* ins = db.prepare("INSERT INTO " + L + "_data (index_x, index_y, index_z, data) VALUES (?1, ?2, ?3, ?4);", err);
      if (!ins) return NVB_ERR_IO;
      for (int i = 0; i < o.n; i++) {
        const int s = o.order[i];
        const int* xyz = o.xyz + 3 * (size_t)s;
        ok = api->bind_int(ins, 1, xyz[0]) == kSqliteOk && api->bind_int(ins, 2, xyz[1]) == kSqliteOk &&
             api->bind_int(ins, 3, xyz[2]) == kSqliteOk &&
             api->bind_blob(ins, 4, o.voxels + (size_t)s * o.block_bytes, o.block_bytes, nullptr) == kSqliteOk &&
             api->step(ins) == kSqliteDone && api->reset(ins) == kSqliteOk;
        if (!ok) return db.error("blocks of " + L, err), NVB_ERR_IO;
      }
    }
    if (!db.exec("END TRANSACTION;", err)) return NVB_ERR_IO;
  }
  return NVB_OK;
}

int readMapFile(const char* path, const bool want[kMapFileLayers], MapFileLayerIn in[kMapFileLayers], std::string* err) {
  const SqliteApi* api = sqliteApi();
  if (!api) return *err = "libsqlite3.so.0 could not be loaded", NVB_ERR_IO;
  Db db(api);
  if (!db.open(path, kOpenReadOnly, err)) return NVB_ERR_IO;
  // the layers of the file are its *_metadata tables (Serializer::getLayerNames)
  sqlite3_stmt* has = db.prepare("SELECT count(*) FROM sqlite_master WHERE type='table' AND name=?1;", err);
  if (!has) return NVB_ERR_IO;
  float block_size = 0.0f;
  for (int k = 0; k < kMapFileLayers; k++) {
    const std::string L = kTableNames[k];
    const std::string meta = L + "_metadata";
    if (api->bind_text(has, 1, meta.c_str(), -1, nullptr) != kSqliteOk || api->step(has) != kSqliteRow)
      return db.error(std::string("tables of ") + path, err), NVB_ERR_IO;
    in[k].present = api->column_int64(has, 0) > 0;
    api->reset(has);
    if (!in[k].present) continue;
    sqlite3_stmt* q = db.prepare("SELECT value_float FROM " + meta + " WHERE param_name='block_size';", err);
    if (!q) return NVB_ERR_IO;
    if (api->step(q) != kSqliteRow || api->column_type(q, 0) == kSqliteNull)
      return *err = L + " has no block_size", NVB_ERR_IO;
    in[k].block_size = (float)api->column_double(q, 0);
    if (!(in[k].block_size > 0.0f) || !std::isfinite(in[k].block_size))
      return *err = L + " has block_size " + std::to_string(in[k].block_size), NVB_ERR_IO;
    // the reference CHECKs that every layer's voxel size agrees (serializer.cpp, loadLayerCake)
    if (block_size != 0.0f && in[k].block_size != block_size)
      return *err = "the layers' block sizes differ (" + L + ": " + std::to_string(in[k].block_size) + ")", NVB_ERR_IO;
    block_size = in[k].block_size;
  }
  // Mapper::loadMap refuses a file without a TSDF layer (mapper.cpp:654-660)
  if (!in[NVB_LAYER_TSDF].present) return *err = std::string(path) + " has no tsdf_layer table", NVB_ERR_IO;
  for (int k = 0; k < kMapFileLayers; k++) {
    if (!in[k].present || !want[k]) continue;
    const std::string L = kTableNames[k];
    const int bytes = nvb_layer_block_bytes(k);
    sqlite3_stmt* cnt = db.prepare("SELECT count(*) FROM " + L + "_data;", err);
    if (!cnt) return NVB_ERR_IO;
    if (api->step(cnt) != kSqliteRow) return db.error("blocks of " + L, err), NVB_ERR_IO;
    const long long n = api->column_int64(cnt, 0);
    if (n > (1ll << 28)) return *err = L + " holds more than 2^28 blocks", NVB_ERR_CAPACITY;
    in[k].n = (int)n;
    in[k].xyz.resize(3 * (size_t)n);
    if (n > 0) {
      void* p = nullptr;
      if (cudaMallocHost(&p, (size_t)n * bytes) != cudaSuccess) return *err = "pinned staging of " + L, NVB_ERR_CUDA;
      in[k].voxels.reset(static_cast<unsigned char*>(p));
    }
    sqlite3_stmt* q = db.prepare("SELECT index_x,index_y,index_z,data FROM " + L + "_data ORDER BY index_x,index_y,index_z;", err);
    if (!q) return NVB_ERR_IO;
    long long i = 0;
    int rc;
    while ((rc = api->step(q)) == kSqliteRow) {
      if (i >= n) return *err = L + " changed while it was read", NVB_ERR_IO;
      const long long x = api->column_int64(q, 0), y = api->column_int64(q, 1), z = api->column_int64(q, 2);
      if (x < -kIndexBias || x >= kIndexBias || y < -kIndexBias || y >= kIndexBias || z < -kIndexBias || z >= kIndexBias)
        return *err = L + ": block index outside +-2^20", NVB_ERR_INDEX_RANGE;
      int* o = in[k].xyz.data() + 3 * i;
      o[0] = (int)x, o[1] = (int)y, o[2] = (int)z;
      if (i > 0 && o[0] == o[-3] && o[1] == o[-2] && o[2] == o[-1]) return *err = L + ": a block index appears twice", NVB_ERR_IO;
      const void* blob = api->column_blob(q, 3);
      const int nb = api->column_bytes(q, 3);
      if (nb != bytes || !blob)
        return *err = L + ": a block of " + std::to_string(nb) + " bytes, not " + std::to_string(bytes), NVB_ERR_IO;
      memcpy(in[k].voxels.get() + (size_t)i * bytes, blob, bytes);
      i++;
    }
    if (rc != kSqliteDone || i != n) return db.error("blocks of " + L, err), NVB_ERR_IO;
  }
  return NVB_OK;
}

// ---- ESDF parent boxes of loaded blocks: the words ownStore (nvb_esdf_wavex.cu) publishes, from the voxels in the slab.
// One 64-thread group per block, thread = (x, y) z-row, so warp 0 covers x < 4 and warp 1 x >= 4, as there.
__global__ void esdfParentBoxesKernel(DevLayer esdf, unsigned int* psum) {
  const int slot = blockIdx.x, lane64 = threadIdx.x;
  const int x = lane64 >> 3, y = lane64 & 7;
  const unsigned int* blk = reinterpret_cast<const unsigned int*>(esdf.blocks + (size_t)slot * kEsdfBlockBytes);
  int lo0 = 99, lo1 = 99, lo2 = 99, hi0 = -99, hi1 = -99, hi2 = -99;
#pragma unroll
  for (int z = 0; z < kVps; z++) {
    const unsigned int* c = esdfCell(blk, lane64 * kVps + z);
    const int px = (int)c[1], py = (int)c[2], pz = (int)c[3];
    if ((px | py | pz) != 0) {
      const int b0 = (x + px) >> 3, b1 = (y + py) >> 3, b2 = (z + pz) >> 3;  // floor: arithmetic shift
      lo0 = min(lo0, b0), hi0 = max(hi0, b0), lo1 = min(lo1, b1), hi1 = max(hi1, b1), lo2 = min(lo2, b2), hi2 = max(hi2, b2);
    }
  }
  lo0 = __reduce_min_sync(0xffffffffu, lo0), lo1 = __reduce_min_sync(0xffffffffu, lo1), lo2 = __reduce_min_sync(0xffffffffu, lo2);
  hi0 = __reduce_max_sync(0xffffffffu, hi0), hi1 = __reduce_max_sync(0xffffffffu, hi1), hi2 = __reduce_max_sync(0xffffffffu, hi2);
  if ((lane64 & 31) == 0) psum[2 * (size_t)slot + (lane64 >> 5)] = parentBoxWord(lo0, hi0, lo1, hi1, lo2, hi2);
}

void launchEsdfParentBoxes(const DevLayer& esdf, int n, unsigned int* psum, cudaStream_t stream) {
  if (n > 0) esdfParentBoxesKernel<<<n, 64, 0, stream>>>(esdf, psum);
}

// ---- Point export: io::outputVoxelLayerToPly's per-layer rule (pointcloud_io.cpp:23-73) for voxel v of a block.
__device__ __forceinline__ bool exportVoxel(const ExportPointsArgs& a, const unsigned char* blk, int v, float* intensity) {
  if (a.layer_id == NVB_LAYER_TSDF) {
    const float* t = reinterpret_cast<const float*>(blk) + 2 * v;
    *intensity = t[0];
    return t[1] > 1e-4f;
  }
  if (a.layer_id == NVB_LAYER_OCCUPANCY) {
    const float l = reinterpret_cast<const float*>(blk)[v];
    const float p = expf(l) / (1.0f + expf(l));  // probabilityFromLogOdds (core/log_odds.h:32-34)
    *intensity = p;
    return p > 0.5f;
  }
  if (a.layer_id == NVB_LAYER_FREESPACE) {
    *intensity = blk[(size_t)v * kFreespaceVoxelBytes + 16] ? 1.0f : 0.0f;  // is_high_confidence_freespace
    return true;
  }
  const unsigned int* b = reinterpret_cast<const unsigned int*>(blk);
  const unsigned int fl = *esdfFlag(b, v);
  float d = a.voxel_size * sqrtf(__uint_as_float(*esdfCell(b, v)));
  if (fl & 0xffu) d = -d;  // is_inside
  *intensity = d;
  return (fl & 0xff00u) != 0;  // observed
}

// One CTA per listed block, one thread per voxel (v = (x * 8 + y) * 8 + z, the order of voxels[x][y][z]).
__global__ void exportCountKernel(ExportPointsArgs a) {
  const int slot = a.slots[blockIdx.x];
  bool keep = false;
  float t;
  if (slot >= 0) keep = exportVoxel(a, a.layer.blocks + (size_t)slot * a.layer.block_bytes, threadIdx.x, &t);
  const int c = __syncthreads_count(keep);
  if (threadIdx.x == 0) a.counts[blockIdx.x] = make_int2(c, 0);
}

__global__ void exportEmitKernel(ExportPointsArgs a) {
  __shared__ int warp_base[kVpb / 32];
  const int slot = a.slots[blockIdx.x];
  if (slot < 0) return;
  const int v = threadIdx.x, lane = v & 31, w = v >> 5;
  float intensity = 0.0f;
  const bool keep = exportVoxel(a, a.layer.blocks + (size_t)slot * a.layer.block_bytes, v, &intensity);
  const unsigned int ballot = __ballot_sync(0xffffffffu, keep);
  if (lane == 0) warp_base[w] = __popc(ballot);
  __syncthreads();
  if (v == 0) {
    int s = a.counts[blockIdx.x].x;
    for (int i = 0; i < kVpb / 32; i++) {
      const int c = warp_base[i];
      warp_base[i] = s;
      s += c;
    }
  }
  __syncthreads();
  if (!keep) return;
  // getCenterPositionFromBlockIndexAndVoxelIndex (core/internal/impl/indexing_impl.h:50-81):
  // (block_size * block_index + voxel_size * voxel_index) + half_voxel_size, per axis
  const float bs = a.block_size, vs = bs * (1.0f / kVps), half = bs * (0.5f / kVps);
  const int* b = a.layer.block_index + 3 * (size_t)slot;
  float4 p;
  p.x = (bs * (float)b[0] + vs * (float)(v >> 6)) + half;
  p.y = (bs * (float)b[1] + vs * (float)((v >> 3) & 7)) + half;
  p.z = (bs * (float)b[2] + vs * (float)(v & 7)) + half;
  p.w = intensity;
  a.out[warp_base[w] + __popc(ballot & ((1u << lane) - 1u))] = p;
}

void launchExportCount(const ExportPointsArgs& a, cudaStream_t stream) {
  exportCountKernel<<<a.num_blocks, kVpb, 0, stream>>>(a);
  launchExclusiveScanInt2(a.counts, a.num_blocks, a.totals, stream);
}

void launchExportEmit(const ExportPointsArgs& a, cudaStream_t stream) { exportEmitKernel<<<a.num_blocks, kVpb, 0, stream>>>(a); }

}  // namespace nvb
