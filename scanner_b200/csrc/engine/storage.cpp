// storage.cpp -- see storage.h.
#include "storage.h"

#include <thread>

#include <atomic>

#include <dirent.h>
#include <fcntl.h>
#include <sys/file.h>
#include <sys/stat.h>
#include <unistd.h>

#include <chrono>
#include <cstdio>
#include <cstring>
#include <fstream>

#include "mp4.h"

namespace scanner {
namespace internal {
namespace {

Result ok() {
  Result r;
  r.set_success(true);
  return r;
}

bool mkdirs(const std::string& path) {
  std::string cur;
  for (size_t i = 0; i <= path.size(); ++i) {
    if (i == path.size() || path[i] == '/') {
      if (!cur.empty() && cur != "/") {
        if (mkdir(cur.c_str(), 0755) != 0 && errno != EEXIST) return false;
      }
    }
    if (i < path.size()) cur.push_back(path[i]);
  }
  return true;
}

bool read_file(const std::string& path, std::string& out) {
  std::ifstream f(path, std::ios::binary | std::ios::ate);
  if (!f) return false;
  const std::streamsize n = f.tellg();
  f.seekg(0);
  out.resize((size_t)n);
  if (n) f.read(&out[0], n);
  return (bool)f;
}

// write to a temporary name, then rename: a reader never sees a half-written descriptor
bool write_file_atomic(const std::string& path, const void* data, size_t n) {
  const std::string tmp = path + ".tmp";
  {
    std::ofstream f(tmp, std::ios::binary | std::ios::trunc);
    if (!f) return false;
    if (n) f.write((const char*)data, (std::streamsize)n);
    if (!f) return false;
  }
  return rename(tmp.c_str(), path.c_str()) == 0;
}

void remove_tree(const std::string& dir) {
  DIR* d = opendir(dir.c_str());
  if (!d) return;
  while (dirent* e = readdir(d)) {
    const std::string name = e->d_name;
    if (name == "." || name == "..") continue;
    const std::string p = dir + "/" + name;
    struct stat st;
    if (lstat(p.c_str(), &st) == 0 && S_ISDIR(st.st_mode)) remove_tree(p);
    else unlink(p.c_str());
  }
  closedir(d);
  rmdir(dir.c_str());
}

// Exclusive advisory lock on <db>/db_metadata.lock for a read-modify-write of the catalogue: several
// processes (one rank per GPU) may share a database directory; the reference serialises these updates
// in its single master process.
class MetaLock {
 public:
  explicit MetaLock(const std::string& root) {
    fd_ = ::open((root + "db_metadata.lock").c_str(), O_CREAT | O_RDWR, 0644);
    if (fd_ >= 0) flock(fd_, LOCK_EX);
  }
  ~MetaLock() {
    if (fd_ >= 0) {
      flock(fd_, LOCK_UN);
      ::close(fd_);
    }
  }

 private:
  int fd_ = -1;
};

i64 now_seconds() {
  return std::chrono::duration_cast<std::chrono::seconds>(std::chrono::system_clock::now().time_since_epoch())
      .count();
}

}  // namespace

// ---------------------------------------------------------------------------------------------
Result Database::open(const std::string& path, std::unique_ptr<Database>& out) {
  Result r = ok();
  std::unique_ptr<Database> db(new Database());
  db->root_ = path;
  if (db->root_.empty()) {
    RESULT_ERROR(&r, "database path is empty");
    return r;
  }
  if (db->root_.back() != '/') db->root_.push_back('/');
  if (!mkdirs(db->root_ + "tables")) {
    RESULT_ERROR(&r, "cannot create database directory %s: %s", db->root_.c_str(), strerror(errno));
    return r;
  }
  r = db->load_meta();
  if (r.success()) out = std::move(db);
  return r;
}

Result Database::load_meta() {
  Result r = ok();
  std::string bytes;
  const std::string p = root_ + "db_metadata.bin";
  if (!read_file(p, bytes)) {  // fresh database (reference: master creates it on first start)
    // several ranks may open the same new directory at once: only one of them writes the empty catalogue, and
    // none overwrites a catalogue another rank has meanwhile created (and perhaps already added tables to)
    MetaLock file_lock(root_);
    if (!read_file(p, bytes)) {
      meta_ = tables::DatabaseDescriptor();
      return save_meta();
    }
  }
  if (!meta_.ParseFromString(bytes)) RESULT_ERROR(&r, "%s is not a DatabaseDescriptor", p.c_str());
  return r;
}

void Database::refresh_meta() {
  std::string bytes;
  tables::DatabaseDescriptor fresh;
  if (read_file(root_ + "db_metadata.bin", bytes) && fresh.ParseFromString(bytes)) meta_ = fresh;
}

Result Database::save_meta() const {
  Result r = ok();
  const std::string s = meta_.SerializeAsString();
  if (!write_file_atomic(root_ + "db_metadata.bin", s.data(), s.size()))
    RESULT_ERROR(&r, "cannot write %sdb_metadata.bin: %s", root_.c_str(), strerror(errno));
  return r;
}

std::vector<std::string> Database::table_names() const {
  std::lock_guard<std::mutex> g(mu_);
  const_cast<Database*>(this)->refresh_meta();
  std::vector<std::string> out;
  for (const auto& t : meta_.tables())
    if (t.committed()) out.push_back(t.name());
  return out;
}

i32 Database::table_id(const std::string& name) const {
  std::lock_guard<std::mutex> g(mu_);
  const_cast<Database*>(this)->refresh_meta();
  for (const auto& t : meta_.tables())
    if (t.committed() && t.name() == name) return t.id();
  return -1;
}

bool Database::has_table(const std::string& name) const { return table_id(name) >= 0; }

std::string Database::table_dir(i32 id) const { return root_ + "tables/" + std::to_string(id); }

std::string Database::item_base(i32 table_id, i32 column_id, i32 item_id) const {
  return table_dir(table_id) + "/" + std::to_string(column_id) + "_" + std::to_string(item_id);
}

Result Database::delete_table(const std::string& name) { return delete_tables({name}); }

Result Database::delete_tables(const std::vector<std::string>& names) {
  Result r = ok();
  std::vector<i32> ids;
  {
    std::lock_guard<std::mutex> g(mu_);
    MetaLock file_lock(root_);
    refresh_meta();
    auto* ts = meta_.mutable_tables();
    for (const std::string& name : names) {
      i32 id = -1;
      for (size_t i = 0; i < ts->size(); ++i)
        if ((*ts)[i].name() == name) {
          id = (*ts)[i].id();
          ts->erase(ts->begin() + (long)i);
          break;
        }
      if (id < 0) {
        RESULT_ERROR(&r, "table %s does not exist", name.c_str());
        break;
      }
      ids.push_back(id);
    }
    Result sr = save_meta();  // tables found before a missing one are gone either way
    if (r.success()) r = sr;
  }
  for (i32 id : ids) remove_tree(table_dir(id));
  return r;
}

Result Database::new_table(const std::string& name, const std::vector<ColumnSpec>& columns, i32 job_id,
                           i32& table_id) {
  std::vector<i32> ids;
  Result r = new_tables({NewTable{name, columns, job_id}}, ids);
  if (r.success()) table_id = ids[0];
  return r;
}

Result Database::new_tables(const std::vector<NewTable>& specs, std::vector<i32>& table_ids) {
  Result r = ok();
  table_ids.clear();
  std::lock_guard<std::mutex> g(mu_);
  MetaLock file_lock(root_);
  refresh_meta();
  for (size_t k = 0; k < specs.size(); ++k) {
    const std::string& name = specs[k].name;
    bool taken = false;
    for (const auto& t : meta_.tables()) taken = taken || t.name() == name;
    if (taken) {
      refresh_meta();  // drop the entries added so far: nothing of this call is kept
      for (i32 id : table_ids) pending_.erase(id);
      table_ids.clear();
      RESULT_ERROR(&r, "table %s already exists", name.c_str());
      return r;
    }
    const i32 table_id = meta_.next_table_id();
    meta_.set_next_table_id(table_id + 1);
    tables::DbTable* t = meta_.add_tables();
    t->set_id(table_id);
    t->set_name(name);
    t->set_committed(false);
    tables::TableDescriptor td;
    td.set_id(table_id);
    td.set_name(name);
    td.set_job_id(specs[k].job_id);
    td.set_timestamp(now_seconds());
    {
      tables::ColumnDescriptor* c = td.add_columns();  // column 0 is always the index column
      c->set_id(0);
      c->set_name("index");
      c->set_type((int)proto::Bytes);
    }
    for (size_t i = 0; i < specs[k].columns.size(); ++i) {
      tables::ColumnDescriptor* c = td.add_columns();
      c->set_id((i32)i + 1);
      c->set_name(specs[k].columns[i].name);
      c->set_type((int)specs[k].columns[i].type);
      c->set_type_name(specs[k].columns[i].type_name);
    }
    pending_[table_id] = td;
    table_ids.push_back(table_id);
    if (!mkdirs(table_dir(table_id))) {
      RESULT_ERROR(&r, "cannot create %s: %s", table_dir(table_id).c_str(), strerror(errno));
      return r;
    }
  }
  return save_meta();
}

Result Database::write_index_item(i32 table_id, i32 item_id, i64 row0, i64 row1) {
  // reference ingest.cpp:321-345: row i = little-endian int64 i, metadata = n then n sizes of 8
  std::vector<i64> idx;
  for (i64 i = row0; i < row1; ++i) idx.push_back(i);
  std::vector<u64> sizes(idx.size(), 8);
  ItemColumn c;
  c.data = (const u8*)idx.data();
  c.bytes = idx.size() * 8;
  c.sizes = &sizes;
  return write_item(table_id, 0, item_id, c, false);
}

// The H.264 part of a VideoDescriptor from the index of its `bytes`-byte stream (reference ingest.cpp:211-224,
// 347-366): ingested videos and the items of compressed job outputs are described alike.
static void describe_h264(const H264Index& idx, size_t bytes, tables::VideoDescriptor& vd) {
  vd.set_frames(idx.frames());
  vd.set_width(idx.width);
  vd.set_height(idx.height);
  vd.set_channels(3);
  vd.set_frame_type((int)proto::U8);
  vd.set_codec_type(0);
  vd.set_chroma_format(1);
  vd.set_num_encoded_videos(1);
  vd.add_frames_per_video(idx.frames());
  vd.add_keyframes_per_video((i64)idx.keyframe_indices.size());
  vd.add_size_per_video((i64)bytes);
  for (u64 v : idx.sample_offsets) vd.add_sample_offsets(v);
  for (u64 v : idx.sample_sizes) vd.add_sample_sizes(v);
  for (i64 v : idx.keyframe_indices) vd.add_keyframe_indices((u64)v);
  vd.mutable_metadata_packets()->assign((const char*)idx.metadata_packets.data(), idx.metadata_packets.size());
}

Result Database::write_item(i32 table_id, i32 column_id, i32 item_id, const ItemColumn& col, bool is_video) {
  Result r = ok();
  const std::string base = item_base(table_id, column_id, item_id);
  {
    std::ofstream f(base + ".bin", std::ios::binary | std::ios::trunc);
    if (col.bytes) f.write((const char*)col.data, (std::streamsize)col.bytes);
    if (!f) {
      RESULT_ERROR(&r, "cannot write %s.bin: %s", base.c_str(), strerror(errno));
      return r;
    }
  }
  const std::vector<u64> none;
  const std::vector<u64>& sizes = col.sizes ? *col.sizes : none;
  if (!is_video) {
    std::string m;
    const u64 n = sizes.size();
    m.append((const char*)&n, 8);
    if (n) m.append((const char*)sizes.data(), 8 * sizes.size());
    if (!write_file_atomic(base + "_metadata.bin", m.data(), m.size()))
      RESULT_ERROR(&r, "cannot write %s_metadata.bin: %s", base.c_str(), strerror(errno));
    return r;
  }
  tables::VideoDescriptor vd;
  vd.set_table_id(table_id);
  vd.set_column_id(column_id);
  vd.set_item_id(item_id);
  if (col.h264) {
    // the rows are the access units of one stream (scn_job_set_sink_encoding): indexed like an ingested video
    H264Index idx;
    r = index_bytestream(col.data, col.bytes, idx);
    if (!r.success()) return r;
    if ((size_t)idx.frames() != sizes.size()) {
      RESULT_ERROR(&r, "item %d of table %d: %ld pictures in the H.264 stream of %zu rows", item_id, table_id,
                   (long)idx.frames(), sizes.size());
      return r;
    }
    describe_h264(idx, col.bytes, vd);
    vd.set_data_path(base + ".bin");
    const std::string s = vd.SerializeAsString();
    if (!write_file_atomic(base + "_video_metadata.bin", s.data(), s.size()))
      RESULT_ERROR(&r, "cannot write %s_video_metadata.bin: %s", base.c_str(), strerror(errno));
    return r;
  }
  // frame column stored uncompressed (reference column_sink.cpp:159-176): codec RAW, one "sample"
  // per frame so rows stay addressable; null rows have size 0
  vd.set_frames((i64)sizes.size());
  vd.set_codec_type(2);
  vd.set_chroma_format(1);
  u64 off = 0;
  bool have_shape = false;
  for (size_t i = 0; i < sizes.size(); ++i) {
    vd.add_sample_offsets(off);
    vd.add_sample_sizes(sizes[i]);
    off += sizes[i];
    if (sizes[i] && col.shapes && col.shapes->size() >= 4 * (i + 1)) {
      const i32* sh = col.shapes->data() + 4 * i;
      if (!have_shape) {
        vd.set_height(sh[0]);
        vd.set_width(sh[1]);
        vd.set_channels(sh[2]);
        vd.set_frame_type(sh[3]);
        have_shape = true;
      } else if (sh[0] != vd.height() || sh[1] != vd.width() || sh[2] != vd.channels() || sh[3] != vd.frame_type()) {
        // a VideoDescriptor carries ONE frame shape per item (metadata.proto:63-128); rows of another
        // shape could be stored but never read back
        RESULT_ERROR(&r, "frame column %d of table %d: row %zu of item %d is %dx%dx%d, earlier rows are %dx%dx%d "
                         "(frames of one stored item must share a shape)",
                     column_id, table_id, i, item_id, sh[0], sh[1], sh[2], vd.height(), vd.width(), vd.channels());
        return r;
      }
    }
  }
  vd.set_num_encoded_videos(1);
  vd.add_frames_per_video((i64)sizes.size());
  vd.add_keyframes_per_video((i64)sizes.size());
  vd.add_size_per_video((i64)off);
  vd.set_data_path(base + ".bin");
  const std::string s = vd.SerializeAsString();
  if (!write_file_atomic(base + "_video_metadata.bin", s.data(), s.size()))
    RESULT_ERROR(&r, "cannot write %s_video_metadata.bin: %s", base.c_str(), strerror(errno));
  return r;
}

Result Database::commit_table(i32 table_id, const std::vector<i64>& end_rows) {
  return commit_tables({{table_id, end_rows}});
}

Result Database::commit_tables(const std::vector<std::pair<i32, std::vector<i64>>>& tables) {
  Result r = ok();
  std::lock_guard<std::mutex> g(mu_);
  std::vector<std::pair<i32, std::string>> files;  // (table id, serialised descriptor)
  for (const auto& te : tables) {
    auto it = pending_.find(te.first);
    if (it == pending_.end()) {
      RESULT_ERROR(&r, "table id %d is not being written", te.first);
      return r;
    }
    tables::TableDescriptor& td = it->second;
    td.clear_end_rows();
    for (i64 e : te.second) td.add_end_rows(e);
    files.emplace_back(te.first, td.SerializeAsString());
  }
  // One small file per table (create, write, rename): a job list with hundreds of output tables writes them from a
  // few threads -- at 8 ranks x 112 tables per step this was most of the commit's ~25 ms
  const size_t workers = files.size() >= 64 ? 4 : 1;
  std::atomic<size_t> next{0};
  std::atomic<int> failed_id{-1};
  std::atomic<int> failed_errno{0};
  auto write_some = [&] {
    for (size_t k = next.fetch_add(1); k < files.size(); k = next.fetch_add(1)) {
      const std::string& bytes = files[k].second;
      if (!write_file_atomic(table_dir(files[k].first) + "/descriptor.bin", bytes.data(), bytes.size())) {
        failed_errno = errno;
        failed_id = files[k].first;
      }
    }
  };
  {
    std::vector<std::thread> pool;
    for (size_t t = 1; t < workers; ++t) pool.emplace_back(write_some);
    write_some();
    for (auto& th : pool) th.join();
  }
  if (failed_id.load() >= 0) {
    RESULT_ERROR(&r, "cannot write the descriptor of table %d: %s", failed_id.load(), strerror(failed_errno.load()));
    return r;
  }
  MetaLock file_lock(root_);
  refresh_meta();
  for (const auto& te : tables) {
    for (auto& t : *meta_.mutable_tables())
      if (t.id() == te.first) t.set_committed(true);
    pending_.erase(te.first);
  }
  return save_meta();
}

// ---------------------------------------------------------------------------------------------
Result Database::ingest_video(const std::string& table, const std::string& video_path, bool inplace) {
  Result r = ok();
  std::string keep;
  if (inplace) {
    char* abs = realpath(video_path.c_str(), nullptr);
    if (!abs) {
      RESULT_ERROR(&r, "cannot read %s: %s", video_path.c_str(), strerror(errno));
      return r;
    }
    keep = abs;
    free(abs);
  }
  std::string bytes;
  if (!read_file(video_path, bytes)) {
    RESULT_ERROR(&r, "cannot read %s: %s", video_path.c_str(), strerror(errno));
    return r;
  }
  const u8* p = (const u8*)bytes.data();
  if (looks_like_mp4(p, bytes.size())) {
    Mp4Track trk;
    r = demux_mp4(p, bytes.size(), trk);
    if (!r.success()) return r;
    // time base of one tick (reference stores the codec context's time_base, ingest.cpp:303-304)
    return ingest_h264(table, trk.annexb.data(), trk.annexb.size(), 1, (i32)trk.timescale, keep);
  }
  return ingest_h264(table, p, bytes.size(), 1, 25, keep);
}

Result Database::ingest_h264(const std::string& table, const u8* annexb, size_t size, i32 tb_num, i32 tb_den,
                             const std::string& inplace_path) {
  H264Index idx;
  Result r = index_bytestream(annexb, size, idx);
  if (!r.success()) return r;
  if (idx.frames() == 0) {
    RESULT_ERROR(&r, "no H.264 pictures found while ingesting table %s", table.c_str());
    return r;
  }
  i32 id = -1;
  r = new_table(table, {ColumnSpec{"frame", proto::Video, ""}}, -1, id);
  if (!r.success()) return r;
  const std::string base = item_base(id, 1, 0);
  if (inplace_path.empty()) {
    std::ofstream f(base + ".bin", std::ios::binary | std::ios::trunc);
    f.write((const char*)annexb, (std::streamsize)size);
    if (!f) {
      RESULT_ERROR(&r, "cannot write %s.bin: %s", base.c_str(), strerror(errno));
      return r;
    }
  }
  tables::VideoDescriptor vd;
  vd.set_table_id(id);
  vd.set_column_id(1);
  vd.set_item_id(0);
  describe_h264(idx, size, vd);
  vd.set_time_base_num(tb_num);
  vd.set_time_base_denom(tb_den);
  vd.set_data_path(inplace_path.empty() ? base + ".bin" : inplace_path);
  vd.set_inplace(!inplace_path.empty());
  const std::string s = vd.SerializeAsString();
  if (!write_file_atomic(base + "_video_metadata.bin", s.data(), s.size())) {
    RESULT_ERROR(&r, "cannot write %s_video_metadata.bin: %s", base.c_str(), strerror(errno));
    return r;
  }
  r = write_index_item(id, 0, 0, idx.frames());
  if (!r.success()) return r;
  return commit_table(id, {idx.frames()});
}

// ---------------------------------------------------------------------------------------------
Result Database::read_table(const std::string& table, tables::TableDescriptor& out) const {
  Result r = ok();
  const i32 id = table_id(table);
  if (id < 0) {
    RESULT_ERROR(&r, "table %s does not exist", table.c_str());
    return r;
  }
  std::string bytes;
  const std::string p = table_dir(id) + "/descriptor.bin";
  if (!read_file(p, bytes) || !out.ParseFromString(bytes)) RESULT_ERROR(&r, "cannot read %s", p.c_str());
  return r;
}

Result Database::read_video(const std::string& table, tables::VideoDescriptor& out, std::string& data_file,
                            const std::string& column, std::vector<std::string>* item_files) const {
  tables::TableDescriptor td;
  Result r = read_table(table, td);
  if (!r.success()) return r;
  i32 col = -1;
  for (const auto& c : td.columns())
    if (c.type() == (int)proto::Video && (column.empty() || c.name() == column)) {
      col = c.id();
      break;
    }
  if (col < 0) {
    RESULT_ERROR(&r, "table %s has no video column %s", table.c_str(), column.c_str());
    return r;
  }
  auto read_item = [&](i32 item, tables::VideoDescriptor& vd) {
    const std::string base = item_base(td.id(), col, item);
    std::string bytes;
    if (!read_file(base + "_video_metadata.bin", bytes) || !vd.ParseFromString(bytes))
      RESULT_ERROR(&r, "cannot read %s_video_metadata.bin", base.c_str());
    // the stored data_path is absolute for the writer's mount point; the file next to the
    // descriptor is authoritative (a database directory can be moved)
    return base + ".bin";
  };
  data_file = read_item(0, out);
  if (item_files) item_files->assign(1, data_file);
  if (!r.success() || out.codec_type() != 0 || td.end_rows_size() <= 1) return r;
  // A job writes one item per task, so a compressed output column has several: they read as one stream, samples
  // back to back, keyframe indices offset by each item's first row.
  i64 bytes = out.size_per_video_size() ? out.size_per_video(0) : 0;
  for (i32 item = 1; item < td.end_rows_size(); ++item) {
    tables::VideoDescriptor vd;
    const std::string file = read_item(item, vd);
    if (!r.success()) return r;
    const i64 first = td.end_rows(item - 1);
    if (vd.codec_type() != 0 || vd.width() != out.width() || vd.height() != out.height() || first != out.frames() ||
        vd.size_per_video_size() != 1) {
      RESULT_ERROR(&r, "item %d of video column %d of table %s (%s, %dx%d, from row %ld) does not continue item 0's "
                       "H.264 stream (%dx%d, %ld rows before it): the items of a compressed column must share one "
                       "geometry to be read as one stream", item, col, table.c_str(),
                   vd.codec_type() == 0 ? "H.264" : "not H.264", vd.width(), vd.height(), (long)first, out.width(),
                   out.height(), (long)out.frames());
      return r;
    }
    for (u64 o : vd.sample_offsets()) out.add_sample_offsets(o + (u64)bytes);
    for (u64 z : vd.sample_sizes()) out.add_sample_sizes(z);
    for (u64 k : vd.keyframe_indices()) out.add_keyframe_indices(k + (u64)first);
    out.set_frames(out.frames() + vd.frames());
    bytes += vd.size_per_video(0);
    if (item_files) item_files->push_back(file);
  }
  out.clear_frames_per_video();
  out.add_frames_per_video(out.frames());
  out.clear_keyframes_per_video();
  out.add_keyframes_per_video(out.keyframe_indices_size());
  out.clear_size_per_video();
  out.add_size_per_video(bytes);
  return r;
}

Result Database::load_video(const std::string& table, tables::VideoDescriptor& vd, std::vector<u8>& annexb) const {
  std::string file;
  std::vector<std::string> items;
  Result r = read_video(table, vd, file, "", &items);
  if (!r.success()) return r;
  if (items.size() > 1) {  // a compressed job output: its items back to back
    annexb.clear();
    for (const std::string& f : items) {
      std::string part;
      if (!read_file(f, part)) {
        RESULT_ERROR(&r, "cannot read %s (video data of table %s): %s", f.c_str(), table.c_str(), strerror(errno));
        return r;
      }
      annexb.insert(annexb.end(), part.begin(), part.end());
    }
    if ((i64)annexb.size() != vd.size_per_video(0))
      RESULT_ERROR(&r, "table %s: its items hold %zu stream bytes, their descriptors %ld", table.c_str(),
                   annexb.size(), (long)vd.size_per_video(0));
    return r;
  }
  if (vd.inplace()) file = vd.data_path();
  std::string bytes;
  if (!read_file(file, bytes)) {
    RESULT_ERROR(&r, "cannot read %s (video data of table %s%s): %s", file.c_str(), table.c_str(),
                 vd.inplace() ? ", ingested in place" : "", strerror(errno));
    return r;
  }
  const u8* p = (const u8*)bytes.data();
  if (vd.inplace() && looks_like_mp4(p, bytes.size())) {
    Mp4Track trk;
    r = demux_mp4(p, bytes.size(), trk);
    if (!r.success()) return r;
    annexb.swap(trk.annexb);
  } else {
    annexb.assign(p, p + bytes.size());
  }
  if (vd.inplace() && vd.size_per_video_size() > 0 && (i64)annexb.size() != vd.size_per_video(0)) {
    RESULT_ERROR(&r, "%s changed since table %s was ingested in place (%zu stream bytes now, %ld then)", file.c_str(),
                 table.c_str(), annexb.size(), (long)vd.size_per_video(0));
    return r;
  }
  return r;
}

Result Database::read_rows(const std::string& table, const std::string& column, const std::vector<i64>& rows,
                           std::vector<u8>& data, std::vector<u64>& sizes, std::vector<i32>& shapes) const {
  tables::TableDescriptor td;
  Result r = read_table(table, td);
  if (!r.success()) return r;
  const tables::ColumnDescriptor* cd = nullptr;
  for (const auto& c : td.columns())
    if (c.name() == column) cd = &c;
  if (!cd) {
    RESULT_ERROR(&r, "table %s has no column %s", table.c_str(), column.c_str());
    return r;
  }
  const bool video = cd->type() == (int)proto::Video;
  // item -> (row offsets, sizes) loaded lazily
  struct Item {
    std::vector<u64> offs, sizes;
    i32 shape[4] = {0, 0, 0, -1};
    std::ifstream f;
  };
  std::map<i32, Item> items;
  data.clear();
  sizes.clear();
  shapes.clear();
  const i64 total = td.end_rows_size() ? td.end_rows(td.end_rows_size() - 1) : 0;
  for (i64 row : rows) {
    if (row < 0 || row >= total) {
      RESULT_ERROR(&r, "row %ld is outside table %s (%ld rows)", (long)row, table.c_str(), (long)total);
      return r;
    }
    i32 item = 0;
    while (item < td.end_rows_size() && row >= td.end_rows(item)) ++item;
    const i64 first = item ? td.end_rows(item - 1) : 0;
    auto it = items.find(item);
    if (it == items.end()) {
      Item& I = items[item];
      const std::string base = item_base(td.id(), cd->id(), item);
      std::string bytes;
      if (video) {
        tables::VideoDescriptor vd;
        if (!read_file(base + "_video_metadata.bin", bytes) || !vd.ParseFromString(bytes)) {
          RESULT_ERROR(&r, "cannot read %s_video_metadata.bin", base.c_str());
          return r;
        }
        if (vd.codec_type() != 2) {
          RESULT_ERROR(&r, "column %s of table %s is compressed video: decode it through a job", column.c_str(),
                       table.c_str());
          return r;
        }
        I.offs = vd.sample_offsets();
        I.sizes = vd.sample_sizes();
        if (I.offs.size() != I.sizes.size()) {
          RESULT_ERROR(&r, "%s_video_metadata.bin: %zu sample offsets for %zu sizes", base.c_str(), I.offs.size(),
                       I.sizes.size());
          return r;
        }
        I.shape[0] = vd.height();
        I.shape[1] = vd.width();
        I.shape[2] = vd.channels();
        I.shape[3] = vd.frame_type();
      } else {
        if (!read_file(base + "_metadata.bin", bytes) || bytes.size() < 8) {
          RESULT_ERROR(&r, "cannot read %s_metadata.bin", base.c_str());
          return r;
        }
        u64 n;
        memcpy(&n, bytes.data(), 8);
        if (n > (bytes.size() - 8) / 8) {  // (not 8 + 8 * n: n comes from the file and may overflow)
          RESULT_ERROR(&r, "%s_metadata.bin is truncated", base.c_str());
          return r;
        }
        I.sizes.resize(n);
        if (n) memcpy(I.sizes.data(), bytes.data() + 8, 8 * n);
        u64 off = 0;
        for (u64 s : I.sizes) {
          I.offs.push_back(off);
          off += s;
        }
      }
      I.f.open(base + ".bin", std::ios::binary);
      if (!I.f) {
        RESULT_ERROR(&r, "cannot open %s.bin", base.c_str());
        return r;
      }
      it = items.find(item);
    }
    Item& I = it->second;
    const size_t k = (size_t)(row - first);
    if (k >= I.sizes.size()) {
      RESULT_ERROR(&r, "item %d of %s.%s holds %zu rows, row %ld wanted", item, table.c_str(), column.c_str(),
                   I.sizes.size(), (long)row);
      return r;
    }
    const size_t at = data.size();
    data.resize(at + I.sizes[k]);
    if (I.sizes[k]) {
      I.f.seekg((std::streamoff)I.offs[k]);
      I.f.read((char*)data.data() + at, (std::streamsize)I.sizes[k]);
      if (!I.f) {
        RESULT_ERROR(&r, "short read in item %d of %s.%s", item, table.c_str(), column.c_str());
        return r;
      }
    }
    sizes.push_back(I.sizes[k]);
    shapes.insert(shapes.end(), I.shape, I.shape + 4);
  }
  return r;
}

Result index_from_descriptor(const tables::VideoDescriptor& vd, H264Index& out) {
  Result r = ok();
  if (vd.codec_type() != 0) {
    RESULT_ERROR(&r, "video column is not H.264 (codec type %d)", vd.codec_type());
    return r;
  }
  // coded size and cropping come from the stored SPS
  H264Index meta;
  const std::string& mp = vd.metadata_packets();
  r = index_bytestream((const u8*)mp.data(), mp.size(), meta, true);
  if (!r.success()) return r;
  out = H264Index();
  out.width = vd.width();
  out.height = vd.height();
  out.coded_width = meta.coded_width;
  out.coded_height = meta.coded_height;
  out.may_reorder = meta.may_reorder;
  out.sample_offsets = vd.sample_offsets();
  out.sample_sizes = vd.sample_sizes();
  for (u64 k : vd.keyframe_indices()) out.keyframe_indices.push_back((i64)k);
  out.metadata_packets.assign(mp.begin(), mp.end());
  if ((i64)out.sample_offsets.size() != vd.frames() || out.sample_sizes.size() != out.sample_offsets.size()) {
    RESULT_ERROR(&r, "video descriptor is inconsistent: %ld frames, %zu offsets, %zu sizes", (long)vd.frames(),
                 out.sample_offsets.size(), out.sample_sizes.size());
  }
  return r;
}

}  // namespace internal
}  // namespace scanner
