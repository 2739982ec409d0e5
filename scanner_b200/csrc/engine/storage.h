// storage.h -- a Scanner database directory on a POSIX file system: the descriptors and item files
// the decode -> evaluate -> save path reads and writes, in the reference's layout so that tables
// are interchangeable (scanner/engine/metadata.h:37-86 paths, metadata.proto descriptors,
// ingest.cpp:175-380 what ingest writes, column_sink.cpp:71-265 what a job writes):
//
//   <db>/db_metadata.bin                         DatabaseDescriptor (table name <-> id, next ids)
//   <db>/tables/<id>/descriptor.bin              TableDescriptor (columns, end_rows per item)
//   <db>/tables/<id>/<col>_<item>.bin            concatenated element bytes of the item
//   <db>/tables/<id>/<col>_<item>_metadata.bin   u64 n, then n x u64 element sizes (Bytes columns)
//   <db>/tables/<id>/<col>_<item>_video_metadata.bin   VideoDescriptor (Video columns)
//
// An ingested video is the table {column 0 "index": row i = int64 i; column 1 "frame": H.264
// Annex-B byte stream + VideoDescriptor with the sample / keyframe index}.  The storehouse
// abstraction (S3, GCS) of the reference is out of scope: POSIX only.
#pragma once
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "h264.h"
#include "scanner/util/common.h"
#include "table_formats.pb.h"

namespace scanner {
namespace internal {

struct ColumnSpec {
  std::string name;
  proto::ColumnType type = proto::Bytes;  // Video: rows are frames
  std::string type_name;
};

// One stored element column of one item, as the save stage hands it over.
struct ItemColumn {
  const u8* data = nullptr;
  size_t bytes = 0;
  const std::vector<u64>* sizes = nullptr;   // per row
  const std::vector<i32>* shapes = nullptr;  // 4 per row (h, w, c, frame type), frame columns only
  bool h264 = false;                         // the rows are the access units of one H.264 stream
};

class Database {
 public:
  // Opens (and creates if absent) the database rooted at `path`.
  static Result open(const std::string& path, std::unique_ptr<Database>& out);

  const std::string& path() const { return root_; }
  std::vector<std::string> table_names() const;
  bool has_table(const std::string& name) const;
  i32 table_id(const std::string& name) const;  // -1 if absent
  Result delete_table(const std::string& name);
  // Several tables under ONE catalogue lock and ONE rewrite of db_metadata.bin (a job with hundreds of output
  // streams would otherwise take the lock once per table, and ranks sharing the directory queue behind it)
  Result delete_tables(const std::vector<std::string>& names);

  // ---- ingest: `video_path` is an .mp4/.mov (demuxed here) or a raw H.264 Annex-B file
  // inplace (reference ingest.cpp:175-215 `inplace`): the bitstream is not copied into the database;
  // the descriptor records the absolute path and the sample table of the Annex-B view of that file
  // (what demuxing it yields), and binding the table demuxes the file again.
  Result ingest_video(const std::string& table, const std::string& video_path, bool inplace = false);
  Result ingest_h264(const std::string& table, const u8* annexb, size_t size, i32 time_base_num,
                     i32 time_base_denom, const std::string& inplace_path = "");
  // descriptor + the Annex-B bytes of a compressed video column, wherever they live
  Result load_video(const std::string& table, tables::VideoDescriptor& vd, std::vector<u8>& annexb) const;

  // ---- read side
  Result read_table(const std::string& table, tables::TableDescriptor& out) const;
  // descriptor of video column `column` (default: the first Video column) and its data file.  A compressed column
  // of several items (a job's output, one item per task) is described as one stream over all of them; item_files
  // then lists their data files in order.
  Result read_video(const std::string& table, tables::VideoDescriptor& out, std::string& data_file,
                    const std::string& column = "", std::vector<std::string>* item_files = nullptr) const;
  // rows of a column -> concatenated bytes + per-row sizes (+ shapes for frame columns)
  Result read_rows(const std::string& table, const std::string& column, const std::vector<i64>& rows,
                   std::vector<u8>& data, std::vector<u64>& sizes, std::vector<i32>& shapes) const;

  // ---- write side (a job's output table)
  // Reserves an id + directory; the table becomes visible with commit_table.
  Result new_table(const std::string& name, const std::vector<ColumnSpec>& columns, i32 job_id, i32& table_id);
  struct NewTable {
    std::string name;
    std::vector<ColumnSpec> columns;
    i32 job_id = -1;
  };
  Result new_tables(const std::vector<NewTable>& specs, std::vector<i32>& table_ids);
  std::string table_dir(i32 table_id) const;
  // Writes one item (= one task) of one column.  Index column (id 0) is written by write_index_item.
  Result write_item(i32 table_id, i32 column_id, i32 item_id, const ItemColumn& col, bool is_video);
  Result write_index_item(i32 table_id, i32 item_id, i64 row0, i64 row1);
  Result commit_table(i32 table_id, const std::vector<i64>& end_rows);
  Result commit_tables(const std::vector<std::pair<i32, std::vector<i64>>>& tables);

 private:
  Database() = default;
  Result load_meta();
  void refresh_meta();  // re-read db_metadata.bin (another process may have changed it)
  Result save_meta() const;
  std::string item_base(i32 table_id, i32 column_id, i32 item_id) const;

  std::string root_;  // with trailing '/'
  mutable std::mutex mu_;
  tables::DatabaseDescriptor meta_;
  std::map<i32, tables::TableDescriptor> pending_;  // new_table .. commit_table
};

// Fills an H264Index from a stored VideoDescriptor (no rescan of the byte stream).
Result index_from_descriptor(const tables::VideoDescriptor& vd, H264Index& out);

}  // namespace internal
}  // namespace scanner
