// evaluate.cpp -- see evaluate.h.  Row semantics follow reference
// scanner/engine/evaluate_worker.cpp:710-1261 (EvaluateWorker::feed):
//   * an op takes from its input columns only rows in valid_input_rows, in order (:772-807);
//   * compute row r is producible once clamp(r + stencil.back()) has arrived on every input
//     (:855-879); the producible count is rounded down to a whole number of batches unless fewer
//     than one batch of input rows remains in the task (:899-908);
//   * the stencil window for offset s is the cached element of row clamp(r+s, 0, domain-1)
//     (REPEAT_EDGE, :1078-1086);
//   * after execution only rows in valid_output_rows survive (:1146-1188) -- warmup rows are
//     computed and dropped; cached inputs no future compute row can touch are released
//     (:1190-1221); columns nobody downstream reads are released (:1225-1238).
// Differences by design: per-row lookups are binary searches over the (sorted) cache instead of a
// hash map rebuilt per packet; cross-device marshalling is one async DMA per contiguous run.
#include "evaluate.h"

#include <algorithm>

namespace scanner {
namespace internal {

namespace {
Result ok() {
  Result r;
  r.set_success(true);
  return r;
}
inline i64 clamp_row(i64 r, i64 domain) {
  if (r < 0) return 0;
  if (domain > 0 && r >= domain) return domain - 1;
  return r;
}
}  // namespace

void delete_elements(DeviceHandle device, Elements& elements) {
  for (Element& e : elements) delete_element(device, e);
  elements.clear();
}

Elements copy_or_ref_elements(DeviceHandle src, DeviceHandle dst, const Elements& in) {
  Elements out;
  out.reserve(in.size());
  if (src.is_same_address_space(dst)) {
    for (const Element& e : in) {
      Element c = add_element_ref(src, const_cast<Element&>(e));
      out.push_back(c);
    }
    return out;
  }
  // one block on the target for all payloads of this packet
  std::vector<size_t> sizes;
  std::vector<u8*> srcs;
  size_t total = 0;
  // an element without payload bytes crosses as a null element (stored rows cannot tell the two
  // apart: null = size 0, column_sink.cpp:181-195); giving it the address one past the block would
  // make delete_element reject it
  auto payload = [](const Element& e) -> size_t {
    return e.is_null() ? 0 : (e.is_frame ? e.as_const_frame()->size() : e.size);
  };
  for (const Element& e : in) {
    const size_t s = payload(e);
    if (s == 0) continue;
    sizes.push_back(s);
    srcs.push_back(e.is_frame ? e.as_const_frame()->data : e.buffer);
    total += s;
  }
  u8* block = sizes.empty() ? nullptr : new_block_buffer_sizes(dst, sizes);
  std::vector<u8*> dsts;
  size_t off = 0;
  for (size_t s : sizes) {
    dsts.push_back(block + off);
    off += s;
  }
  if (!sizes.empty()) memcpy_vec(dsts, dst, srcs, src, sizes);
  size_t k = 0;
  for (const Element& e : in) {
    Element c;
    if (payload(e) != 0) {
      if (e.is_frame) c = Element(new Frame(e.as_const_frame()->as_frame_info(), dsts[k]));
      else c = Element(dsts[k], e.size);
      ++k;
    }
    c.index = e.index;
    out.push_back(c);
  }
  (void)total;
  return out;
}

EvaluateWorker::EvaluateWorker(const Graph& graph, const GraphAnalysis& analysis, i32 gpu_id,
                               i32 node_id, Profiler* profiler, ResourceGate* gate)
  : graph_(graph), an_(analysis), gpu_id_(gpu_id), node_id_(node_id), profiler_(profiler), gate_(gate) {
  state_.resize(graph_.ops.size());
}

EvaluateWorker::~EvaluateWorker() {
  clear_caches();
  // kernels may hold device memory: destroy them while their device is still usable
  for (auto& st : state_) st.kernel.reset();
}

Result EvaluateWorker::init() {
  Result r;
  for (size_t i = 0; i < graph_.ops.size(); ++i) {
    const GraphOp& op = graph_.ops[i];
    OpState& st = state_[i];
    st.in_idx.assign(op.inputs.size(), 0);
    st.cache.resize(op.inputs.size());
    st.cache_rows.resize(op.inputs.size());
    if (op.kind != OpKind::Kernel) {
      // builtin ops pass elements through on whatever device they arrive
      continue;
    }
    const OpInfo* info = get_op_registry()->get_op_info(op.name);
    const KernelFactory* kf = get_kernel_registry()->get_kernel(op.name, op.device_type);
    if (!info || !kf) {
      RESULT_ERROR(&r, "Op %s has no %s kernel", op.name.c_str(), op.device_type == proto::GPU ? "GPU" : "CPU");
      return r;
    }
    auto handle_for = [&](proto::DeviceType t) {
      return t == proto::GPU ? DeviceHandle(DeviceType::GPU, gpu_id_) : CPU_DEVICE;
    };
    if (op.device_type == proto::GPU && gpu_id_ < 0) {
      RESULT_ERROR(&r, "Op %s requested a GPU kernel but this pipeline instance owns no GPU", op.name.c_str());
      return r;
    }
    st.device = handle_for(op.device_type);
    KernelConfig cfg;
    cfg.devices.push_back(st.device);
    cfg.node_id = node_id_;
    cfg.args = op.args;
    for (size_t k = 0; k < op.inputs.size(); ++k) {
      const std::string col_name =
          info->variadic_inputs ? op.inputs[k].column : info->input_columns[k].name;
      cfg.input_columns.push_back(col_name);
      cfg.input_column_types.push_back(info->variadic_inputs ? proto::Bytes : info->input_columns[k].type);
      auto it = kf->input_devices.find(col_name);
      st.in_dev.push_back(handle_for(it == kf->input_devices.end() ? op.device_type : it->second));
    }
    for (auto& c : info->output_columns) {
      cfg.output_columns.push_back(c.name);
      cfg.output_column_types.push_back(c.type);
      auto it = kf->output_devices.find(c.name);
      st.out_dev.push_back(handle_for(it == kf->output_devices.end() ? op.device_type : it->second));
    }
    st.kernel.reset(kf->new_instance(cfg));
    st.kernel->set_profiler(profiler_);
    Result v;
    st.kernel->validate(&v);
    if (!v.success()) {
      RESULT_ERROR(&r, "Op %s failed validation: %s", op.name.c_str(), v.msg().c_str());
      return r;
    }
    bool fetch_here = true;
    if (gate_) {
      std::unique_lock<std::mutex> lk(gate_->mu);
      int& s = gate_->state[(i32)i];
      if (s == 0) {
        s = 1;
      } else {
        fetch_here = false;
        gate_->cv.wait(lk, [&] { return gate_->state[(i32)i] >= 2; });
        if (gate_->state[(i32)i] == 3) {
          RESULT_ERROR(&r, "Op %s failed to fetch resources: %s", op.name.c_str(), gate_->error[(i32)i].c_str());
          return r;
        }
      }
    }
    if (fetch_here) {
      st.kernel->fetch_resources(&v);
      if (gate_) {
        std::lock_guard<std::mutex> lk(gate_->mu);
        gate_->state[(i32)i] = v.success() ? 2 : 3;
        if (!v.success()) gate_->error[(i32)i] = v.msg();
        gate_->cv.notify_all();
      }
      if (!v.success()) {
        RESULT_ERROR(&r, "Op %s failed to fetch resources: %s", op.name.c_str(), v.msg().c_str());
        return r;
      }
    }
    st.kernel->setup_with_resources(&v);
    if (!v.success()) {
      RESULT_ERROR(&r, "Op %s failed setup: %s", op.name.c_str(), v.msg().c_str());
      return r;
    }
  }
  return ok();
}

void EvaluateWorker::clear_caches() {
  for (size_t i = 0; i < state_.size(); ++i) {
    OpState& st = state_[i];
    for (size_t k = 0; k < st.cache.size(); ++k) {
      const DeviceHandle d = st.in_dev.size() > k ? st.in_dev[k] : st.device;
      for (Element& e : st.cache[k]) delete_element(d, e);
      st.cache[k].clear();
      st.cache_rows[k].clear();
    }
  }
}

Result EvaluateWorker::new_task(const JobParams& job, const std::vector<i64>& rows_per_op,
                                const std::vector<TaskStream>& task_streams) {
  Result r;
  clear_caches();
  for (size_t i = 0; i < graph_.ops.size(); ++i) {
    const GraphOp& op = graph_.ops[i];
    OpState& st = state_[i];
    st.ts = task_streams[i];
    std::fill(st.in_idx.begin(), st.in_idx.end(), 0);
    st.next_compute = 0;
    st.next_out = 0;
    st.domain_rows = op.inputs.empty() ? 0 : rows_per_op[op.inputs[0].op_index];
    st.sampler.reset();
    if (op.kind == OpKind::Sample || op.kind == OpKind::Space) {
      auto it = job.samplers.find((i32)i);
      if (it == job.samplers.end()) {
        RESULT_ERROR(&r, "no sampling args for op %zu", i);
        return r;
      }
      Result sr = make_domain_sampler(it->second.first, it->second.second, st.sampler);
      if (!sr.success()) return sr;
    }
    if (st.kernel) {
      st.kernel->reset();
      auto it = job.stream_args.find((i32)i);
      st.kernel->new_stream(it == job.stream_args.end() ? std::vector<u8>() : it->second);
      std::string kerr;
      if (take_kernel_error(&kerr)) {
        RESULT_ERROR(&r, "Op %s failed in reset / new_stream: %s", op.name.c_str(), kerr.c_str());
        return r;
      }
    }
  }
  return ok();
}

const Element* EvaluateWorker::find_cached(const OpState& st, size_t input, i64 row) const {
  const auto& rows = st.cache_rows[input];
  auto it = std::lower_bound(rows.begin(), rows.end(), row);
  if (it == rows.end() || *it != row) return nullptr;
  return &st.cache[input][(size_t)(it - rows.begin())];
}

Result EvaluateWorker::feed(std::map<i32, ColumnBatch>& source_columns,
                            std::map<i32, ColumnBatch>& sink_columns) {
  Result r;
  const size_t n = graph_.ops.size();
  // columns produced during this packet: cols[op][output column]
  std::vector<std::vector<ColumnBatch>> cols(n);
  std::vector<std::vector<bool>> have(n);
  for (size_t i = 0; i < n; ++i) {
    cols[i].resize(std::max<size_t>(1, graph_.ops[i].output_columns.size()));
    have[i].assign(cols[i].size(), false);
  }

  // Whatever this packet still owns when the function is left -- columns whose consumers all ran
  // on the normal path; on an error path also the rows handed in and the sink rows not handed out
  // yet -- is released exactly once, here.
  bool failed = true;
  struct AtExit {
    std::function<void()> fn;
    ~AtExit() { fn(); }
  } at_exit{[&] {
    for (size_t p = 0; p < n; ++p)
      for (size_t c = 0; c < cols[p].size(); ++c)
        if (have[p][c]) delete_elements(cols[p][c].device, cols[p][c].elements);
    if (!failed) return;
    for (auto& kv : source_columns) delete_elements(kv.second.device, kv.second.elements);
    source_columns.clear();
    for (auto& kv : sink_columns) delete_elements(kv.second.device, kv.second.elements);
    sink_columns.clear();
  }};

  auto release_dead = [&](size_t k) {
    // drop every column whose last reader is op k (liveness, reference :1225-1238)
    for (size_t p = 0; p < n; ++p)
      for (size_t c = 0; c < an_.last_use[p].size(); ++c)
        if (have[p][c] && an_.last_use[p][c] == (i32)k) {
          delete_elements(cols[p][c].device, cols[p][c].elements);
          cols[p][c].row_ids.clear();
          have[p][c] = false;
        }
  };

  for (size_t k = 0; k < n; ++k) {
    const GraphOp& op = graph_.ops[k];
    OpState& st = state_[k];
    const timepoint_t op_start = now();

    if (op.kind == OpKind::Source) {
      auto it = source_columns.find((i32)k);
      if (it != source_columns.end()) {
        cols[k][0] = std::move(it->second);
        have[k][0] = true;
        if (an_.last_use[k][0] < 0) {
          delete_elements(cols[k][0].device, cols[k][0].elements);
          have[k][0] = false;
        }
      }
      continue;
    }

    // ---- 1. pull the rows this op needs from its producers into its cache (op_marshal)
    for (size_t i = 0; i < op.inputs.size(); ++i) {
      const i32 p = op.inputs[i].op_index;
      const i32 c = an_.input_col_index[k][i];
      if (!have[p][c]) continue;
      const ColumnBatch& src = cols[p][c];
      Elements picked;
      std::vector<i64> picked_rows;
      size_t& idx = st.in_idx[i];
      for (size_t e = 0; e < src.row_ids.size(); ++e) {
        if (idx < st.ts.valid_input_rows.size() && src.row_ids[e] > st.ts.valid_input_rows[idx]) {
          RESULT_ERROR(&r, "Not enough rows in argument %zu for op %s: expected row %ld, saw %ld", i,
                       op.name.c_str(), (long)st.ts.valid_input_rows[idx], (long)src.row_ids[e]);
          return r;
        }
        if (idx < st.ts.valid_input_rows.size() && src.row_ids[e] == st.ts.valid_input_rows[idx]) {
          Element el = src.elements[e];
          el.index = src.row_ids[e];
          picked.push_back(el);
          picked_rows.push_back(src.row_ids[e]);
          ++idx;
        }
      }
      if (!picked.empty()) {
        const timepoint_t t0 = now();
        const DeviceHandle target = st.kernel ? st.in_dev[i] : src.device;
        if (!st.kernel && st.in_dev.size() <= i) st.in_dev.resize(i + 1, src.device);
        if (!st.kernel) st.in_dev[i] = src.device;
        Elements list = copy_or_ref_elements(src.device, target, picked);
        if (profiler_) profiler_->add_interval("op_marshal", t0, now());
        st.cache[i].insert(st.cache[i].end(), list.begin(), list.end());
        st.cache_rows[i].insert(st.cache_rows[i].end(), picked_rows.begin(), picked_rows.end());
      }
    }

    // ---- 2. how many compute rows can be produced now
    i64 max_row_seen = -1;
    bool any_empty = false;
    for (size_t i = 0; i < op.inputs.size(); ++i) {
      if (st.cache_rows[i].empty()) {
        any_empty = true;
        break;
      }
      max_row_seen = (i == 0) ? st.cache_rows[i].back() : std::min(max_row_seen, st.cache_rows[i].back());
    }
    if (any_empty) max_row_seen = -1;

    const std::vector<i32>& stencil = op.kind == OpKind::Kernel ? an_.stencil[k] : std::vector<i32>{0};
    static const std::vector<i32> kZero = {0};
    const std::vector<i32>& sten = op.kind == OpKind::Kernel ? stencil : kZero;
    i64 batch = op.kind == OpKind::Kernel ? an_.batch[k] : 1;
    const i64 rows_left = (i64)st.ts.valid_input_rows.size() - (i64)(st.in_idx.empty() ? 0 : st.in_idx[0]);
    i64 bs = batch;
    if (rows_left < batch) bs = 1;  // task tail: flush whatever is left (reference :899-906)
    i64 producible = 0;
    for (size_t q = st.next_compute; q < st.ts.compute_input_rows.size(); ++q) {
      const i64 need = clamp_row(st.ts.compute_input_rows[q] + sten.back(), st.domain_rows);
      if (need > max_row_seen) break;
      ++producible;
    }
    producible -= producible % bs;
    const size_t row_start = st.next_compute, row_end = st.next_compute + (size_t)producible;

    const size_t n_out = std::max<size_t>(1, op.output_columns.size());
    std::vector<ColumnBatch> produced(op.kind == OpKind::Sink ? 1 : n_out);
    // rows produced by earlier batches of this op in this packet, until step 4 hands them on
    bool produced_owned = true;
    AtExit drop_produced{[&] {
      if (!produced_owned) return;
      for (ColumnBatch& pc : produced) delete_elements(pc.device, pc.elements);
    }};

    // ---- 3. produce
    if (op.kind == OpKind::Sample || op.kind == OpKind::Space) {
      std::vector<i64> up(st.ts.compute_input_rows.begin() + row_start, st.ts.compute_input_rows.begin() + row_end);
      std::vector<i64> down, mapping;
      Result sr = st.sampler->get_downstream_rows(up, down, mapping);
      if (!sr.success()) return sr;
      const DeviceHandle d = st.in_dev.empty() ? CPU_DEVICE : st.in_dev[0];
      produced[0].device = d;
      for (size_t i = 0; i < down.size(); ++i) {
        if (mapping[i] < 0) {
          produced[0].elements.emplace_back();  // null element (SpaceNull)
        } else {
          const Element* e = find_cached(st, 0, up[(size_t)mapping[i]]);
          if (!e) {
            RESULT_ERROR(&r, "%s op %zu lost row %ld", op.name.c_str(), k, (long)up[(size_t)mapping[i]]);
            return r;
          }
          produced[0].elements.push_back(add_element_ref(d, const_cast<Element&>(*e)));
        }
        produced[0].row_ids.push_back(down[i]);
      }
    } else if (op.kind == OpKind::Sink) {
      const DeviceHandle d = st.in_dev.empty() ? CPU_DEVICE : st.in_dev[0];
      produced[0].device = d;
      for (size_t q = row_start; q < row_end; ++q) {
        const i64 row = st.ts.compute_input_rows[q];
        const Element* e = find_cached(st, 0, row);
        if (!e) {
          RESULT_ERROR(&r, "Sink %zu lost row %ld", k, (long)row);
          return r;
        }
        produced[0].elements.push_back(add_element_ref(d, const_cast<Element&>(*e)));
        produced[0].row_ids.push_back(row);
      }
    } else {  // regular kernel
      for (size_t c = 0; c < n_out; ++c) produced[c].device = st.out_dev[c];
      for (size_t start = row_start; start < row_end; start += (size_t)batch) {
        const size_t end = std::min(row_end, start + (size_t)batch);
        const size_t nb = end - start;
        StenciledBatchedElements in(op.inputs.size());
        for (size_t i = 0; i < op.inputs.size(); ++i) {
          in[i].resize(nb);
          for (size_t q = start; q < end; ++q) {
            Elements& window = in[i][q - start];
            window.reserve(sten.size());
            for (i32 s : sten) {
              const i64 want = clamp_row(st.ts.compute_input_rows[q] + s, st.domain_rows);
              const Element* e = find_cached(st, i, want);
              if (!e) {
                RESULT_ERROR(&r, "Op %s: stencil row %ld (compute row %ld, offset %d) is not cached", op.name.c_str(),
                             (long)want, (long)st.ts.compute_input_rows[q], s);
                return r;
              }
              window.push_back(*e);
            }
          }
        }
        BatchedElements out(n_out);
        const timepoint_t t0 = now();
        st.kernel->execute_kernel(in, out);
        if (profiler_) profiler_->add_interval("evaluate:" + op.name, t0, now());
        std::string kerr;
        if (take_kernel_error(&kerr)) {  // a host-language kernel failed: the run fails, the process lives
          for (size_t c = 0; c < n_out; ++c) delete_elements(st.out_dev[c], out[c]);
          RESULT_ERROR(&r, "Op %s failed: %s", op.name.c_str(), kerr.c_str());
          return r;
        }
        for (size_t c = 0; c < n_out; ++c) {
          if (out[c].size() != nb) {
            RESULT_ERROR(&r, "Op %s produced %zu output elements for column %zu. Expected %zu outputs.",
                         op.name.c_str(), out[c].size(), c, nb);
            // columns before c are already in `produced` (or freed); the rest are still the kernel's
            for (size_t c2 = c; c2 < n_out; ++c2) delete_elements(st.out_dev[c2], out[c2]);
            return r;
          }
          if (an_.last_use[k][c] < 0) {  // unused output: free immediately (:1105-1114)
            delete_elements(st.out_dev[c], out[c]);
            continue;
          }
          for (size_t q = 0; q < nb; ++q) {
            produced[c].elements.push_back(out[c][q]);
            produced[c].row_ids.push_back(st.ts.compute_input_rows[start + q]);
          }
        }
      }
    }
    st.next_compute = row_end;

    // ---- 4. keep only rows that are valid outputs of this op for this task (:1146-1188)
    produced_owned = false;  // from here every element of `produced` is either handed on or deleted
    if (op.kind == OpKind::Sink) {
      ColumnBatch& dst = sink_columns[(i32)k];
      dst.device = produced[0].device;
      dst.elements.insert(dst.elements.end(), produced[0].elements.begin(), produced[0].elements.end());
      dst.row_ids.insert(dst.row_ids.end(), produced[0].row_ids.begin(), produced[0].row_ids.end());
    } else {
      const size_t nrows = produced[0].row_ids.size();
      std::vector<bool> keep(nrows, false);
      // a column that is never read has no rows (freed above); use the first populated column
      size_t ref_col = 0;
      while (ref_col < produced.size() && produced[ref_col].row_ids.empty() && ref_col + 1 < produced.size()) ++ref_col;
      const std::vector<i64>& rows = produced[ref_col].row_ids;
      keep.assign(rows.size(), false);
      for (size_t q = 0; q < rows.size(); ++q) {
        while (st.next_out < st.ts.valid_output_rows.size() && st.ts.valid_output_rows[st.next_out] < rows[q])
          ++st.next_out;
        if (st.next_out < st.ts.valid_output_rows.size() && st.ts.valid_output_rows[st.next_out] == rows[q]) {
          keep[q] = true;
          ++st.next_out;
        }
      }
      for (size_t c = 0; c < produced.size(); ++c) {
        if (produced[c].row_ids.empty()) continue;
        ColumnBatch& dst = cols[k][c];
        dst.device = produced[c].device;
        for (size_t q = 0; q < produced[c].row_ids.size(); ++q) {
          if (keep[q]) {
            dst.elements.push_back(produced[c].elements[q]);
            dst.row_ids.push_back(produced[c].row_ids[q]);
          } else {
            delete_element(produced[c].device, produced[c].elements[q]);
          }
        }
        have[k][c] = true;
      }
    }

    // ---- 5. retire cached inputs no future compute row can reach (:1190-1221)
    {
      i64 min_needed;
      if (st.next_compute < st.ts.compute_input_rows.size())
        min_needed = clamp_row(st.ts.compute_input_rows[st.next_compute] + sten.front(), st.domain_rows);
      else
        min_needed = INT64_MAX;
      for (size_t i = 0; i < op.inputs.size(); ++i) {
        const DeviceHandle d = st.in_dev.size() > i ? st.in_dev[i] : CPU_DEVICE;
        while (!st.cache_rows[i].empty() && st.cache_rows[i].front() < min_needed) {
          delete_element(d, st.cache[i].front());
          st.cache[i].pop_front();
          st.cache_rows[i].pop_front();
        }
      }
    }
    release_dead(k);
    if (profiler_) profiler_->add_interval("op:" + op.name, op_start, now());
  }
  failed = false;
  return ok();
}

Result EvaluateWorker::end_task() {
  Result r;
  for (size_t i = 0; i < graph_.ops.size(); ++i) {
    const OpState& st = state_[i];
    for (size_t k = 0; k < st.in_idx.size(); ++k)
      if (st.in_idx[k] != st.ts.valid_input_rows.size()) {
        RESULT_ERROR(&r, "Evaluate worker did not use all rows for op %s input %zu: used %zu, expected %zu",
                     graph_.ops[i].name.c_str(), k, st.in_idx[k], st.ts.valid_input_rows.size());
        return r;
      }
    if (graph_.ops[i].kind != OpKind::Source && st.next_compute != st.ts.compute_input_rows.size()) {
      RESULT_ERROR(&r, "Op %s computed %zu of %zu rows", graph_.ops[i].name.c_str(), st.next_compute,
                   st.ts.compute_input_rows.size());
      return r;
    }
  }
  clear_caches();
  return ok();
}

}  // namespace internal
}  // namespace scanner
