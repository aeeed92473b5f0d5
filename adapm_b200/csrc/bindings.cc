// Python bindings of the core (pybind11 only: tensors cross the boundary as raw
// addresses, so the extension does not depend on a particular torch ABI). The
// torch/numpy-facing API with the reference's method names (bindings/bindings.cc:79-374)
// lives in adapm_b200/__init__.py on top of these classes.
#include <pybind11/functional.h>
#include <pybind11/pybind11.h>
#include <pybind11/stl.h>

#include <pybind11/numpy.h>

#include "adapm/corpus.h"
#include "adapm/io.h"
#include "adapm/node.h"
#include "adapm/nvtx.h"

namespace py = pybind11;
using namespace adapm;

namespace adapm { namespace cudaops { void bind(py::module_& m); } }

namespace {

template <class T> T* ptr(uintptr_t a) { return reinterpret_cast<T*>(a); }

Options make_options(const std::map<std::string, std::string>& kv) {
  Options o;
  for (auto& p : kv) ADAPM_CHECK(o.set(p.first, p.second), "unknown option '" << p.first << "'");
  return o;
}

IoDesc make_io(bool on_device, uintptr_t stream, uintptr_t offsets = 0) {
  IoDesc io;
  io.on_device = on_device;
  io.has_stream = on_device;
  io.stream = reinterpret_cast<void*>(stream);
  io.offsets = reinterpret_cast<const int64_t*>(offsets);
  return io;
}

}  // namespace

PYBIND11_MODULE(_C, m) {
  m.doc() = "adapm_b200 native core";
  py::register_exception<adapm::Error>(m, "AdapmError", PyExc_RuntimeError);

  m.attr("LOCAL") = (int)LOCAL;
  m.attr("CLOCK_MAX") = (int64_t)CLOCK_MAX;
  m.attr("MAX_RANKS") = (int)MAX_RANKS;
  m.def("cuda_available", [] { return cudamem::available(); });
  m.def("_fdpass_selftest", [] { return fabric_fdpass_selftest(); });
  m.def("nvtx_compiled_in", [] { return nvtx_compiled_in(); });
  m.def("cuda_device_count", [] { return cudamem::available() ? cudamem::device_count() : 0; });
  m.def("poisson_quantile", &poisson_quantile);

  py::class_<KeyDistribution, std::shared_ptr<KeyDistribution>>(m, "KeyDistribution")
      .def_readonly("name", &KeyDistribution::name)
      .def_readonly("min_key", &KeyDistribution::min_key)
      .def_readonly("max_key", &KeyDistribution::max_key);
  m.def("uniform_distribution", &make_uniform_distribution);
  m.def("log_uniform_distribution", &make_log_uniform_distribution);
  m.def("alias_distribution", [](uintptr_t weights_f64, int64_t n, Key first, Key stride) {
    return make_alias_distribution(ptr<const double>(weights_f64), n, first, stride);
  });
  m.def("build_alias_table", [](uintptr_t weights_f64, int64_t n, uintptr_t prob_f32, uintptr_t alias_i32) {
    build_alias_table(ptr<const double>(weights_f64), n, ptr<float>(prob_f32), ptr<int32_t>(alias_i32));
  }, py::call_guard<py::gil_scoped_release>());
  m.def("callback_distribution", [](py::function fn, Key mn, Key mx) {
    auto f = std::make_shared<py::function>(std::move(fn));
    return make_callback_distribution([f]() { py::gil_scoped_acquire g; return (*f)().cast<Key>(); }, mn, mx);
  });

  py::class_<Server, std::shared_ptr<Server>>(m, "Server")
      .def(py::init([](const std::map<std::string, std::string>& opts, int64_t num_keys, uint32_t uniform_len,
                       uintptr_t lens_i64, int64_t n_lens) {
             Options o = make_options(opts);
             ValueSpec spec;
             spec.num_keys = num_keys;
             spec.uniform_len = uniform_len;
             if (n_lens > 0) {
               ADAPM_CHECK(n_lens == num_keys, "value_lengths has " << n_lens << " entries but num_keys is " << num_keys);
               const int64_t* l = ptr<const int64_t>(lens_i64);
               spec.lens.resize(n_lens);
               for (int64_t i = 0; i < n_lens; ++i) { ADAPM_CHECK(l[i] > 0, "value length must be positive"); spec.lens[i] = (uint32_t)l[i]; }
             }
             py::gil_scoped_release rel;
             return std::make_shared<Server>(o, spec);
           }),
           py::arg("options"), py::arg("num_keys"), py::arg("uniform_len"), py::arg("lens_ptr") = 0, py::arg("n_lens") = 0)
      .def("enable_sampling_support", &Server::enable_sampling_support, py::arg("distribution"), py::arg("scheme") = "",
           py::arg("with_replacement") = -1)
      .def("barrier", &Server::barrier, py::call_guard<py::gil_scoped_release>())
      .def("allreduce_sum", [](Server& s, std::vector<double> v) {
        { py::gil_scoped_release r; s.allreduce_sum(v.data(), (int)v.size()); }
        return v;
      })
      .def("shutdown", &Server::shutdown, py::call_guard<py::gil_scoped_release>())
      .def("my_rank", &Server::my_rank)
      .def("num_servers", &Server::num_servers)
      .def("num_workers", &Server::num_workers)
      .def("num_keys", &Server::num_keys)
      .def("get_len", &Server::get_len)
      .def("owner_of", &Server::owner_of)
      .def("home_of", &Server::home_of)
      .def("is_local", &Server::is_local)
      .def("counters", &Server::counters)
      .def("stats_string", &Server::stats_string)
      .def("reset_stats", &Server::reset_stats)
      .def("sync_rounds", [](Server& s) { return s.sync().rounds_done(); })
      .def("sync_report", [](Server& s) { return s.sync().report(); })
      .def("worker_clocks", &Server::worker_clocks)
      .def("is_cuda", [](Server& s) { return s.backend().is_cuda(); })
      .def("val_bytes", [](Server& s) { return s.backend().ctx().L.val_bytes; })
      .def("heap_bytes", [](Server& s) { return s.backend().ctx().L.heap_bytes; })
      .def("total_slots", [](Server& s) { return s.backend().ctx().L.total_slots; })
      .def("dtype", [](Server& s) { return s.options().dtype; })
      .def("device", [](Server& s) { return s.fabric().device(); })
      .def("peek", [](Server& s, const std::vector<Key>& keys) {
        std::vector<uint8_t> st(keys.size()), ow(keys.size());
        s.backend().peek_states(keys.data(), keys.size(), st.data(), ow.data());
        std::vector<std::pair<int, int>> out;
        for (size_t i = 0; i < keys.size(); ++i) out.emplace_back((int)st[i], (int)ow[i]);
        return out;
      })
      .def("peek_into", [](Server& s, uintptr_t keys, size_t n, uintptr_t states_u8, uintptr_t owners_u8) {
        s.backend().peek_states(ptr<const Key>(keys), n, ptr<uint8_t>(states_u8), ptr<uint8_t>(owners_u8));
      }, py::call_guard<py::gil_scoped_release>())
      .def("sampling_stats", [](Server& s) {
        std::map<std::string, uint64_t> m;
        if (s.sampling()) { m["checks"] = s.sampling()->local_checks(); m["pulls"] = s.sampling()->local_pulls(); }
        return m;
      })
      .def("slot_histogram", [](Server& s) {
        // debugging / tests: number of slots per state on this rank + free-stack fill per class
        const Layout& L = s.backend().ctx().L;
        std::vector<uint32_t> meta(L.total_slots);
        s.backend().read_heap(L.off_meta, meta.data(), meta.size() * 4);
        std::map<int, int64_t> h;
        for (uint32_t m : meta) h[(int)meta_state(m)]++;
        int32_t tops[MAX_CLASSES];
        s.backend().read_heap(L.off_free_top, tops, sizeof(tops));
        for (int c = 0; c < L.num_classes; ++c) h[100 + c] = tops[c];
        return h;
      })
      .def("backend_handle", [](Server& s) { return (uintptr_t)&s.backend(); })
      .def("trace_mark", [](Server& s, const std::string& name, uintptr_t stream) {
        // names are interned: the tracer keeps the pointer
        static std::mutex mu;
        static std::unordered_set<std::string> names;
        const char* p;
        { std::lock_guard<std::mutex> lk(mu); p = names.insert(name).first->c_str(); }
        s.backend().trace_mark(p, reinterpret_cast<void*>(stream));
      })
      .def("dump_trace", [](Server& s, const std::string& path) { s.backend().dump_trace(path); });

  py::class_<Worker, std::shared_ptr<Worker>>(m, "Worker")
      .def(py::init([](int customer_id, std::shared_ptr<Server> server) {
             return std::make_shared<Worker>(customer_id, *server);
           }),
           py::keep_alive<1, 3>())
      .def("pull", [](Worker& w, uintptr_t keys, size_t n, uintptr_t vals, bool on_device, uintptr_t stream, uintptr_t offsets) {
             return w.Pull(ptr<const Key>(keys), n, ptr<void>(vals), make_io(on_device, stream, offsets));
           }, py::arg("keys"), py::arg("n"), py::arg("vals"), py::arg("on_device"), py::arg("stream"), py::arg("offsets") = 0,
           py::call_guard<py::gil_scoped_release>())
      .def("push", [](Worker& w, uintptr_t keys, size_t n, uintptr_t vals, bool set, bool on_device, uintptr_t stream, uintptr_t offsets) {
             return w.Push(ptr<const Key>(keys), n, ptr<const void>(vals), set, make_io(on_device, stream, offsets));
           }, py::arg("keys"), py::arg("n"), py::arg("vals"), py::arg("set"), py::arg("on_device"), py::arg("stream"),
           py::arg("offsets") = 0, py::call_guard<py::gil_scoped_release>())
      .def("pull_if_local", [](Worker& w, Key key, uintptr_t vals) { return w.PullIfLocal(key, ptr<void>(vals)); },
           py::call_guard<py::gil_scoped_release>())
      .def("intent", [](Worker& w, uintptr_t keys, size_t n, Clock start, Clock end) {
             return w.Intent(ptr<const Key>(keys), n, start, end);
           }, py::call_guard<py::gil_scoped_release>())
      .def("intent_fast", [](Worker& w, uintptr_t keys, size_t n, Clock start, Clock end) {
             return w.IntentFast(ptr<const Key>(keys), n, start, end);
           }, py::call_guard<py::gil_scoped_release>())
      .def("handle", [](Worker& w) { return (uintptr_t)&w; })   // for native step drivers (ops.SgnsLoop)
      .def("advance_clock", &Worker::advanceClock)
      .def("current_clock", &Worker::currentClock)
      .def("prepare_sample", &Worker::PrepareSample, py::call_guard<py::gil_scoped_release>())
      .def("pull_sample", [](Worker& w, SampleID id, uintptr_t keys, size_t n, uintptr_t vals) {
             return w.PullSample(id, ptr<Key>(keys), n, ptr<void>(vals));
           }, py::call_guard<py::gil_scoped_release>())
      .def("finish_sample", &Worker::FinishSample)
      .def("wait", &Worker::Wait, py::call_guard<py::gil_scoped_release>())
      .def("is_finished", &Worker::IsFinished)
      .def("wait_all", &Worker::WaitAll, py::call_guard<py::gil_scoped_release>())
      .def("wait_sync", &Worker::WaitSync, py::call_guard<py::gil_scoped_release>())
      .def("barrier", &Worker::Barrier, py::call_guard<py::gil_scoped_release>())
      .def("begin_setup", &Worker::BeginSetup, py::call_guard<py::gil_scoped_release>())
      .def("end_setup", &Worker::EndSetup, py::call_guard<py::gil_scoped_release>())
      .def("reset_stats", &Worker::ResetStats)
      .def("finalize", &Worker::Finalize, py::call_guard<py::gil_scoped_release>())
      .def("get_len", &Worker::GetLen)
      .def("num_keys", &Worker::GetNumKeys)
      .def("total_len", [](Worker& w, uintptr_t keys, size_t n) { return w.total_len(ptr<const Key>(keys), n); })
      .def("id", &Worker::id)
      .def("worker_id", &Worker::worker_id)
      .def("locality", [](Worker& w) {
        std::map<std::string, uint64_t> m;
        m["pull_ops"] = w.num_pull_ops; m["pull_ops_local"] = w.num_pull_ops_local;
        m["push_ops"] = w.num_push_ops; m["push_ops_local"] = w.num_push_ops_local;
        m["pull_params"] = w.num_pull_params; m["pull_params_local"] = w.num_pull_params_local;
        m["push_params"] = w.num_push_params; m["push_params_local"] = w.num_push_params_local;
        return m;
      });

  // fast text parsers (io.h)
  m.def("read_triples", [](const std::string& path) {
    std::vector<int64_t> v;
    { py::gil_scoped_release r; v = read_triples_file(path); }
    py::array_t<int64_t> a({(py::ssize_t)(v.size() / 3), (py::ssize_t)3});
    if (!v.empty()) memcpy(a.mutable_data(), v.data(), v.size() * sizeof(int64_t));
    return a;
  });
  m.def("read_matrix_market_coo", [](const std::string& path) {
    CooMatrix c;
    { py::gil_scoped_release r; c = read_matrix_market_coo_file(path); }
    const py::ssize_t n = (py::ssize_t)c.x.size();
    py::array_t<int64_t> i(n), j(n);
    py::array_t<float> x(n);
    if (n) {
      memcpy(i.mutable_data(), c.i.data(), (size_t)n * 8);
      memcpy(j.mutable_data(), c.j.data(), (size_t)n * 8);
      memcpy(x.mutable_data(), c.x.data(), (size_t)n * 4);
    }
    return py::make_tuple(i, j, x, c.rows, c.cols);
  });
  m.def("read_edge_list", [](const std::string& path) {
    EdgeList g;
    { py::gil_scoped_release r; g = read_edge_list_file(path); }
    const py::ssize_t n = (py::ssize_t)g.src.size();
    py::array_t<int64_t> src(n), dst(n), ids((py::ssize_t)g.ids.size());
    if (n) {
      memcpy(src.mutable_data(), g.src.data(), (size_t)n * 8);
      memcpy(dst.mutable_data(), g.dst.data(), (size_t)n * 8);
    }
    if (!g.ids.empty()) memcpy(ids.mutable_data(), g.ids.data(), g.ids.size() * 8);
    py::object w = py::none();
    if (!g.weight.empty()) {
      py::array_t<double> wa(n);
      memcpy(wa.mutable_data(), g.weight.data(), (size_t)n * 8);
      w = wa;
    }
    return py::make_tuple(src, dst, w, ids);
  });

  m.attr("max_huffman_depth") = kMaxHuffmanDepth;
  m.def("huffman_tree", [](py::array_t<double, py::array::c_style | py::array::forcecast> counts) {
    HuffmanTree t;
    {
      const double* c = counts.data();
      const int64_t n = (int64_t)counts.size();
      py::gil_scoped_release r;
      t = huffman_tree(c, n);
    }
    py::array_t<int64_t> off((py::ssize_t)t.offsets.size());
    py::array_t<int32_t> nodes((py::ssize_t)t.nodes.size());
    py::array_t<uint32_t> codes((py::ssize_t)t.codes.size());
    memcpy(off.mutable_data(), t.offsets.data(), t.offsets.size() * sizeof(int64_t));
    if (!t.nodes.empty()) memcpy(nodes.mutable_data(), t.nodes.data(), t.nodes.size() * sizeof(int32_t));
    memcpy(codes.mutable_data(), t.codes.data(), t.codes.size() * sizeof(uint32_t));
    return py::make_tuple(off, nodes, codes, t.max_len);
  });

  // native data loader (corpus.h)
  py::class_<Corpus, std::shared_ptr<Corpus>>(m, "Corpus")
      .def_static("build", &Corpus::build, py::arg("path"), py::arg("min_count") = 5,
                  py::call_guard<py::gil_scoped_release>())
      .def_static("from_vocab", &Corpus::from_vocab)
      .def("encode", &Corpus::encode, py::arg("path"), py::arg("rank") = 0, py::arg("world") = 1,
           py::call_guard<py::gil_scoped_release>())
      .def("words", &Corpus::words)
      .def("counts", &Corpus::counts)
      .def("vocab_size", &Corpus::vocab_size)
      .def("num_tokens", &Corpus::num_tokens)
      .def("num_sentences", &Corpus::num_sentences)
      .def("lookup", &Corpus::lookup)
      .def("tokens_ptr", [](Corpus& c) { return (uintptr_t)c.tokens(); })
      .def("sentence_offsets_ptr", [](Corpus& c) { return (uintptr_t)c.sentence_offsets(); })
      .def("sentence_lines_ptr", [](Corpus& c) { return (uintptr_t)c.sentence_lines(); })
      .def("num_lines", &Corpus::num_lines);
  py::class_<PairStream, std::shared_ptr<PairStream>>(m, "PairStream")
      .def(py::init<std::shared_ptr<Corpus>, int, double, int64_t, uint64_t, int>(), py::arg("corpus"), py::arg("window"),
           py::arg("subsample"), py::arg("batch_pairs"), py::arg("seed"), py::arg("queue_depth") = 8)
      .def("start_epoch", &PairStream::start_epoch, py::call_guard<py::gil_scoped_release>())
      .def("next", [](PairStream& p, uintptr_t out) { return p.next(ptr<Key>(out)); },
           py::call_guard<py::gil_scoped_release>())
      .def("next_with_unique", [](PairStream& p, uintptr_t out, uintptr_t uniq) {
             int64_t n = 0;
             int64_t valid;
             { py::gil_scoped_release r; valid = p.next_with_unique(ptr<Key>(out), ptr<Key>(uniq), &n); }
             return py::make_tuple(valid, n);
           })
      .def("batch_pairs", &PairStream::batch_pairs)
      .def("pairs_produced", &PairStream::pairs_produced);
  py::class_<WindowStream, std::shared_ptr<WindowStream>>(m, "WindowStream")
      .def(py::init<std::shared_ptr<Corpus>, int, double, int64_t, uint64_t, int>(), py::arg("corpus"), py::arg("window"),
           py::arg("subsample"), py::arg("batch_windows"), py::arg("seed"), py::arg("queue_depth") = 8)
      .def("start_epoch", &WindowStream::start_epoch, py::call_guard<py::gil_scoped_release>())
      .def("next_with_unique", [](WindowStream& p, uintptr_t out, uintptr_t uniq) {
             int64_t n = 0;
             int64_t valid;
             { py::gil_scoped_release r; valid = p.next_with_unique(ptr<Key>(out), ptr<Key>(uniq), &n); }
             return py::make_tuple(valid, n);
           })
      .def("batch_windows", &WindowStream::batch_windows)
      .def("columns", &WindowStream::columns)
      .def("windows_produced", &WindowStream::windows_produced);
  m.attr("window_stream_max_window") = WindowStream::kMaxWindow;
  py::class_<DocPairStream, std::shared_ptr<DocPairStream>>(m, "DocPairStream")
      .def(py::init<std::shared_ptr<Corpus>, int, double, int64_t, uint64_t, bool, int>(), py::arg("corpus"),
           py::arg("window"), py::arg("subsample"), py::arg("batch_pairs"), py::arg("seed"), py::arg("dbow_words"),
           py::arg("queue_depth") = 8)
      .def("start_epoch", &DocPairStream::start_epoch, py::call_guard<py::gil_scoped_release>())
      .def("next_with_unique", [](DocPairStream& p, uintptr_t out, uintptr_t uniq) {
             int64_t n = 0;
             int64_t valid;
             { py::gil_scoped_release r; valid = p.next_with_unique(ptr<Key>(out), ptr<Key>(uniq), &n); }
             return py::make_tuple(valid, n);
           })
      .def("batch_pairs", &DocPairStream::batch_pairs);
  py::class_<DocWindowStream, std::shared_ptr<DocWindowStream>>(m, "DocWindowStream")
      .def(py::init<std::shared_ptr<Corpus>, int, double, int64_t, uint64_t, int>(), py::arg("corpus"),
           py::arg("window"), py::arg("subsample"), py::arg("batch_windows"), py::arg("seed"), py::arg("queue_depth") = 8)
      .def("start_epoch", &DocWindowStream::start_epoch, py::call_guard<py::gil_scoped_release>())
      .def("next_with_unique", [](DocWindowStream& p, uintptr_t out, uintptr_t uniq) {
             int64_t n = 0;
             int64_t valid;
             { py::gil_scoped_release r; valid = p.next_with_unique(ptr<Key>(out), ptr<Key>(uniq), &n); }
             return py::make_tuple(valid, n);
           })
      .def("batch_windows", &DocWindowStream::batch_windows)
      .def("columns", &DocWindowStream::columns);
  m.attr("doc_window_stream_max_window") = DocWindowStream::kMaxWindow;

  // host RPC (legacy SimpleApp capability, rpc.h)
  m.attr("kServerGroup") = (int)kServerGroup;
  m.attr("kWorkerGroup") = (int)kWorkerGroup;
  m.attr("kAllNodes") = (int)kAllNodes;
  py::class_<SimpleData>(m, "SimpleData")
      .def(py::init<>())
      .def_readwrite("head", &SimpleData::head)
      .def_property("body", [](const SimpleData& d) { return py::bytes(d.body); },
                    [](SimpleData& d, const std::string& b) { d.body = b; })
      .def_readwrite("sender", &SimpleData::sender)
      .def_readwrite("timestamp", &SimpleData::timestamp)
      .def_readwrite("customer_id", &SimpleData::customer_id);
  auto wrap_handle = [](py::function fn) {
    // the handle runs on the router thread: take the GIL there; the Python callable gets (SimpleData, app)
    auto f = std::shared_ptr<py::function>(new py::function(std::move(fn)), [](py::function* p) {
      py::gil_scoped_acquire g;
      delete p;
    });
    return SimpleApp::Handle([f](const SimpleData& d, SimpleApp* app) {
      py::gil_scoped_acquire g;
      try {
        (*f)(d, py::cast(app, py::return_value_policy::reference));
      } catch (py::error_already_set& e) {
        ALOG("[adapm] rpc handle raised: " << e.what());
      }
    });
  };
  py::class_<SimpleApp, std::shared_ptr<SimpleApp>>(m, "SimpleApp")
      .def(py::init([](int app_id, int customer_id, std::shared_ptr<Server> server, bool serves_requests) {
             return std::make_shared<SimpleApp>(app_id, customer_id, *server, serves_requests);
           }),
           py::keep_alive<1, 4>())
      .def("request", [](SimpleApp& a, int head, const std::string& body, int recv_id) {
             return a.Request(head, body, recv_id);
           }, py::call_guard<py::gil_scoped_release>())
      .def("response", [](SimpleApp& a, const SimpleData& req, const std::string& body) { a.Response(req, body); },
           py::arg("req"), py::arg("body") = std::string(), py::call_guard<py::gil_scoped_release>())
      .def("wait", &SimpleApp::Wait, py::call_guard<py::gil_scoped_release>())
      .def("num_response", &SimpleApp::NumResponse)
      .def("set_request_handle", [wrap_handle](SimpleApp& a, py::function fn) { a.set_request_handle(wrap_handle(std::move(fn))); })
      .def("set_response_handle", [wrap_handle](SimpleApp& a, py::function fn) { a.set_response_handle(wrap_handle(std::move(fn))); })
      .def_property_readonly("app_id", &SimpleApp::app_id)
      .def_property_readonly("customer_id", &SimpleApp::customer_id);

  adapm::cudaops::bind(m);
}
