// gc_pybind.cpp -- thin pybind11 module `medpy_b200._mgc` over the C ABI (include/medpy_b200_graphcut.h).
//
// It plays the role of the reference's Boost.Python module `medpy.graphcut.maxflow`
// (lib/maxflow/src/wrapper.cpp:59-89,125-134): one Python class owning one native graph.  Unlike the
// reference binding, whole arrays cross the boundary (numpy buffers or anything exposing
// __cuda_array_interface__, e.g. torch CUDA tensors) and the GIL is released around every native call.
// No arithmetic lives here.
#include <pybind11/numpy.h>
#include <pybind11/pybind11.h>
#include <pybind11/stl.h>

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstring>
#include <memory>
#include <stdexcept>
#include <thread>
#include <string>
#include <vector>

#if defined(__x86_64__)
#include <immintrin.h>
#endif

#include "../../include/medpy_b200_graphcut.h"
#include "host_pack.hpp"

namespace py = pybind11;

namespace {

void check(int rc, const mgc_graph* g)
{
    if (rc == MGC_OK) return;
    std::string msg = mgc_last_error(g);
    if (msg.empty()) msg = "medpy_b200 graph-cut error " + std::to_string(rc);
    if (rc == MGC_E_ARG || rc == MGC_E_WEIGHT) throw py::value_error(msg);
    throw std::runtime_error(msg);
}

int dtype_code(const std::string& kind_size)
{
    if (kind_size == "f4") return MGC_F32;
    if (kind_size == "f8") return MGC_F64;
    if (kind_size == "u1" || kind_size == "b1") return MGC_U8;
    if (kind_size == "i2") return MGC_I16;
    if (kind_size == "i4") return MGC_I32;
    return -1;
}

// Holds the mgc_array plus whatever keeps the memory alive for the duration of the call.
struct ArrayRef {
    mgc_array a{};
    py::object keep;
    std::vector<int64_t> shape;
};

ArrayRef make_ref(const py::object& obj, int want_dtype /* -1 any */, const char* what)
{
    ArrayRef r;
    if (py::hasattr(obj, "__cuda_array_interface__")) {
        py::dict d = obj.attr("__cuda_array_interface__");
        py::tuple data = d["data"];
        r.a.data = reinterpret_cast<const void*>(data[0].cast<uintptr_t>());
        r.a.mem = MGC_MEM_DEVICE;
        std::string ts = d["typestr"].cast<std::string>();  // e.g. "<f4", "|u1", "|b1"
        r.a.dtype = dtype_code(ts.substr(1));
        py::tuple shp = d["shape"];
        for (auto s : shp) r.shape.push_back(s.cast<int64_t>());
        size_t es = (size_t)std::stoi(ts.substr(2));
        if (d.contains("strides") && !d["strides"].is_none()) {
            py::tuple st = d["strides"];
            for (size_t i = 0; i < st.size() && i < MGC_MAX_NDIM; ++i) r.a.strides[i] = st[i].cast<int64_t>();
        } else {
            int64_t acc = (int64_t)es;
            for (int i = (int)r.shape.size() - 1; i >= 0; --i) { if (i < MGC_MAX_NDIM) r.a.strides[i] = acc; acc *= r.shape[i]; }
        }
        r.keep = obj;
    } else {
        py::array arr = py::array::ensure(obj);
        if (!arr) throw py::value_error(std::string(what) + ": expected an array");
        std::string ks(1, arr.dtype().kind());
        ks += std::to_string(arr.dtype().itemsize());
        r.a.dtype = dtype_code(ks);
        r.a.data = arr.data();
        r.a.mem = MGC_MEM_HOST;
        for (py::ssize_t i = 0; i < arr.ndim(); ++i) {
            r.shape.push_back(arr.shape(i));
            if (i < MGC_MAX_NDIM) r.a.strides[i] = arr.strides(i);
        }
        r.keep = arr;
    }
    if (r.a.dtype < 0) throw py::value_error(std::string(what) + ": unsupported dtype");
    if (want_dtype >= 0 && r.a.dtype != want_dtype) throw py::value_error(std::string(what) + ": wrong dtype");
    return r;
}

class PyGraph {
public:
    PyGraph(const std::vector<int64_t>& shape, int device) : shape_(shape)
    {
        int rc = mgc_create((int32_t)shape.size(), shape.data(), device, &g_);
        if (rc != MGC_OK) { std::string m = mgc_last_error(nullptr); if (rc == MGC_E_ARG) throw py::value_error(m); throw std::runtime_error(m); }
    }
    PyGraph(const std::vector<int64_t>& shape, int64_t z0, int64_t z1, int device) : shape_(shape)
    {
        int rc = mgc_create_slab((int32_t)shape.size(), shape.data(), z0, z1, device, &g_);
        if (rc != MGC_OK) { std::string m = mgc_last_error(nullptr); if (rc == MGC_E_ARG) throw py::value_error(m); throw std::runtime_error(m); }
        shape_[0] = (z1 - z0) + (z0 > 0 ? 1 : 0) + (z1 < shape[0] ? 1 : 0);  // local extent incl. ghost planes
        owned_planes_ = z1 - z0;
    }
    // a batch of `batch` images of shape image_shape (mgc_create_batch): the graph's arrays are (batch, ...image)
    struct BatchTag {};
    PyGraph(BatchTag, const std::vector<int64_t>& image_shape, int64_t batch, int device) : shape_(image_shape)
    {
        int rc = mgc_create_batch((int32_t)image_shape.size(), image_shape.data(), batch, device, &g_);
        if (rc != MGC_OK) { std::string m = mgc_last_error(nullptr); if (rc == MGC_E_ARG) throw py::value_error(m); throw std::runtime_error(m); }
        shape_.insert(shape_.begin(), batch);
    }
    static std::unique_ptr<PyGraph> batch(const std::vector<int64_t>& image_shape, int64_t batch, int device)
    {
        return std::unique_ptr<PyGraph>(new PyGraph(BatchTag{}, image_shape, batch, device));
    }
    ~PyGraph() { if (g_) mgc_destroy(g_); }
    PyGraph(const PyGraph&) = delete;
    PyGraph& operator=(const PyGraph&) = delete;

    void check_shape(const ArrayRef& r, const char* what) const
    {
        if (r.shape != shape_) throw py::value_error(std::string(what) + ": shape does not match the graph's lattice");
    }

    void add_regional_probability(const py::object& prob, double alpha, bool compute_f32)
    {
        ArrayRef r = make_ref(prob, -1, "probability_map");
        check_shape(r, "probability_map");
        check_inputs();
        int rc;
        { py::gil_scoped_release rel; rc = mgc_add_regional_probability(g_, &r.a, alpha, compute_f32 ? MGC_F32 : MGC_F64); }
        check(rc, g_);
        held_live_ = false;
    }
    void add_tweights_dense(const py::object& src, const py::object& snk)
    {
        ArrayRef a = make_ref(src, MGC_F64, "src"), b = make_ref(snk, MGC_F64, "snk");
        check_shape(a, "src"); check_shape(b, "snk");
        check_inputs();
        int rc;
        { py::gil_scoped_release rel; rc = mgc_add_tweights_dense(g_, &a.a, &b.a); }
        check(rc, g_);
        held_live_ = false;
    }
    void add_markers(const py::object& fg, const py::object& bg)
    {
        ArrayRef a, b;
        bool hf = !fg.is_none(), hb = !bg.is_none();
        if (hf) { a = make_ref(fg, MGC_U8, "fg_markers"); check_shape(a, "fg_markers"); }
        if (hb) { b = make_ref(bg, MGC_U8, "bg_markers"); check_shape(b, "bg_markers"); }
        check_inputs();
        int rc;
        { py::gil_scoped_release rel; rc = mgc_add_markers(g_, hf ? &a.a : nullptr, hb ? &b.a : nullptr); }
        check(rc, g_);
        held_live_ = false;
    }
    void add_boundary(int kind, const py::object& image, double sigma, const py::object& spacing, double norm)
    {
        ArrayRef r = make_ref(image, -1, "image");
        check_shape(r, "image");
        std::vector<double> sp;
        if (!spacing.is_none()) {
            sp = spacing.cast<std::vector<double>>();
            if (sp.size() < shape_.size()) throw py::value_error("spacing has fewer entries than the image has dimensions");
        }
        check_inputs();
        int rc;
        { py::gil_scoped_release rel; rc = mgc_add_boundary(g_, kind, &r.a, sigma, sp.empty() ? nullptr : sp.data(), norm); }
        check(rc, g_);
        held_live_ = false;
    }
    // everything graph_from_voxels adds, in one native call (mgc_build_voxel_graph); None = term absent, kind -1 = no boundary
    void build_voxel_graph(const py::object& prob, double alpha, bool compute_f32, int kind, const py::object& image, double sigma,
                           const py::object& spacing, double norm, const py::object& fg, const py::object& bg)
    {
        ArrayRef rp, ri, rf, rb;
        mgc_voxel_terms t{};
        t.alpha = alpha;
        t.compute_dtype = compute_f32 ? MGC_F32 : MGC_F64;
        t.boundary_kind = kind;
        t.sigma = sigma;
        t.norm = norm;
        if (!prob.is_none()) { rp = make_ref(prob, -1, "probability_map"); check_shape(rp, "probability_map"); t.prob = &rp.a; }
        if (!image.is_none()) { ri = make_ref(image, -1, "image"); check_shape(ri, "image"); t.image = &ri.a; }
        if (!fg.is_none()) { rf = make_ref(fg, MGC_U8, "fg_markers"); check_shape(rf, "fg_markers"); t.fg = &rf.a; }
        if (!bg.is_none()) { rb = make_ref(bg, MGC_U8, "bg_markers"); check_shape(rb, "bg_markers"); t.bg = &rb.a; }
        std::vector<double> sp;
        if (!spacing.is_none()) {
            sp = spacing.cast<std::vector<double>>();
            if (sp.size() < shape_.size()) throw py::value_error("spacing has fewer entries than the image has dimensions");
            t.spacing = sp.data();
        }
        // large host marker volumes cross PCIe bit-packed (packed on worker threads while the image is already uploading)
        std::unique_ptr<MarkerPacker> packer;
        void* bits[2] = {nullptr, nullptr};
        size_t n = 1;
        for (auto d : shape_) n *= (size_t)d;
        auto dense_host = [&](const ArrayRef& r) {
            if (r.a.mem != MGC_MEM_HOST) return false;
            int64_t expect = 1;
            for (int i = (int)r.shape.size() - 1; i >= 0; --i) { if (r.shape[i] > 1 && r.a.strides[i] != expect) return false; expect *= r.shape[i]; }
            return true;
        };
        const bool pack = pack_markers_ && n >= ((size_t)1 << 22) && mgc_can_fuse(g_) && kind >= 0 && (t.fg || t.bg) &&
                          (!t.fg || dense_host(rf)) && (!t.bg || dense_host(rb));
        if (pack) {
            const size_t words = (n + 31) / 32;
            for (int p = 0; p < 2; ++p)
                if ((p == 0 ? t.fg : t.bg) && mgc_host_alloc(words * 4, &bits[p]) != MGC_OK) throw std::runtime_error("pinned host allocation failed");
            packer.reset(new MarkerPacker(t.fg ? (const uint8_t*)rf.a.data : nullptr, t.bg ? (const uint8_t*)rb.a.data : nullptr,
                                          (uint32_t*)bits[0], (uint32_t*)bits[1], n));
            t.fg = nullptr; t.bg = nullptr;
            t.fg_bits = (const uint32_t*)bits[0]; t.bg_bits = (const uint32_t*)bits[1];
            t.bits_mem = MGC_MEM_HOST;
            t.bits_ready_words = reinterpret_cast<const volatile int64_t*>(&packer->ready);
        }
        // device image and map: the lazy build reads them in place until the next build or reset (no copy), so they stay
        // referenced here for as long as the handle may read them
        std::vector<Held> hold;
        if (keep_inputs_)
            for (const ArrayRef* r : {&ri, &rp})
                if (r->keep && r->a.mem == MGC_MEM_DEVICE) hold.push_back(Held{r->keep, version_of(r->keep)});
        check(mgc_set_option(g_, MGC_OPT_KEEP_DEVICE_INPUTS, hold.empty() ? 0 : 1), g_);
        int rc;
        { py::gil_scoped_release rel; rc = mgc_build_voxel_graph(g_, &t); packer.reset(); }
        for (int p = 0; p < 2; ++p) if (bits[p]) mgc_host_free(bits[p]);
        if (rc != MGC_OK) {
            // the handle may still read what it held before this call, and queued work may read the new arrays
            held_.insert(held_.end(), hold.begin(), hold.end());
            check(rc, g_);
        }
        hold_inputs(std::move(hold));
        held_live_ = !held_.empty() && kind >= 0 && mgc_can_fuse(g_);
    }
    // mgc_build_voxel_batch: arrays over (batch, ...image); sigmas / norms one per image (norm NaN: reduced on the device)
    void build_voxel_batch(const py::object& prob, double alpha, bool compute_f32, int kind, const py::object& image,
                           const std::vector<double>& sigmas, const py::object& spacing, const std::vector<double>& norms,
                           const py::object& fg, const py::object& bg)
    {
        if ((int64_t)sigmas.size() != shape_[0] || (int64_t)norms.size() != shape_[0])
            throw py::value_error("sigmas and norms need one entry per image");
        ArrayRef rp, ri, rf, rb;
        mgc_voxel_terms t{};
        t.alpha = alpha;
        t.compute_dtype = compute_f32 ? MGC_F32 : MGC_F64;
        t.boundary_kind = kind;
        ri = make_ref(image, -1, "image"); check_shape(ri, "image"); t.image = &ri.a;
        if (!prob.is_none()) { rp = make_ref(prob, -1, "probability_map"); check_shape(rp, "probability_map"); t.prob = &rp.a; }
        if (!fg.is_none()) { rf = make_ref(fg, MGC_U8, "fg_markers"); check_shape(rf, "fg_markers"); t.fg = &rf.a; }
        if (!bg.is_none()) { rb = make_ref(bg, MGC_U8, "bg_markers"); check_shape(rb, "bg_markers"); t.bg = &rb.a; }
        std::vector<double> sp;
        if (!spacing.is_none()) {
            sp = spacing.cast<std::vector<double>>();
            if (sp.size() + 1 < shape_.size()) throw py::value_error("spacing has fewer entries than the images have dimensions");
            t.spacing = sp.data();
        }
        int rc;
        { py::gil_scoped_release rel; rc = mgc_build_voxel_batch(g_, &t, sigmas.data(), norms.data()); }
        check(rc, g_);
    }
    py::array_t<double> get_batch_energies()
    {
        py::array_t<double> out((py::ssize_t)shape_[0]);
        int rc;
        { py::gil_scoped_release rel; rc = mgc_get_batch_energies(g_, out.mutable_data()); }
        check(rc, g_);
        return out;
    }
    void set_pack_markers(bool on) { pack_markers_ = on; }
    // off: device inputs are borrowed for the build call only and the build keeps its own copies (the C default)
    void set_keep_device_inputs(bool on) { keep_inputs_ = on; }
    bool can_fuse() const { return mgc_can_fuse(g_) != 0; }
    void add_nweights_dense(int axis, const py::object& fwd, const py::object& bwd)
    {
        ArrayRef a = make_ref(fwd, MGC_F64, "fwd"), b = make_ref(bwd, MGC_F64, "bwd");
        check_shape(a, "fwd"); check_shape(b, "bwd");
        check_inputs();
        int rc;
        { py::gil_scoped_release rel; rc = mgc_add_nweights_dense(g_, axis, &a.a, &b.a); }
        check(rc, g_);
        held_live_ = false;
    }
    // contiguous 1-D array on the host (numpy, converted to T) or on the device (__cuda_array_interface__ of typestr `ts`,
    // read in place); None = absent
    struct Vec { const void* p = nullptr; int64_t n = 0; int mem = -1; py::object keep; };
    template <typename T>
    static Vec vec_of(const py::object& o, const char* ts, const char* what)
    {
        Vec r;
        if (o.is_none()) return r;
        const std::string bad = std::string(what) + ": expected a 1-D " + (ts[0] == 'i' ? "int64" : "float64") + " array";
        if (py::hasattr(o, "__cuda_array_interface__")) {
            py::dict d = o.attr("__cuda_array_interface__");
            py::tuple shp = d["shape"];
            if (shp.size() != 1 || d["typestr"].cast<std::string>().substr(1) != ts) throw py::value_error(bad);
            if (d.contains("strides") && !d["strides"].is_none()) {
                py::tuple st = d["strides"];
                if (st[0].cast<int64_t>() != 8) throw py::value_error(std::string(what) + ": array must be contiguous");
            }
            r.p = reinterpret_cast<const void*>(py::tuple(d["data"])[0].cast<uintptr_t>());
            r.n = shp[0].cast<int64_t>();
            r.mem = MGC_MEM_DEVICE;
            r.keep = o;
        } else {
            auto a = py::array_t<T, py::array::c_style | py::array::forcecast>::ensure(o);
            if (!a || a.ndim() != 1) throw py::value_error(bad);
            r.p = a.data();
            r.n = a.shape(0);
            r.mem = MGC_MEM_HOST;
            r.keep = a;
        }
        return r;
    }
    // seeds folded into the solved graph (mgc_add_seeds / mgc_remove_seeds): 1-D int64 node-id arrays, both on the host
    // (numpy) or both on the device (__cuda_array_interface__); None = no seeds of that kind
    void add_seeds(const py::object& fg, const py::object& bg) { fold_seeds(fg, bg, mgc_add_seeds); }
    void remove_seeds(const py::object& fg, const py::object& bg) { fold_seeds(fg, bg, mgc_remove_seeds); }
    void fold_seeds(const py::object& fg, const py::object& bg,
                    int (*fold)(mgc_graph*, const int64_t*, int64_t, const int64_t*, int64_t, int32_t))
    {
        Vec f = vec_of<int64_t>(fg, "i8", "fg_ids"), b = vec_of<int64_t>(bg, "i8", "bg_ids");
        if (f.n && b.n && f.mem != b.mem) throw py::value_error("fg_ids and bg_ids must both be host or both be device arrays");
        const int mem = f.n ? f.mem : (b.n ? b.mem : MGC_MEM_HOST);
        check_inputs();
        int rc;
        { py::gil_scoped_release rel; rc = fold(g_, f.n ? (const int64_t*)f.p : nullptr, f.n, b.n ? (const int64_t*)b.p : nullptr, b.n, mem); }
        check(rc, g_);
    }
    // add_tweights calls folded into the solved graph (mgc_add_tweights_warm): ids = 1-D int64 node ids (None: the dense
    // form, one call per voxel in C order), src / snk = 1-D float64 of the same length; all three on the host or all on
    // the device
    void add_tweights_warm(const py::object& ids, const py::object& src, const py::object& snk)
    {
        Vec i = vec_of<int64_t>(ids, "i8", "ids"), s = vec_of<double>(src, "f8", "src"), t = vec_of<double>(snk, "f8", "snk");
        if (s.mem < 0 || t.mem < 0) throw py::value_error("src and snk are required");
        if (s.n != t.n || (!ids.is_none() && i.n != s.n)) throw py::value_error("ids, src and snk differ in length");
        if (s.mem != t.mem || (!ids.is_none() && i.mem != s.mem))
            throw py::value_error("ids, src and snk must all be host or all be device arrays");
        check_inputs();
        int rc;
        {
            py::gil_scoped_release rel;
            rc = mgc_add_tweights_warm(g_, ids.is_none() ? nullptr : (const int64_t*)i.p, (const double*)s.p,
                                       (const double*)t.p, s.n, s.mem);
        }
        check(rc, g_);
    }
    // sum_edge calls folded into the solved graph (mgc_add_nweights_warm): i / j = 1-D int64 node ids, cap / rev = 1-D
    // float64 of the same length, all four on the host or all on the device
    void add_nweights_warm(const py::object& i, const py::object& j, const py::object& cap, const py::object& rev)
    {
        fold_nweights(i, j, cap, rev, mgc_add_nweights_warm);
    }
    // the same with the decrements of mgc_remove_nweights_warm
    void remove_nweights_warm(const py::object& i, const py::object& j, const py::object& cap, const py::object& rev)
    {
        fold_nweights(i, j, cap, rev, mgc_remove_nweights_warm);
    }
    void fold_nweights(const py::object& i, const py::object& j, const py::object& cap, const py::object& rev,
                       int (*fold)(mgc_graph*, const int64_t*, const int64_t*, const double*, const double*, int64_t, int32_t))
    {
        Vec a = vec_of<int64_t>(i, "i8", "i"), b = vec_of<int64_t>(j, "i8", "j");
        Vec c = vec_of<double>(cap, "f8", "cap"), r = vec_of<double>(rev, "f8", "rev_cap");
        if (a.mem < 0 || b.mem < 0 || c.mem < 0 || r.mem < 0) throw py::value_error("i, j, cap and rev_cap are required");
        if (a.n != b.n || a.n != c.n || a.n != r.n) throw py::value_error("i, j, cap and rev_cap differ in length");
        if (a.mem != b.mem || a.mem != c.mem || a.mem != r.mem)
            throw py::value_error("i, j, cap and rev_cap must all be host or all be device arrays");
        check_inputs();
        int rc;
        {
            py::gil_scoped_release rel;
            rc = fold(g_, (const int64_t*)a.p, (const int64_t*)b.p, (const double*)c.p, (const double*)r.p, a.n, a.mem);
        }
        check(rc, g_);
    }
    // the dense forms (mgc_add_nweights_dense_warm / mgc_remove_nweights_dense_warm): fwd / bwd float64 arrays of the
    // lattice shape
    void add_nweights_dense_warm(int axis, const py::object& fwd, const py::object& bwd)
    {
        fold_nweights_dense(axis, fwd, bwd, mgc_add_nweights_dense_warm);
    }
    void remove_nweights_dense_warm(int axis, const py::object& fwd, const py::object& bwd)
    {
        fold_nweights_dense(axis, fwd, bwd, mgc_remove_nweights_dense_warm);
    }
    void fold_nweights_dense(int axis, const py::object& fwd, const py::object& bwd,
                             int (*fold)(mgc_graph*, int32_t, const mgc_array*, const mgc_array*))
    {
        ArrayRef a = make_ref(fwd, MGC_F64, "fwd"), b = make_ref(bwd, MGC_F64, "bwd");
        check_shape(a, "fwd"); check_shape(b, "bwd");
        check_inputs();
        int rc;
        { py::gil_scoped_release rel; rc = fold(g_, axis, &a.a, &b.a); }
        check(rc, g_);
    }
    double maxflow()
    {
        check_inputs();
        double e = 0;
        int rc;
        { py::gil_scoped_release rel; rc = mgc_maxflow(g_, &e); }
        check(rc, g_);
        return e;
    }
    py::array_t<uint8_t> get_mask()
    {
        std::vector<py::ssize_t> shp(shape_.begin(), shape_.end());
        if (owned_planes_ >= 0) shp[0] = owned_planes_;
        size_t n = 1;
        for (auto d : shp) n *= (size_t)d;
        // pinned, pooled destination: the numpy array owns it through a capsule that returns it to the pool
        void* mem = nullptr;
        if (mgc_host_alloc(n ? n : 1, &mem) != MGC_OK) throw std::runtime_error("pinned host allocation failed");
        py::capsule owner(mem, [](void* p) { mgc_host_free(p); });
        int rc;
        { py::gil_scoped_release rel; rc = mgc_get_mask(g_, (uint8_t*)mem, MGC_MEM_HOST); }
        check(rc, g_);
        return py::array_t<uint8_t>(shp, (const uint8_t*)mem, owner);
    }
    void get_mask_into(uintptr_t device_ptr)
    {
        int rc;
        { py::gil_scoped_release rel; rc = mgc_get_mask(g_, reinterpret_cast<uint8_t*>(device_ptr), MGC_MEM_DEVICE); }
        check(rc, g_);
    }
    int what_segment(int64_t i) { int32_t s = 0; check(mgc_what_segment(g_, i, &s), g_); return s; }
    double get_edge(int64_t i, int64_t j) { check_inputs(); double c = 0; check(mgc_get_edge(g_, i, j, &c), g_); return c; }
    double get_trcap(int64_t i) { check_inputs(); double c = 0; check(mgc_get_trcap(g_, i, &c), g_); return c; }
    int64_t get_node_num() { int64_t n = 0; check(mgc_get_node_num(g_, &n), g_); return n; }
    int64_t get_arc_num() { int64_t n = 0; check(mgc_get_arc_num(g_, &n), g_); return n; }
    // the handle forgets the build's inputs; their references go at the next build, once its stream is done with them
    void reset() { check(mgc_reset(g_), g_); held_live_ = false; }
    void set_option(int option, long long value) { check(mgc_set_option(g_, option, value), g_); }
    void check_deferred() { int rc; { py::gil_scoped_release rel; rc = mgc_check(g_); } check(rc, g_); }
    void set_stream(uintptr_t s) { check(mgc_set_stream(g_, reinterpret_cast<void*>(s)), g_); }
    void synchronize() { int rc; { py::gil_scoped_release rel; rc = mgc_synchronize(g_); } check(rc, g_); }
    py::dict stats()
    {
        mgc_stats s{};
        check(mgc_get_stats(g_, &s), g_);
        py::dict d;
        d["n_voxels"] = s.n_voxels; d["push_sweeps"] = s.push_sweeps; d["global_relabels"] = s.global_relabels;
        d["relabel_sweeps"] = s.relabel_sweeps; d["kernel_launches"] = s.kernel_launches; d["active_last"] = s.active_last;
        d["ms_terms"] = s.ms_terms; d["ms_solve"] = s.ms_solve; d["ms_readout"] = s.ms_readout;
        d["ms_push"] = s.ms_push; d["ms_relabel"] = s.ms_relabel; d["ms_boundary"] = s.ms_boundary; d["ms_init"] = s.ms_init;
        d["flow_const"] = s.flow_const; d["energy"] = s.energy; d["device_bytes"] = s.device_bytes;
        d["tiles_materialised"] = s.tiles_materialised; d["ms_caps"] = s.ms_caps;
        d["seed_folds"] = s.seed_folds; d["ms_seeds"] = s.ms_seeds; d["ms_seeds_host"] = s.ms_seeds_host;
        d["tiles_deferred"] = s.tiles_deferred; d["tiles_dropped"] = s.tiles_dropped;
        d["relabel_passes"] = s.relabel_passes; d["ms_relabel_first"] = s.ms_relabel_first;
        d["relabel_passes_first"] = s.relabel_passes_first;
        d["build_blocks_refused"] = s.build_blocks_refused;
        return d;
    }
    // ---- z-slab stepping (device pointers as integers, e.g. torch.Tensor.data_ptr()) ----
    int64_t slab_plane_elems() { int64_t n = 0; check(mgc_slab_plane_elems(g_, &n), g_); return n; }
    void slab_begin() { int rc; { py::gil_scoped_release rel; rc = mgc_slab_begin(g_); } check(rc, g_); }
    void slab_push(int n) { int rc; { py::gil_scoped_release rel; rc = mgc_slab_push(g_, n); } check(rc, g_); }
    void slab_pack(uintptr_t hlo, uintptr_t flo, uintptr_t hhi, uintptr_t fhi)
    {
        int rc;
        { py::gil_scoped_release rel; rc = mgc_slab_pack(g_, (int32_t*)hlo, (double*)flo, (int32_t*)hhi, (double*)fhi); }
        check(rc, g_);
    }
    void slab_unpack(uintptr_t hlo, uintptr_t flo, uintptr_t hhi, uintptr_t fhi, uintptr_t changed_dev)
    {
        int rc;
        { py::gil_scoped_release rel; rc = mgc_slab_unpack(g_, (const int32_t*)hlo, (const double*)flo, (const int32_t*)hhi, (const double*)fhi, (int32_t*)changed_dev); }
        check(rc, g_);
    }
    void slab_count_active_dev(uintptr_t count_dev)
    {
        int rc;
        { py::gil_scoped_release rel; rc = mgc_slab_count_active_dev(g_, (unsigned long long*)count_dev); }
        check(rc, g_);
    }
    void slab_relabel_begin() { int rc; { py::gil_scoped_release rel; rc = mgc_slab_relabel_begin(g_); } check(rc, g_); }
    int slab_relabel_relax(bool want_changed)
    {
        int32_t c = 0;
        int rc;
        { py::gil_scoped_release rel; rc = mgc_slab_relabel_relax(g_, want_changed ? &c : nullptr); }
        check(rc, g_);
        return c;
    }
    int64_t slab_count_active() { int64_t a = 0; int rc; { py::gil_scoped_release rel; rc = mgc_slab_count_active(g_, &a); } check(rc, g_); return a; }
    double slab_finish() { double e = 0; int rc; { py::gil_scoped_release rel; rc = mgc_slab_finish(g_, &e); } check(rc, g_); return e; }

    // ---- native distributed solve (NCCL inside the library) ----
    static py::bytes slab_comm_unique_id()
    {
        char id[128];
        int rc = mgc_slab_comm_unique_id(id);
        if (rc != MGC_OK) throw std::runtime_error(mgc_last_error(nullptr));
        return py::bytes(id, 128);
    }
    void slab_comm_init(int rank, int world, const py::bytes& id)
    {
        std::string s = id;
        if (s.size() != 128) throw py::value_error("the NCCL unique id has 128 bytes");
        int rc;
        { py::gil_scoped_release rel; rc = mgc_slab_comm_init(g_, rank, world, s.data()); }
        check(rc, g_);
    }
    double slab_solve()
    {
        double e = 0;
        int rc;
        { py::gil_scoped_release rel; rc = mgc_slab_solve(g_, &e); }
        check(rc, g_);
        return e;
    }
    py::dict slab_solve_stats()
    {
        int64_t a = 0, b = 0, c = 0, d = 0;
        check(mgc_slab_solve_stats(g_, &a, &b, &c, &d), g_);
        py::dict out;
        out["exchanges"] = a; out["relabel_rounds"] = b; out["push_passes"] = c; out["global_relabels"] = d;
        double ph[6] = {0, 0, 0, 0, 0, 0};
        check(mgc_slab_solve_phase_ms(g_, ph), g_);
        py::dict phase;
        phase["local_bfs_ms"] = ph[0]; phase["exchange_ms"] = ph[1]; phase["stop_test_ms"] = ph[2]; phase["push_ms"] = ph[3];
        phase["readout_ms"] = ph[4]; phase["host_blocked_ms"] = ph[5];
        out["phase_ms"] = phase;
        return out;
    }

    std::vector<int64_t> shape() const { return shape_; }

private:
    // a device array the last build may still read, and its torch version counter at the build (-1: not a tensor)
    struct Held { py::object obj; int64_t version; };
    static int64_t version_of(const py::object& o)
    {
        return py::hasattr(o, "_version") ? o.attr("_version").cast<int64_t>() : -1;
    }
    // take the arrays of a new build; the ones it replaces are dropped only after the handle's stream is done with them
    // (the caching allocator may hand their memory out again at once).  The same arrays again (a resident loop) cost
    // no synchronisation.
    void hold_inputs(std::vector<Held> hold)
    {
        bool same = hold.size() == held_.size();
        for (size_t i = 0; same && i < hold.size(); ++i) same = hold[i].obj.is(held_[i].obj);
        if (!same && !held_.empty()) {
            int rc;
            { py::gil_scoped_release rel; rc = mgc_synchronize(g_); }
            check(rc, g_);
        }
        held_ = std::move(hold);
    }
    // before a call that may read the inputs of the last build: an array changed in place since would give another graph
    void check_inputs() const
    {
        if (!held_live_) return;
        for (const Held& h : held_)
            if (h.version >= 0 && version_of(h.obj) != h.version)
                throw std::runtime_error("an image or probability map passed to the graph build was modified in place after "
                                         "the build; rebuild the graph");
    }

    mgc_graph* g_ = nullptr;
    std::vector<int64_t> shape_;
    int64_t owned_planes_ = -1;
    std::vector<Held> held_;
    bool held_live_ = false;           // the handle may read held_ (until reset or a per-term call)
    bool keep_inputs_ = true;
    bool pack_markers_ = std::getenv("MEDPY_GC_PACK_MARKERS") ? std::atoi(std::getenv("MEDPY_GC_PACK_MARKERS")) != 0 : true;
};

// ---- general sparse graph (mgc_sparse_*) ------------------------------------------------------------------------
void check_sparse(int rc, const mgc_sparse* g)
{
    if (rc == MGC_OK) return;
    std::string msg = mgc_sparse_last_error(g);
    if (msg.empty()) msg = "medpy_b200 sparse graph error " + std::to_string(rc);
    if (rc == MGC_E_ARG || rc == MGC_E_WEIGHT) throw py::value_error(msg);
    throw std::runtime_error(msg);
}

class PySparse {
public:
    PySparse(int64_t n, int device)
    {
        int rc = mgc_sparse_create(n, device, &g_);
        if (rc != MGC_OK) { std::string m = mgc_sparse_last_error(nullptr); if (rc == MGC_E_ARG) throw py::value_error(m); throw std::runtime_error(m); }
    }
    ~PySparse() { if (g_) mgc_sparse_destroy(g_); }
    PySparse(const PySparse&) = delete;
    PySparse& operator=(const PySparse&) = delete;

    void sum_edges(py::array_t<int32_t, py::array::c_style | py::array::forcecast> i,
                   py::array_t<int32_t, py::array::c_style | py::array::forcecast> j,
                   py::array_t<double, py::array::c_style | py::array::forcecast> cap,
                   py::array_t<double, py::array::c_style | py::array::forcecast> rev)
    {
        const py::ssize_t m = i.size();
        if (j.size() != m || cap.size() != m || rev.size() != m) throw py::value_error("edge arrays differ in length");
        int rc;
        { py::gil_scoped_release rel; rc = mgc_sparse_sum_edges(g_, (int64_t)m, i.data(), j.data(), cap.data(), rev.data()); }
        check_sparse(rc, g_);
    }
    void remove_edges_warm(py::array_t<int32_t, py::array::c_style | py::array::forcecast> i,
                           py::array_t<int32_t, py::array::c_style | py::array::forcecast> j,
                           py::array_t<double, py::array::c_style | py::array::forcecast> cap,
                           py::array_t<double, py::array::c_style | py::array::forcecast> rev)
    {
        const py::ssize_t m = i.size();
        if (j.size() != m || cap.size() != m || rev.size() != m) throw py::value_error("edge arrays differ in length");
        int rc;
        { py::gil_scoped_release rel; rc = mgc_sparse_remove_edges_warm(g_, (int64_t)m, i.data(), j.data(), cap.data(), rev.data()); }
        check_sparse(rc, g_);
    }
    void set_option(int32_t option, int64_t value) { check_sparse(mgc_sparse_set_option(g_, option, value), g_); }
    py::array_t<double> segment_energies(py::array_t<int64_t, py::array::c_style | py::array::forcecast> node_off)
    {
        const py::ssize_t b = node_off.size() - 1;
        if (b < 1) throw py::value_error("node offsets of at least one range expected");
        py::array_t<double> out(b);
        int rc;
        { double* p = out.mutable_data(); const int64_t* o = node_off.data(); py::gil_scoped_release rel; rc = mgc_sparse_get_segment_energies(g_, (int64_t)b, o, p); }
        check_sparse(rc, g_);
        return out;
    }
    void add_tweights(const py::object& nodes, py::array_t<double, py::array::c_style | py::array::forcecast> src,
                      py::array_t<double, py::array::c_style | py::array::forcecast> snk)
    {
        const py::ssize_t m = src.size();
        if (snk.size() != m) throw py::value_error("t-weight arrays differ in length");
        py::array_t<int32_t, py::array::c_style | py::array::forcecast> nd;
        const int32_t* np_ = nullptr;
        if (!nodes.is_none()) {
            nd = py::array_t<int32_t, py::array::c_style | py::array::forcecast>::ensure(nodes);
            if (!nd || nd.size() != m) throw py::value_error("node array does not match the t-weight arrays");
            np_ = nd.data();
        }
        int rc;
        { py::gil_scoped_release rel; rc = mgc_sparse_add_tweights(g_, (int64_t)m, np_, src.data(), snk.data()); }
        check_sparse(rc, g_);
    }
    double maxflow()
    {
        double e = 0;
        int rc;
        { py::gil_scoped_release rel; rc = mgc_sparse_maxflow(g_, &e); }
        check_sparse(rc, g_);
        return e;
    }
    py::array_t<uint8_t> get_mask()
    {
        int64_t n = 0;
        check_sparse(mgc_sparse_get_node_num(g_, &n), g_);
        py::array_t<uint8_t> out((py::ssize_t)n);
        int rc;
        { uint8_t* p = out.mutable_data(); py::gil_scoped_release rel; rc = mgc_sparse_get_mask(g_, p); }
        check_sparse(rc, g_);
        return out;
    }
    int what_segment(int64_t i) { int32_t s = 0; check_sparse(mgc_sparse_what_segment(g_, i, &s), g_); return s; }
    double get_edge(int64_t i, int64_t j) { double c = 0; check_sparse(mgc_sparse_get_edge(g_, i, j, &c), g_); return c; }
    double get_trcap(int64_t i) { double c = 0; check_sparse(mgc_sparse_get_trcap(g_, i, &c), g_); return c; }
    int64_t get_node_num() { int64_t n = 0; check_sparse(mgc_sparse_get_node_num(g_, &n), g_); return n; }
    int64_t get_arc_num() { int64_t n = 0; check_sparse(mgc_sparse_get_arc_num(g_, &n), g_); return n; }
    void reset() { check_sparse(mgc_sparse_reset(g_), g_); }
    py::dict stats()
    {
        mgc_stats s{};
        check_sparse(mgc_sparse_get_stats(g_, &s), g_);
        py::dict d;
        d["n_nodes"] = s.n_voxels; d["push_sweeps"] = s.push_sweeps; d["global_relabels"] = s.global_relabels;
        d["relabel_sweeps"] = s.relabel_sweeps; d["kernel_launches"] = s.kernel_launches; d["active_last"] = s.active_last;
        d["ms_solve"] = s.ms_solve; d["flow_const"] = s.flow_const; d["energy"] = s.energy; d["device_bytes"] = s.device_bytes;
        return d;
    }

private:
    mgc_sparse* g_ = nullptr;
};

// ---- label image resident on the device (mgc_labels_*) ------------------------------------------------------------
class PyLabels {
public:
    PyLabels(const py::object& labels, int device)
    {
        ArrayRef r = make_ref(labels, MGC_I32, "label_image");
        if (r.shape.empty() || r.shape.size() > MGC_MAX_NDIM) throw py::value_error("label_image must have 1 to 4 dimensions");
        shape_ = r.shape;
        int rc;
        { py::gil_scoped_release rel; rc = mgc_labels_create((int32_t)shape_.size(), shape_.data(), &r.a, device, &l_); }
        if (rc != MGC_OK) {
            std::string m = mgc_labels_last_error(nullptr);
            if (rc == MGC_E_LABELS) { PyErr_SetString(PyExc_AttributeError, m.c_str()); throw py::error_already_set(); }
            if (rc == MGC_E_ARG) throw py::value_error(m);
            throw std::runtime_error(m);
        }
    }
    // a batch: `shapes` one extent list per image (one ndim), `labels` the images' C-ordered voxels concatenated (1-D)
    static std::unique_ptr<PyLabels> batch(const std::vector<std::vector<int64_t>>& shapes, const py::object& labels, int device)
    {
        if (shapes.empty()) throw py::value_error("a batch holds at least one label image");
        const size_t nd = shapes[0].size();
        std::vector<int64_t> flat;
        for (const auto& s : shapes) {
            if (s.size() != nd) throw py::value_error("the images of a batch must have one number of dimensions");
            flat.insert(flat.end(), s.begin(), s.end());
        }
        ArrayRef r = make_ref(labels, MGC_I32, "label_images");
        if (r.shape.size() != 1) throw py::value_error("label_images: the concatenated images as one 1-D array expected");
        std::unique_ptr<PyLabels> out(new PyLabels());
        out->shape_ = r.shape;
        int rc;
        { py::gil_scoped_release rel; rc = mgc_labels_create_batch((int32_t)shapes.size(), (int32_t)nd, flat.data(), &r.a, device, &out->l_); }
        if (rc != MGC_OK) {
            std::string m = mgc_labels_last_error(nullptr);
            if (rc == MGC_E_LABELS) { PyErr_SetString(PyExc_AttributeError, m.c_str()); throw py::error_already_set(); }
            if (rc == MGC_E_ARG) throw py::value_error(m);
            throw std::runtime_error(m);
        }
        out->batch_ = (int64_t)shapes.size();
        return out;
    }
    py::array_t<int64_t> batch_offsets() const
    {
        py::array_t<int64_t> off((py::ssize_t)batch_ + 1);
        check(mgc_labels_batch_offsets(l_, off.mutable_data()));
        return off;
    }
    ~PyLabels() { if (l_) mgc_labels_destroy(l_); }
    PyLabels(const PyLabels&) = delete;
    PyLabels& operator=(const PyLabels&) = delete;

    void check(int rc) const
    {
        if (rc == MGC_OK) return;
        std::string msg = mgc_labels_last_error(l_);
        if (msg.empty()) msg = "medpy_b200 label image error " + std::to_string(rc);
        if (rc == MGC_E_ARG) throw py::value_error(msg);
        throw std::runtime_error(msg);
    }
    ArrayRef ref(const py::object& a, int want, const char* what) const
    {
        ArrayRef r = make_ref(a, want, what);
        if (r.shape != shape_) throw py::value_error(std::string(what) + ": shape does not match the label image");
        return r;
    }
    int64_t region_count() const { int64_t k = 0; check(mgc_labels_region_count(l_, &k)); return k; }

    // -> (i, j, w_ij, w_ji), one entry per adjacent region pair, sorted by (i, j), i < j (0-based node ids)
    py::tuple boundary(int kind, const py::object& values, double directedness)
    {
        ArrayRef r;
        const bool need = kind != MGC_LABELS_ADJACENCY;
        if (need) r = ref(values, -1, "image");
        int64_t m = 0;
        int rc;
        { py::gil_scoped_release rel; rc = mgc_labels_boundary(l_, kind, need ? &r.a : nullptr, directedness, &m); }
        check(rc);
        py::array_t<int32_t> i((py::ssize_t)m), j((py::ssize_t)m);
        py::array_t<double> w((py::ssize_t)m), wr((py::ssize_t)m);
        check(mgc_labels_fetch_edges(l_, i.mutable_data(), j.mutable_data(), w.mutable_data(), wr.mutable_data()));
        return py::make_tuple(i, j, w, wr);
    }
    py::tuple region_sums(const py::object& values, int mode)
    {
        ArrayRef r = ref(values, -1, "values");
        const int64_t k = region_count();
        py::array_t<double> sums((py::ssize_t)k);
        py::array_t<int64_t> counts((py::ssize_t)k);
        int rc;
        {
            double* ps = sums.mutable_data();
            int64_t* pc = counts.mutable_data();
            py::gil_scoped_release rel;
            rc = mgc_labels_region_sums(l_, &r.a, mode, ps, pc);
        }
        check(rc);
        return py::make_tuple(sums, counts);
    }
    py::array_t<uint8_t> region_flags(const py::object& markers)
    {
        ArrayRef r = ref(markers, MGC_U8, "markers");
        py::array_t<uint8_t> flags((py::ssize_t)region_count());
        int rc;
        { uint8_t* p = flags.mutable_data(); py::gil_scoped_release rel; rc = mgc_labels_region_flags(l_, &r.a, p); }
        check(rc);
        return flags;
    }
    // flags over all regions from int64 voxel ids (C order over the image, or over a batch's concatenation)
    py::array_t<uint8_t> voxel_flags(py::array_t<int64_t, py::array::c_style | py::array::forcecast> ids)
    {
        py::array_t<uint8_t> flags((py::ssize_t)region_count());
        int rc;
        { uint8_t* p = flags.mutable_data(); const int64_t* q = ids.data(); const int64_t m = (int64_t)ids.size(); py::gil_scoped_release rel; rc = mgc_labels_voxel_flags(l_, m, q, p); }
        check(rc);
        return flags;
    }
    py::array_t<uint8_t> apply(py::array_t<uint8_t, py::array::c_style | py::array::forcecast> per_region)
    {
        if (per_region.size() != region_count()) throw py::value_error("one value per region expected");
        std::vector<py::ssize_t> shp(shape_.begin(), shape_.end());
        py::array_t<uint8_t> out(shp);
        int rc;
        { uint8_t* p = out.mutable_data(); const uint8_t* q = per_region.data(); py::gil_scoped_release rel; rc = mgc_labels_apply(l_, q, p, MGC_MEM_HOST); }
        check(rc);
        return out;
    }
    // the same gather into a contiguous uint8 device array of the image shape (e.g. a torch CUDA tensor)
    void apply_into(py::array_t<uint8_t, py::array::c_style | py::array::forcecast> per_region, const py::object& out)
    {
        if (per_region.size() != region_count()) throw py::value_error("one value per region expected");
        ArrayRef r = make_ref(out, MGC_U8, "out");
        if (r.a.mem != MGC_MEM_DEVICE || r.shape != shape_) throw py::value_error("out: a device array of the image shape expected");
        int rc;
        { const uint8_t* q = per_region.data(); py::gil_scoped_release rel; rc = mgc_labels_apply(l_, q, (uint8_t*)r.a.data, MGC_MEM_DEVICE); }
        check(rc);
    }
    std::vector<int64_t> shape() const { return shape_; }

private:
    PyLabels() = default;
    mgc_labels* l_ = nullptr;
    std::vector<int64_t> shape_;
    int64_t batch_ = 1;
};

// The C ABI of one expansion unit, by handle type: the calls every expansion class makes
template <typename H> struct ExpansionAbi;
template <> struct ExpansionAbi<mgc_expansion> {
    static constexpr auto destroy = mgc_expansion_destroy;
    static constexpr auto last_error = mgc_expansion_last_error;
    static constexpr auto set_cost = mgc_expansion_set_cost;
    static constexpr auto set_markers = mgc_expansion_set_markers;
    static constexpr auto set_init = mgc_expansion_set_init;
    static constexpr auto set_moves = mgc_expansion_set_moves;
    static constexpr auto set_label_distance = mgc_expansion_set_label_distance;
    static constexpr auto run = mgc_expansion_run;
    static constexpr auto get_labels = mgc_expansion_get_labels;
    static constexpr auto get_stats = mgc_expansion_get_stats;
    static constexpr auto get_switched = mgc_expansion_get_switched;
};
template <> struct ExpansionAbi<mgc_expansion_batch> {
    static constexpr auto destroy = mgc_expansion_batch_destroy;
    static constexpr auto last_error = mgc_expansion_batch_last_error;
    static constexpr auto set_cost = mgc_expansion_batch_set_cost;
    static constexpr auto set_markers = mgc_expansion_batch_set_markers;
    static constexpr auto set_init = mgc_expansion_batch_set_init;
    static constexpr auto set_moves = mgc_expansion_batch_set_moves;
    static constexpr auto set_label_distance = mgc_expansion_batch_set_label_distance;
    static constexpr auto run = mgc_expansion_batch_run;
    static constexpr auto get_labels = mgc_expansion_batch_get_labels;
    static constexpr auto get_stats = mgc_expansion_batch_get_stats;
    static constexpr auto get_switched = mgc_expansion_batch_get_switched;
};
template <> struct ExpansionAbi<mgc_region_expansion> {     // no markers: they are in the caller's costs
    static constexpr auto destroy = mgc_region_expansion_destroy;
    static constexpr auto last_error = mgc_region_expansion_last_error;
    static constexpr auto set_cost = mgc_region_expansion_set_cost;
    static constexpr auto set_init = mgc_region_expansion_set_init;
    static constexpr auto set_moves = mgc_region_expansion_set_moves;
    static constexpr auto set_label_distance = mgc_region_expansion_set_label_distance;
    static constexpr auto run = mgc_region_expansion_run;
    static constexpr auto get_labels = mgc_region_expansion_get_labels;
    static constexpr auto get_stats = mgc_region_expansion_get_stats;
    static constexpr auto get_switched = mgc_region_expansion_get_switched;
};

// What the three K-label alpha-expansion classes share: every array has the handle's shape (`shape_`), and a refused
// call raises ValueError for MGC_E_ARG / MGC_E_WEIGHT, RuntimeError otherwise
template <typename H>
class PyExpansionBase {
public:
    using Abi = ExpansionAbi<H>;
    ~PyExpansionBase() { if (e_) Abi::destroy(e_); }
    PyExpansionBase(const PyExpansionBase&) = delete;
    PyExpansionBase& operator=(const PyExpansionBase&) = delete;

    void check(int rc) const
    {
        if (rc == MGC_OK) return;
        std::string msg = Abi::last_error(e_);
        if (msg.empty()) msg = "medpy_b200 expansion error " + std::to_string(rc);
        if (rc == MGC_E_ARG || rc == MGC_E_WEIGHT) throw py::value_error(msg);
        throw std::runtime_error(msg);
    }
    ArrayRef ref(const py::object& a, int want, const char* what) const
    {
        ArrayRef r = make_ref(a, want, what);
        if (r.shape != shape_) throw py::value_error(std::string(what) + ": " + mismatch_);
        return r;
    }
    void set_cost(int label, const py::object& cost)
    {
        ArrayRef r = ref(cost, -1, "costs");
        int rc;
        { py::gil_scoped_release rel; rc = Abi::set_cost(e_, label, &r.a); }
        check(rc);
    }
    void set_markers(const py::object& markers)
    {
        ArrayRef r = ref(markers, MGC_U8, "markers");
        int rc;
        { py::gil_scoped_release rel; rc = Abi::set_markers(e_, &r.a); }
        check(rc);
    }
    void set_init(const py::object& init)
    {
        ArrayRef r = ref(init, MGC_U8, "init");
        int rc;
        { py::gil_scoped_release rel; rc = Abi::set_init(e_, &r.a); }
        check(rc);
    }
    // MGC_MOVES_EXPANSION (0) or MGC_MOVES_SWAP (1); drops the label distance
    void set_moves(int kind)
    {
        int rc;
        { py::gil_scoped_release rel; rc = Abi::set_moves(e_, kind); }
        check(rc);
    }
    // a (K, K) float64 label distance, or None for Potts
    void set_label_distance(const py::object& dist)
    {
        py::array_t<double, py::array::c_style | py::array::forcecast> v;
        const double* p = nullptr;
        if (!dist.is_none()) {
            v = py::array_t<double, py::array::c_style | py::array::forcecast>::ensure(dist);
            if (!v || v.ndim() != 2 || v.shape(0) != labels_ || v.shape(1) != labels_)
                throw py::value_error("label_distance must be a (K, K) = (" + std::to_string(labels_) + ", " +
                                      std::to_string(labels_) + ") matrix");
            p = v.data();
        }
        int rc;
        { py::gil_scoped_release rel; rc = Abi::set_label_distance(e_, p); }
        check(rc);
    }
    void run(int max_cycles)
    {
        int rc;
        { py::gil_scoped_release rel; rc = Abi::run(e_, max_cycles); }
        check(rc);
    }
    py::array_t<uint8_t> labels()
    {
        std::vector<py::ssize_t> shp(shape_.begin(), shape_.end());
        py::array_t<uint8_t> out(shp);
        int rc;
        { uint8_t* p = out.mutable_data(); py::gil_scoped_release rel; rc = Abi::get_labels(e_, p, MGC_MEM_HOST); }
        check(rc);
        return out;
    }
    // into a contiguous uint8 device array of the handle's shape (e.g. a torch CUDA tensor)
    void labels_into(const py::object& out)
    {
        ArrayRef r = ref(out, MGC_U8, "out");
        if (r.a.mem != MGC_MEM_DEVICE) throw py::value_error("out: a device array expected");
        int rc;
        { py::gil_scoped_release rel; rc = Abi::get_labels(e_, (uint8_t*)r.a.data, MGC_MEM_DEVICE); }
        check(rc);
    }
    // moves, cycles, converged, energy, switched (one count per move) and device ms
    py::dict stats() const { return stats_dict(true); }

protected:
    PyExpansionBase(std::vector<int64_t> shape, int labels, const char* mismatch)
        : shape_(std::move(shape)), labels_(labels), mismatch_(mismatch)
    {
    }
    // after the unit's create(): raise its refusal
    void created(int rc) const
    {
        if (rc == MGC_OK) return;
        std::string m = Abi::last_error(nullptr);
        if (rc == MGC_E_ARG) throw py::value_error(m);
        throw std::runtime_error(m);
    }
    py::dict stats_dict(bool with_switched) const
    {
        mgc_expansion_stats s{};
        check(Abi::get_stats(e_, &s));
        py::dict d;
        d["moves"] = s.moves;
        d["cycles"] = s.cycles;
        d["converged"] = s.converged != 0;
        d["energy"] = s.energy;
        if (with_switched) {
            std::vector<int64_t> sw((size_t)s.moves);
            check(Abi::get_switched(e_, sw.data()));
            d["switched"] = sw;
        }
        d["ms_build"] = s.ms_build;
        d["ms_solve"] = s.ms_solve;
        d["ms_apply"] = s.ms_apply;
        d["ms_total"] = s.ms_total;
        return d;
    }

    H* e_ = nullptr;
    std::vector<int64_t> shape_;
    int labels_;
    const char* mismatch_;
};

// K-label alpha-expansion over one lattice (mgc_expansion_*)
class PyExpansion : public PyExpansionBase<mgc_expansion> {
public:
    PyExpansion(const std::vector<int64_t>& shape, int labels, int device)
        : PyExpansionBase(shape, labels, "shape does not match the lattice")
    {
        created(mgc_expansion_create((int32_t)shape.size(), shape.data(), labels, device, &e_));
    }
    // the GCGraph._add_boundary arguments a boundary term recorded
    void set_boundary(int kind, const py::object& image, double sigma, const py::object& spacing, double norm)
    {
        ArrayRef r = ref(image, -1, "image");
        std::vector<double> sp;
        if (!spacing.is_none()) {
            sp = spacing.cast<std::vector<double>>();
            if (sp.size() < shape_.size()) throw py::value_error("spacing has fewer entries than the image has dimensions");
        }
        int rc;
        { py::gil_scoped_release rel; rc = mgc_expansion_set_boundary(e_, kind, &r.a, sigma, sp.empty() ? nullptr : sp.data(), norm); }
        check(rc);
    }
};

// K-label alpha-expansion of a batch of images of one shape, every move one cut of the whole batch
// (mgc_expansion_batch_*); arrays are (batch, *image) with any positive strides
class PyExpansionBatch : public PyExpansionBase<mgc_expansion_batch> {
public:
    PyExpansionBatch(const std::vector<int64_t>& image_shape, int64_t batch, int labels, int device)
        : PyExpansionBase(image_shape, labels, "shape does not match (batch, *image)")
    {
        created(mgc_expansion_batch_create((int32_t)image_shape.size(), image_shape.data(), batch, labels, device, &e_));
        shape_.insert(shape_.begin(), batch);
    }
    // one sigma and one normaliser per image (NaN: reduced on the device), as build_voxel_batch takes them
    void set_boundary(int kind, const py::object& image, const std::vector<double>& sigmas, const py::object& spacing,
                      const std::vector<double>& norms)
    {
        if ((int64_t)sigmas.size() != shape_[0] || (int64_t)norms.size() != shape_[0])
            throw py::value_error("sigmas and norms need one entry per image");
        ArrayRef r = ref(image, -1, "image");
        std::vector<double> sp;
        if (!spacing.is_none()) {
            sp = spacing.cast<std::vector<double>>();
            if (sp.size() + 1 < shape_.size()) throw py::value_error("spacing has fewer entries than the images have dimensions");
        }
        int rc;
        {
            py::gil_scoped_release rel;
            rc = mgc_expansion_batch_set_boundary(e_, kind, &r.a, sigmas.data(), sp.empty() ? nullptr : sp.data(), norms.data());
        }
        check(rc);
    }
    // the batch loop: moves, cycles, converged (every image), energy (the sum over the images) and device ms
    py::dict stats() const { return stats_dict(false); }
    // per image: arrays of moves, cycles, converged and energy
    py::dict image_stats() const
    {
        const size_t B = (size_t)shape_[0];
        std::vector<mgc_expansion_stats> s(B);
        check(mgc_expansion_batch_get_image_stats(e_, s.data()));
        py::array_t<int64_t> moves((py::ssize_t)B), cycles((py::ssize_t)B);
        py::array_t<bool> conv((py::ssize_t)B);
        py::array_t<double> energy((py::ssize_t)B);
        for (size_t b = 0; b < B; ++b) {
            moves.mutable_data()[b] = s[b].moves;
            cycles.mutable_data()[b] = s[b].cycles;
            conv.mutable_data()[b] = s[b].converged != 0;
            energy.mutable_data()[b] = s[b].energy;
        }
        py::dict d;
        d["moves"] = moves;
        d["cycles"] = cycles;
        d["converged"] = conv;
        d["energy"] = energy;
        return d;
    }
    // (moves, batch) int64: the voxels of every image each move switched
    py::array_t<int64_t> switched() const
    {
        mgc_expansion_stats s{};
        check(mgc_expansion_batch_get_stats(e_, &s));
        py::array_t<int64_t> out({(py::ssize_t)s.moves, (py::ssize_t)shape_[0]});
        check(mgc_expansion_batch_get_switched(e_, out.mutable_data()));
        return out;
    }
    // the pair weights along image axis `axis`, shape (batch, *image)
    py::array_t<double> weights(int axis)
    {
        std::vector<py::ssize_t> shp(shape_.begin(), shape_.end());
        py::array_t<double> out(shp);
        int rc;
        { double* p = out.mutable_data(); py::gil_scoped_release rel; rc = mgc_expansion_batch_get_weights(e_, axis, p, MGC_MEM_HOST); }
        check(rc);
        return out;
    }
};

// K-label alpha-expansion over a region adjacency graph (mgc_region_expansion_*); per-region arrays are (regions,)
class PyRegionExpansion : public PyExpansionBase<mgc_region_expansion> {
public:
    PyRegionExpansion(int64_t regions, int labels, int device) : PyExpansionBase({regions}, labels, "one entry per region expected")
    {
        created(mgc_region_expansion_create(regions, labels, device, &e_));
    }
    void set_pairs(py::array_t<int32_t, py::array::c_style | py::array::forcecast> i,
                   py::array_t<int32_t, py::array::c_style | py::array::forcecast> j,
                   py::array_t<double, py::array::c_style | py::array::forcecast> w)
    {
        if (i.size() != j.size() || i.size() != w.size()) throw py::value_error("i, j and w must have the same length");
        int rc;
        {
            const int32_t *pi = i.data(), *pj = j.data();
            const double* pw = w.data();
            const int64_t m = (int64_t)i.size();
            py::gil_scoped_release rel;
            rc = mgc_region_expansion_set_pairs(e_, m, pi, pj, pw);
        }
        check(rc);
    }
};

}  // namespace

py::array_t<float> gradient_magnitude_prewitt(const py::object& image, int device)
{
    ArrayRef r = make_ref(image, -1, "image");
    if (r.shape.empty() || r.shape.size() > 4) throw py::value_error("image must have 1 to 4 dimensions");
    std::vector<py::ssize_t> shp(r.shape.begin(), r.shape.end());
    py::array_t<float> out(shp);
    int rc;
    {
        float* p = out.mutable_data();
        py::gil_scoped_release rel;
        rc = mgc_gradient_magnitude_prewitt((int32_t)r.shape.size(), r.shape.data(), &r.a, p, MGC_MEM_HOST, device);
    }
    check(rc, nullptr);
    return out;
}

PYBIND11_MODULE(_mgc, m)
{
    m.def("trim_pools", []() { mgc_trim_pools(); }, "Return every cached device / pinned block to the driver (live graphs keep theirs).");
    m.def("gradient_magnitude_prewitt", &gradient_magnitude_prewitt, py::arg("image"), py::arg("device") = -1);
    m.doc() = "pybind11 binding of libmedpy_b200_gc (H100 voxel graph-cut C ABI)";
    m.attr("ABI_VERSION") = mgc_abi_version();
    m.attr("SOURCE") = MGC_SOURCE;
    m.attr("SINK") = MGC_SINK;
    m.attr("OPT_DEFER_WEIGHT_CHECK") = MGC_OPT_DEFER_WEIGHT_CHECK;
    m.attr("OPT_WARM") = MGC_OPT_WARM;
    m.attr("OPT_KEEP_DEVICE_INPUTS") = MGC_OPT_KEEP_DEVICE_INPUTS;
    m.attr("OPT_SEGMENT_ENERGIES") = MGC_OPT_SEGMENT_ENERGIES;
    m.attr("MOVES_EXPANSION") = MGC_MOVES_EXPANSION;
    m.attr("MOVES_SWAP") = MGC_MOVES_SWAP;
    m.attr("LABELS_ADJACENCY") = MGC_LABELS_ADJACENCY;
    m.attr("LABELS_STAWIASKI") = MGC_LABELS_STAWIASKI;
    m.attr("LABELS_STAWIASKI_DIRECTED") = MGC_LABELS_STAWIASKI_DIRECTED;
    m.attr("SUM_BINCOUNT") = MGC_SUM_BINCOUNT;
    m.attr("SUM_PAIRWISE") = MGC_SUM_PAIRWISE;
    py::class_<PyExpansion>(m, "Expansion")
        .def(py::init<const std::vector<int64_t>&, int, int>(), py::arg("shape"), py::arg("labels"), py::arg("device") = -1)
        .def("set_cost", &PyExpansion::set_cost)
        .def("set_boundary", &PyExpansion::set_boundary)
        .def("set_markers", &PyExpansion::set_markers)
        .def("set_init", &PyExpansion::set_init)
        .def("set_moves", &PyExpansion::set_moves)
        .def("set_label_distance", &PyExpansion::set_label_distance)
        .def("run", &PyExpansion::run)
        .def("labels", &PyExpansion::labels)
        .def("labels_into", &PyExpansion::labels_into)
        .def("stats", &PyExpansion::stats);
    py::class_<PyExpansionBatch>(m, "ExpansionBatch")
        .def(py::init<const std::vector<int64_t>&, int64_t, int, int>(), py::arg("image_shape"), py::arg("batch"),
             py::arg("labels"), py::arg("device") = -1)
        .def("set_cost", &PyExpansionBatch::set_cost)
        .def("set_boundary", &PyExpansionBatch::set_boundary)
        .def("set_markers", &PyExpansionBatch::set_markers)
        .def("set_init", &PyExpansionBatch::set_init)
        .def("set_moves", &PyExpansionBatch::set_moves)
        .def("set_label_distance", &PyExpansionBatch::set_label_distance)
        .def("run", &PyExpansionBatch::run)
        .def("labels", &PyExpansionBatch::labels)
        .def("labels_into", &PyExpansionBatch::labels_into)
        .def("stats", &PyExpansionBatch::stats)
        .def("image_stats", &PyExpansionBatch::image_stats)
        .def("switched", &PyExpansionBatch::switched)
        .def("weights", &PyExpansionBatch::weights);
    py::class_<PyRegionExpansion>(m, "RegionExpansion")
        .def(py::init<int64_t, int, int>(), py::arg("regions"), py::arg("labels"), py::arg("device") = -1)
        .def("set_cost", &PyRegionExpansion::set_cost)
        .def("set_pairs", &PyRegionExpansion::set_pairs)
        .def("set_init", &PyRegionExpansion::set_init)
        .def("set_moves", &PyRegionExpansion::set_moves)
        .def("set_label_distance", &PyRegionExpansion::set_label_distance)
        .def("run", &PyRegionExpansion::run)
        .def("labels", &PyRegionExpansion::labels)
        .def("stats", &PyRegionExpansion::stats);
    py::class_<PySparse>(m, "SparseGraph")
        .def(py::init<int64_t, int>(), py::arg("n_nodes"), py::arg("device") = -1)
        .def("sum_edges", &PySparse::sum_edges)
        .def("remove_edges_warm", &PySparse::remove_edges_warm)
        .def("set_option", &PySparse::set_option)
        .def("segment_energies", &PySparse::segment_energies)
        .def("add_tweights", &PySparse::add_tweights)
        .def("maxflow", &PySparse::maxflow)
        .def("get_mask", &PySparse::get_mask)
        .def("what_segment", &PySparse::what_segment)
        .def("get_edge", &PySparse::get_edge)
        .def("get_trcap", &PySparse::get_trcap)
        .def("get_node_num", &PySparse::get_node_num)
        .def("get_arc_num", &PySparse::get_arc_num)
        .def("reset", &PySparse::reset)
        .def("stats", &PySparse::stats);
    py::class_<PyLabels>(m, "LabelImage")
        .def(py::init<const py::object&, int>(), py::arg("label_image"), py::arg("device") = -1)
        .def("region_count", &PyLabels::region_count)
        .def("boundary", &PyLabels::boundary, py::arg("kind"), py::arg("values") = py::none(), py::arg("directedness") = 0.0)
        .def("region_sums", &PyLabels::region_sums)
        .def("region_flags", &PyLabels::region_flags)
        .def("voxel_flags", &PyLabels::voxel_flags)
        .def("apply", &PyLabels::apply)
        .def("apply_into", &PyLabels::apply_into)
        .def_static("batch", &PyLabels::batch, py::arg("shapes"), py::arg("label_images"), py::arg("device") = -1)
        .def("batch_offsets", &PyLabels::batch_offsets)
        .def_property_readonly("shape", &PyLabels::shape);
    py::class_<PyGraph>(m, "Graph")
        .def(py::init<const std::vector<int64_t>&, int>(), py::arg("shape"), py::arg("device") = -1)
        .def(py::init<const std::vector<int64_t>&, int64_t, int64_t, int>(), py::arg("shape"), py::arg("z0"), py::arg("z1"), py::arg("device") = -1)
        .def("add_regional_probability", &PyGraph::add_regional_probability)
        .def("add_tweights_dense", &PyGraph::add_tweights_dense)
        .def("add_markers", &PyGraph::add_markers)
        .def("add_boundary", &PyGraph::add_boundary)
        .def("add_nweights_dense", &PyGraph::add_nweights_dense)
        .def("add_seeds", &PyGraph::add_seeds, py::arg("fg_ids"), py::arg("bg_ids"))
        .def("remove_seeds", &PyGraph::remove_seeds, py::arg("fg_ids"), py::arg("bg_ids"))
        .def("add_tweights_warm", &PyGraph::add_tweights_warm, py::arg("ids"), py::arg("src"), py::arg("snk"))
        .def("add_nweights_warm", &PyGraph::add_nweights_warm, py::arg("i"), py::arg("j"), py::arg("cap"), py::arg("rev_cap"))
        .def("add_nweights_dense_warm", &PyGraph::add_nweights_dense_warm, py::arg("axis"), py::arg("fwd"), py::arg("bwd"))
        .def("remove_nweights_warm", &PyGraph::remove_nweights_warm, py::arg("i"), py::arg("j"), py::arg("cap"), py::arg("rev_cap"))
        .def("remove_nweights_dense_warm", &PyGraph::remove_nweights_dense_warm, py::arg("axis"), py::arg("fwd"), py::arg("bwd"))
        .def("build_voxel_graph", &PyGraph::build_voxel_graph)
        .def_static("batch", &PyGraph::batch, py::arg("image_shape"), py::arg("batch"), py::arg("device") = -1)
        .def("build_voxel_batch", &PyGraph::build_voxel_batch)
        .def("get_batch_energies", &PyGraph::get_batch_energies)
        .def_static("slab_comm_unique_id", &PyGraph::slab_comm_unique_id)
        .def("slab_comm_init", &PyGraph::slab_comm_init)
        .def("slab_solve", &PyGraph::slab_solve)
        .def("slab_solve_stats", &PyGraph::slab_solve_stats)
        .def("can_fuse", &PyGraph::can_fuse)
        .def("set_pack_markers", &PyGraph::set_pack_markers)
        .def("set_keep_device_inputs", &PyGraph::set_keep_device_inputs)
        .def("maxflow", &PyGraph::maxflow)
        .def("get_mask", &PyGraph::get_mask)
        .def("get_mask_into", &PyGraph::get_mask_into)
        .def("what_segment", &PyGraph::what_segment)
        .def("get_edge", &PyGraph::get_edge)
        .def("get_trcap", &PyGraph::get_trcap)
        .def("get_node_num", &PyGraph::get_node_num)
        .def("get_arc_num", &PyGraph::get_arc_num)
        .def("reset", &PyGraph::reset)
        .def("set_option", &PyGraph::set_option)
        .def("check_deferred", &PyGraph::check_deferred)
        .def("set_stream", &PyGraph::set_stream)
        .def("synchronize", &PyGraph::synchronize)
        .def("stats", &PyGraph::stats)
        .def("slab_plane_elems", &PyGraph::slab_plane_elems)
        .def("slab_begin", &PyGraph::slab_begin)
        .def("slab_push", &PyGraph::slab_push)
        .def("slab_pack", &PyGraph::slab_pack)
        .def("slab_unpack", &PyGraph::slab_unpack)
        .def("slab_relabel_begin", &PyGraph::slab_relabel_begin)
        .def("slab_relabel_relax", &PyGraph::slab_relabel_relax, py::arg("want_changed") = false)
        .def("slab_count_active_dev", &PyGraph::slab_count_active_dev)
        .def("slab_count_active", &PyGraph::slab_count_active)
        .def("slab_finish", &PyGraph::slab_finish)
        .def_property_readonly("shape", &PyGraph::shape);
}
