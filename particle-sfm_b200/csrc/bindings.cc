// bindings.cc — the `particlesfm` Python module (pybind11), same surface as the
// reference's (point_trajectory/optimize/src/bindings.cc:27-77), so that
// `from .optimize.build import particlesfm` (point_trajectory/trajectory.py:23) resolves
// to this build.  optimize_location forwards to the CUDA library through the C ABI
// (psfm_traj_optimize); there is no CPU implementation in this module.
#include <dlfcn.h>
#include <pybind11/numpy.h>
#include <pybind11/pybind11.h>
#include <pybind11/stl.h>

#include <cmath>
#include <cstring>
#include <string>

#include "psfm_b200.h"
#include "trajectory_base.h"

namespace py = pybind11;
using psfm::Trajectory;
using psfm::TrajectorySet;
using psfm::Vec2;

// ---- Vec2 <-> Python (any length-2 sequence / array in, float64 ndarray of shape (2,) out)
namespace pybind11 {
namespace detail {
template <>
struct type_caster<Vec2> {
 public:
  PYBIND11_TYPE_CASTER(Vec2, const_name("numpy.ndarray[float64[2]]"));
  bool load(handle src, bool) {
    if (!src) return false;
    auto arr = array_t<double, array::c_style | array::forcecast>::ensure(src);
    if (!arr) { PyErr_Clear(); return false; }
    if (arr.size() != 2) return false;
    value.x = arr.data()[0];
    value.y = arr.data()[1];
    return true;
  }
  static handle cast(const Vec2& v, return_value_policy, handle) {
    array_t<double> a(2);
    a.mutable_data()[0] = v.x;
    a.mutable_data()[1] = v.y;
    return a.release();
  }
};
}  // namespace detail
}  // namespace pybind11

namespace {

// ---- the CUDA library, resolved next to this module
struct Api {
  void* handle = nullptr;
  int (*traj_optimize)(const double*, const double*, const double*, const double*, const float*, int32_t, int32_t,
                       int32_t, const psfm_traj_options*, double*, psfm_traj_summary*) = nullptr;
  const char* (*last_error)(void) = nullptr;
};

Api& api() {
  static Api a;
  if (a.handle) return a;
  Dl_info info;
  std::string dir = ".";
  if (dladdr((void*)&api, &info) && info.dli_fname) {
    std::string p(info.dli_fname);
    const size_t s = p.find_last_of('/');
    if (s != std::string::npos) dir = p.substr(0, s);
  }
  const std::string path = dir + "/libpsfm_b200.so";
  a.handle = dlopen(path.c_str(), RTLD_NOW | RTLD_LOCAL);
  if (!a.handle) throw std::runtime_error("particlesfm: cannot load " + path + ": " + dlerror() +
                                          " (build it with `python -m particlesfm_b200.build`; no CPU fallback)");
  a.traj_optimize = (decltype(a.traj_optimize))dlsym(a.handle, "psfm_traj_optimize");
  a.last_error = (decltype(a.last_error))dlsym(a.handle, "psfm_last_error");
  if (!a.traj_optimize || !a.last_error) throw std::runtime_error("particlesfm: libpsfm_b200.so lacks psfm_traj_optimize");
  return a;
}

using DArr = py::array_t<double, py::array::c_style | py::array::forcecast>;

// optimize_location(uv12[N,4], uv_ref1[N,2], uv_ref2[N,2], ref2_scale[N,1], flow12_map[H,W,2], total_num, width, height)
py::array_t<double> optimize_location(DArr uv12, DArr ref1, DArr ref2, DArr scale, py::array flow12_map,
                                      int total_num, int width, int height) {
  if (total_num < 0) throw std::runtime_error("optimize_location: negative total_num");
  if (uv12.size() < 4 * (py::ssize_t)total_num || ref1.size() < 2 * (py::ssize_t)total_num ||
      ref2.size() < 2 * (py::ssize_t)total_num || scale.size() < (py::ssize_t)total_num)
    throw std::runtime_error("optimize_location: arrays shorter than total_num rows");
  // The reference widens the map to float64 (py::array_t<double>).  The device keeps
  // float32 (RAFT writes .flo as float32) and widens on load, which is exact; a float64
  // map that is not float32-representable is rejected instead of being silently rounded.
  auto f32 = py::array_t<float, py::array::c_style | py::array::forcecast>::ensure(flow12_map);
  if (!f32) throw std::runtime_error("optimize_location: flow12_map is not a numeric array");
  if ((py::ssize_t)f32.size() != 2 * (py::ssize_t)width * height)
    throw std::runtime_error("optimize_location: flow12_map must have height*width*2 elements");
  if (py::isinstance<py::array_t<double>>(flow12_map)) {
    auto f64 = py::array_t<double, py::array::c_style | py::array::forcecast>::ensure(flow12_map);
    const double* d = f64.data();
    const float* f = f32.data();
    for (py::ssize_t i = 0; i < f64.size(); ++i)
      if ((double)f[i] != d[i] && !(std::isnan(d[i]) && std::isnan(f[i])))
        throw std::runtime_error("optimize_location: float64 flow12_map is not representable in float32");
  }
  py::array_t<double> out({(py::ssize_t)total_num, (py::ssize_t)4});
  if (total_num == 0) return out;
  Api& a = api();
  int rc;
  {
    py::gil_scoped_release nogil;
    rc = a.traj_optimize(uv12.data(), ref1.data(), ref2.data(), scale.data(), f32.data(), total_num, width, height,
                         nullptr, out.mutable_data(), nullptr);
  }
  if (rc != 0) throw std::runtime_error(std::string("optimize_location: ") + a.last_error());
  return out;
}

py::dict traj_as_dict(const Trajectory& t) {
  py::dict d;
  d["frame_ids"] = t.times;
  py::list locs;
  for (const Vec2& p : t.xys) locs.append(py::cast(p));
  d["locations"] = locs;
  d["labels"] = t.labels;
  return d;
}

Trajectory traj_from_dict(const py::dict& d) {
  Trajectory t;
  if (d.contains("frame_ids")) t.times = d["frame_ids"].cast<std::vector<int>>();
  if (d.contains("locations")) t.xys = d["locations"].cast<std::vector<Vec2>>();
  if (d.contains("labels")) t.labels = d["labels"].cast<std::vector<bool>>();
  return t;
}

std::map<int, py::dict> set_as_dict(const TrajectorySet& s) {
  std::map<int, py::dict> out;
  for (const auto& kv : s.trajs) out[kv.first] = traj_as_dict(kv.second);
  return out;
}

TrajectorySet set_from_dict(const std::map<int, py::dict>& in) {
  TrajectorySet s;
  for (const auto& kv : in) s.trajs.emplace(kv.first, traj_from_dict(kv.second));
  return s;
}

// The track set as the window sampler reads it: trajectories in ascending id order; for each, the first observation of
// every frame among its first min(times, xys) entries (build_invert_indexes keeps the first), frames ascending.
py::tuple set_csr(const TrajectorySet& s) {
  std::vector<int64_t> ids, ptr{0};
  std::vector<int32_t> frames;
  std::vector<double> xy;
  for (const auto& kv : s.trajs) {
    const Trajectory& t = kv.second;
    const size_t n = std::min(t.times.size(), t.xys.size());
    std::map<int, size_t> first;
    for (size_t i = 0; i < n; ++i) first.emplace(t.times[i], i);
    for (const auto& f : first) {
      frames.push_back(f.first);
      xy.push_back(t.xys[f.second].x);
      xy.push_back(t.xys[f.second].y);
    }
    ids.push_back(kv.first);
    ptr.push_back((int64_t)frames.size());
  }
  py::array_t<int64_t> a_ids((py::ssize_t)ids.size()), a_ptr((py::ssize_t)ptr.size());
  py::array_t<int32_t> a_frames((py::ssize_t)frames.size());
  py::array_t<double> a_xy({(py::ssize_t)frames.size(), (py::ssize_t)2});
  std::copy(ids.begin(), ids.end(), a_ids.mutable_data());
  std::copy(ptr.begin(), ptr.end(), a_ptr.mutable_data());
  std::copy(frames.begin(), frames.end(), a_frames.mutable_data());
  std::copy(xy.begin(), xy.end(), a_xy.mutable_data());
  return py::make_tuple(a_ids, a_ptr, a_frames, a_xy);
}

}  // namespace

PYBIND11_MODULE(particlesfm, m) {
  m.doc() = "point trajectories + path-consistency optimiser (H100 build)";
  m.def("optimize_location", &optimize_location, py::arg("uv12"), py::arg("uv_ref1"), py::arg("uv_ref2"),
        py::arg("ref2_scale"), py::arg("flow12_map"), py::arg("total_num"), py::arg("width"), py::arg("height"));

  py::class_<Trajectory>(m, "Trajectory")
      .def(py::init([](int time, Vec2 p, int buffer_size) { return Trajectory(time, p, buffer_size); }),
           py::arg("time"), py::arg("point"), py::kw_only(), py::arg("buffer_size") = 0)
      .def(py::init([](double time, Vec2 p, int buffer_size) { return Trajectory((int)time, p, buffer_size); }),
           py::arg("time"), py::arg("point"), py::kw_only(), py::arg("buffer_size") = 0)
      .def(py::init([](std::vector<int> times, std::vector<Vec2> xys, std::vector<bool> labels) {
             return Trajectory(std::move(times), std::move(xys), std::move(labels));
           }),
           py::arg("times"), py::arg("xys"), py::kw_only(), py::arg("labels") = std::vector<bool>())
      .def(py::init([](const py::dict& d) { return traj_from_dict(d); }))
      .def("as_dict", &traj_as_dict)
      .def(py::pickle([](const Trajectory& t) { return traj_as_dict(t); },
                      [](const py::dict& d) { return traj_from_dict(d); }))
      .def_readonly("times", &Trajectory::times)
      .def_readonly("labels", &Trajectory::labels)
      .def_readonly("xys", &Trajectory::xys)
      .def_readonly("buffer_xys", &Trajectory::buffer_xys)
      .def("extend", &Trajectory::extend)
      .def("clear_buffer", &Trajectory::clear_buffer)
      .def("set_buffer_xy", &Trajectory::set_buffer_xy)
      .def("set_label", &Trajectory::set_label)
      .def("set_labels", &Trajectory::set_labels)
      .def("length", &Trajectory::length)
      .def("get_tail_location", &Trajectory::get_tail_location);

  py::class_<TrajectorySet>(m, "TrajectorySet")
      .def(py::init<>())
      .def(py::init([](const std::map<int, Trajectory>& t) { return TrajectorySet(t); }))
      .def(py::init([](const std::map<int, py::dict>& d) { return set_from_dict(d); }))
      .def("as_dict", &set_as_dict)
      .def(py::pickle([](const TrajectorySet& s) { return set_as_dict(s); },
                      [](const std::map<int, py::dict>& d) { return set_from_dict(d); }))
      .def_readonly("trajs", &TrajectorySet::trajs)
      .def("insert", &TrajectorySet::insert)
      .def("build_invert_indexes", &TrajectorySet::build_invert_indexes)
      .def("sample_inside_window",
           [](const TrajectorySet& s, const std::vector<int>& frame_ids, int min_length, int max_num_tracks) {
             const psfm::WindowSample w = s.sample_inside_window(frame_ids, min_length, max_num_tracks);
             py::array_t<double> lx({(py::ssize_t)w.K, (py::ssize_t)w.L}), ly({(py::ssize_t)w.K, (py::ssize_t)w.L});
             py::array_t<int> mk({(py::ssize_t)w.K, (py::ssize_t)w.L});
             if (w.K * w.L > 0) {
               std::memcpy(lx.mutable_data(), w.loc_x.data(), sizeof(double) * w.loc_x.size());
               std::memcpy(ly.mutable_data(), w.loc_y.data(), sizeof(double) * w.loc_y.size());
               std::memcpy(mk.mutable_data(), w.masks.data(), sizeof(int) * w.masks.size());
             }
             py::dict out;
             out["locations"] = py::make_tuple(lx, ly);
             out["masks"] = mk;
             out["traj_ids"] = w.traj_ids;
             return out;
           },
           py::arg("frame_ids"), py::arg("min_length") = 3, py::arg("max_num_tracks") = 100000)
      .def("csr", &set_csr,
           "(ids [T] int64 ascending, ptr [T+1] int64, frame_ids [M] int32, xy [M, 2] float64): every trajectory's "
           "observations as sample_inside_window sees them, one per frame (its first), frames ascending.");
}
