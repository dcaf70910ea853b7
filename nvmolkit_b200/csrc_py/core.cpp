// nvmolkit_b200._core — the C++ / pybind11 host module over the C-ABI of libb200mol.so (include/b200mol.h).
//
// What the reference does with Boost.Python glue per module (nvmolkit/*.cpp: convert arguments, call the C++ entry
// point, translate exceptions) happens here once, generically: every C-ABI function is exported under its own name,
// pointer parameters travel as integers (torch `data_ptr()`, `ctypes.addressof`, CUDA-array-interface addresses), the GIL
// is RELEASED for the duration of the native call (the reference holds it, SURVEY.md 8b "Threading"), and the status
// code comes back as the exception type the reference's bindings raise: B200MOL_ERR_INVALID -> ValueError
// (std::invalid_argument there), anything else -> RuntimeError. A few host-only helpers that were Python loops
// (CSR row gathers, running per-molecule conformer indices) live here as C++ too.
#include <pybind11/numpy.h>
#include <pybind11/pybind11.h>
#include <pybind11/stl.h>

#include <cstdint>
#include <stdexcept>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/b200mol.h"

namespace py = pybind11;

namespace {

struct B200Error : std::runtime_error {
  using std::runtime_error::runtime_error;
};

void raise(int status) {
  if (status == B200MOL_OK) return;
  const std::string msg = b200mol_last_error();
  if (status == B200MOL_ERR_INVALID) throw py::value_error(msg);
  throw B200Error(msg);
}

// Python-facing type of a C parameter: pointers -> integers, C strings -> str, everything else unchanged.
template <class T>
struct Arg {
  using type = T;
  static T to(const T& v) { return v; }
};
template <class T>
struct Arg<T*> {
  using type = std::uintptr_t;
  static T* to(std::uintptr_t v) { return reinterpret_cast<T*>(v); }
};
template <>
struct Arg<const char*> {
  using type = std::string;
  static const char* to(const std::string& v) { return v.c_str(); }
};

template <class... A>
void def(py::module_& m, const char* name, int (*fn)(A...)) {
  m.def(name, [fn](typename Arg<A>::type... a) {
    int status;
    {
      py::gil_scoped_release nogil;
      status = fn(Arg<A>::to(a)...);
    }
    raise(status);
  });
}

// concatenation of arange(starts[c], starts[c+1]) for c in order (CSR row gather)
py::array_t<int64_t> rowsOf(py::array_t<int64_t, py::array::c_style | py::array::forcecast> starts,
                            py::array_t<int64_t, py::array::c_style | py::array::forcecast> order) {
  const auto    st = starts.unchecked<1>();
  const auto    od = order.unchecked<1>();
  int64_t       total = 0;
  for (py::ssize_t k = 0; k < od.shape(0); ++k) {
    if (od(k) < 0 || od(k) + 1 >= st.shape(0)) throw py::value_error("row index out of range");
    total += st(od(k) + 1) - st(od(k));
  }
  py::array_t<int64_t> out(total);
  auto                 o = out.mutable_unchecked<1>();
  int64_t              at = 0;
  for (py::ssize_t k = 0; k < od.shape(0); ++k)
    for (int64_t r = st(od(k)); r < st(od(k) + 1); ++r) o(at++) = r;
  return out;
}

// k-th occurrence number of each key in order of appearance (conformer index within its molecule)
py::array_t<int32_t> runningIndex(py::array_t<int64_t, py::array::c_style | py::array::forcecast> keys) {
  const auto                           k = keys.unchecked<1>();
  py::array_t<int32_t>                 out(k.shape(0));
  auto                                 o = out.mutable_unchecked<1>();
  std::unordered_map<int64_t, int32_t> seen;
  for (py::ssize_t i = 0; i < k.shape(0); ++i) o(i) = seen[k(i)]++;
  return out;
}

}  // namespace

PYBIND11_MODULE(_core, m) {
  m.doc() = "pybind11 host module over libb200mol.so (GIL released around every native call)";
  py::register_exception<B200Error>(m, "B200MolError", PyExc_RuntimeError);
  m.def("last_error", [] { return std::string(b200mol_last_error()); });
  m.def("abi_version", &b200mol_abi_version);
  m.def("launch_count", &b200mol_launch_count);
  m.def("rows_of", &rowsOf);
  m.def("running_index", &runningIndex);
  m.def("get_option", [](const std::string& key) {
    long long v = 0;
    raise(b200mol_get_option(key.c_str(), &v));
    return v;
  });
  m.def("profile_read", [](const std::string& phase) {
    float ms = 0.f;
    raise(b200mol_profile_read(phase.c_str(), &ms));
    return ms;
  });
#define DEF(name) def(m, #name, &name)
  DEF(b200mol_check_device);
  DEF(b200mol_free_async);
  DEF(b200mol_set_option);
  DEF(b200mol_profile_enable);
  DEF(b200mol_stats_read);
  DEF(b200mol_tanimoto_cross);
  DEF(b200mol_cosine_cross);
  DEF(b200mol_similarity_cross_host);
  DEF(b200mol_tanimoto_count_ge);
  DEF(b200mol_similarity_topk);
  DEF(b200mol_similarity_threshold);
  DEF(b200mol_tversky_cross);
  DEF(b200mol_tversky_cross_host);
  DEF(b200mol_tversky_topk);
  DEF(b200mol_tversky_threshold);
  DEF(b200mol_count_cross);
  DEF(b200mol_count_topk);
  DEF(b200mol_count_threshold);
  DEF(b200mol_maxmin_pick);
  DEF(b200mol_leader_pick);
  DEF(b200mol_butina_fused);
  DEF(b200mol_neighbor_edges);
  DEF(b200mol_butina_from_edges);
  DEF(b200mol_butina_dense);
  DEF(b200mol_count_neighbor_edges);
  DEF(b200mol_count_butina_fused);
  DEF(b200mol_morgan);
  DEF(b200mol_morgan_counts);
  DEF(b200mol_schedule_waves);
  DEF(b200mol_dg_terms_from_bounds);
  DEF(b200mol_etk_terms_from_details);
  DEF(b200mol_mmff_energy_grad);
  DEF(b200mol_uff_energy_grad);
  DEF(b200mol_dg_energy_grad);
  DEF(b200mol_etk_energy_grad);
  DEF(b200mol_mmff_minimize);
  DEF(b200mol_uff_minimize);
  DEF(b200mol_dg_minimize);
  DEF(b200mol_etk_minimize);
  DEF(b200mol_poly_minimize);
  DEF(b200mol_etkdg_embed);
  DEF(b200mol_etkdg_initial_coords);
  DEF(b200mol_etkdg_check);
  DEF(b200mol_triangle_smooth);
  DEF(b200mol_eig_topk);
  DEF(b200mol_metric_embed);
  DEF(b200mol_rms_prune);
  DEF(b200mol_tfd_matrices);
  DEF(b200mol_conformer_rmsd);
  DEF(b200mol_conformer_rmsd_mapped);
  DEF(b200mol_align);
  DEF(b200mol_best_align);
  DEF(b200mol_allgather_counts);
  DEF(b200mol_allgather_results);
#undef DEF
}
