/*
 * gtn/pybind.cpp -- Python bindings with the reference's surface
 * (bindings/python/gtn/_graph.cpp, _functions.cpp, _autograd.cpp, _creations.cpp,
 * _parallel.cpp; flattened into one module like gtn/__init__.py:13-20 does): every
 * function has a single-graph and a list-of-graphs overload, calls release the GIL.
 */
#include <pybind11/functional.h>
#include <pybind11/numpy.h>
#include <pybind11/pybind11.h>
#include <pybind11/stl.h>

#include <cstdlib>
#include <cstring>
#include <sstream>

#include "gtn/device.h"
#include "gtn/gtn.h"

using namespace gtn;
namespace py = pybind11;
using namespace py::literals;

namespace {

template <typename F>
auto unary(F f) {
  return [f](const Graph& g) {
    py::gil_scoped_release release;
    return f(g);
  };
}
template <typename F>
auto unaryList(F f) {
  return [f](const std::vector<Graph>& gs) {
    py::gil_scoped_release release;
    return parallelMap(f, gs);
  };
}
template <typename F>
auto binary(F f) {
  return [f](const Graph& a, const Graph& b) {
    py::gil_scoped_release release;
    return f(a, b);
  };
}
template <typename F>
auto binaryList(F f) {
  return [f](const std::vector<Graph>& a, const std::vector<Graph>& b) {
    py::gil_scoped_release release;
    return parallelMap(f, a, b);
  };
}

} // namespace

PYBIND11_MODULE(_gtn, m) {
  m.attr("epsilon") = epsilon;
  m.attr("__version__") = "0.0.0+b200";

  py::enum_<Projection>(m, "Projection")
      .value("NONE", Projection::NONE)
      .value("INPUT", Projection::INPUT)
      .value("OUTPUT", Projection::OUTPUT);

  py::class_<Graph>(m, "Graph")
      .def(py::init<bool>(), "calc_grad"_a = true)
      .def("add_node", &Graph::addNode, "start"_a = false, "accept"_a = false)
      .def("add_arc", py::overload_cast<size_t, size_t, int>(&Graph::addArc), "src_node"_a, "dst_node"_a, "label"_a)
      .def(
          "add_arc", py::overload_cast<size_t, size_t, int, int, float>(&Graph::addArc), "src_node"_a,
          "dst_node"_a, "ilabel"_a, "olabel"_a, "weight"_a = 0.0)
      .def("num_arcs", &Graph::numArcs)
      .def("num_nodes", &Graph::numNodes)
      .def("num_start", &Graph::numStart)
      .def("num_accept", &Graph::numAccept)
      .def("item", &Graph::item)
      .def("arc_sort", &Graph::arcSort, "olabel"_a = false)
      .def("mark_arc_sorted", &Graph::markArcSorted, "olabel"_a = false)
      .def("ilabel_sorted", &Graph::ilabelSorted)
      .def("olabel_sorted", &Graph::olabelSorted)
      .def("weights", [](Graph& g) { return reinterpret_cast<std::uintptr_t>(g.weights()); })
      .def("weights_to_list", [](Graph& g) { return std::vector<float>(g.weights(), g.weights() + g.numArcs()); })
      .def(
          "weights_to_numpy",
          [](Graph& g) {
            py::array_t<float> out(g.numArcs());
            std::memcpy(out.mutable_data(), g.weights(), sizeof(float) * g.numArcs());
            return out;
          })
      .def(
          "set_weights",
          [](Graph& g, std::uintptr_t ptr) { g.setWeights(reinterpret_cast<const float*>(ptr)); }, "weights"_a)
      .def(
          "set_weights",
          [](Graph& g, const std::vector<float>& w) {
            if (w.size() != g.numArcs()) throw std::invalid_argument("[Graph.set_weights] wrong number of weights");
            g.setWeights(w.data());
          },
          "weights"_a)
      .def(
          "set_weights",
          [](Graph& g, py::array_t<float, py::array::c_style | py::array::forcecast> w) {
            if ((size_t)w.size() != g.numArcs())
              throw std::invalid_argument("[Graph.set_weights] wrong number of weights");
            g.setWeights(w.data());
          },
          "weights"_a)
      .def("labels_to_list", &Graph::labelsToVector, "ilabel"_a = true)
      .def("calc_grad", &Graph::calcGrad)
      .def_property("calc_grad", &Graph::calcGrad, &Graph::setCalcGrad)
      .def("is_grad_available", &Graph::isGradAvailable)
      .def("grad", (Graph & (Graph::*)()) & Graph::grad, py::return_value_policy::reference_internal)
      .def("zero_grad", &Graph::zeroGrad)
      .def("is_start", &Graph::isStart)
      .def("is_accept", &Graph::isAccept)
      .def("make_accept", &Graph::makeAccept)
      .def("src_node", &Graph::srcNode)
      .def("dst_node", &Graph::dstNode)
      .def("ilabel", &Graph::ilabel)
      .def("olabel", &Graph::olabel)
      .def("label", &Graph::label)
      .def("weight", &Graph::weight)
      .def("set_weight", &Graph::setWeight)
      .def("num_in", &Graph::numIn)
      .def("num_out", &Graph::numOut)
      .def("is_linear", &Graph::isLinear)
      .def("is_device_resident", &Graph::isDeviceResident)
      .def("__str__", [](const Graph& g) {
        std::ostringstream os;
        saveTxt(os, g);
        return os.str();
      })
      .def("__repr__", [](const Graph& g) {
        std::ostringstream os;
        os << g; // abbreviated for large graphs (utils.cpp:378-381)
        return os.str();
      });

  // functions: single graph + list overloads (bindings/python/gtn/_functions.cpp)
  m.def("negate", unary(negate), "g"_a);
  m.def("negate", unaryList(negate), "graphs"_a);
  m.def("add", binary(add), "g1"_a, "g2"_a);
  m.def("add", binaryList(add), "graphs1"_a, "graphs2"_a);
  m.def("subtract", binary(subtract), "g1"_a, "g2"_a);
  m.def("subtract", binaryList(subtract), "graphs1"_a, "graphs2"_a);
  m.def("compose", binary(static_cast<Graph (*)(const Graph&, const Graph&)>(&compose)), "g1"_a, "g2"_a);
  m.def(
      "compose",
      [](const std::vector<Graph>& a, const std::vector<Graph>& b) {
        py::gil_scoped_release release;
        return compose(a, b); // one packed launch for the whole list where the graphs allow it (gtn/batched.cpp)
      },
      "graphs1"_a, "graphs2"_a);
  m.def("intersect", binary(static_cast<Graph (*)(const Graph&, const Graph&)>(&intersect)), "g1"_a, "g2"_a);
  m.def(
      "intersect",
      [](const std::vector<Graph>& a, const std::vector<Graph>& b) {
        py::gil_scoped_release release;
        return intersect(a, b);
      },
      "graphs1"_a, "graphs2"_a);
  m.def("forward_score", unary(static_cast<Graph (*)(const Graph&)>(&forwardScore)), "g"_a);
  m.def(
      "forward_score",
      [](const std::vector<Graph>& gs) {
        py::gil_scoped_release release;
        return forwardScore(gs);
      },
      "graphs"_a);
  m.def("viterbi_score", unary(static_cast<Graph (*)(const Graph&)>(&viterbiScore)), "g"_a);
  m.def(
      "viterbi_score",
      [](const std::vector<Graph>& gs) {
        py::gil_scoped_release release;
        return viterbiScore(gs);
      },
      "graphs"_a);
  m.def("viterbi_path", unary(static_cast<Graph (*)(const Graph&)>(&viterbiPath)), "g"_a);
  m.def(
      "viterbi_path",
      [](const std::vector<Graph>& gs) {
        py::gil_scoped_release release;
        return viterbiPath(gs); // one decoding launch for the entries of one batched lattice (gtn/batched.cpp)
      },
      "graphs"_a);
  m.def("project_input", unary(projectInput), "g"_a);
  m.def("project_output", unary(projectOutput), "g"_a);
  m.def(
      "clone",
      [](const Graph& g, Projection p) {
        py::gil_scoped_release release;
        return clone(g, p);
      },
      "g"_a, "projection"_a = Projection::NONE);
  m.def("project_input", unaryList(projectInput), "graphs"_a);
  m.def("project_output", unaryList(projectOutput), "graphs"_a);
  using G = Graph;
  using GV = std::vector<Graph>;
  m.def("concat", binary(static_cast<G (*)(const G&, const G&)>(&concat)), "g1"_a, "g2"_a);
  m.def("concat", binaryList(static_cast<G (*)(const G&, const G&)>(&concat)), "graphs1"_a, "graphs2"_a);
  m.def(
      "concat",
      [](const GV& graphs) {
        py::gil_scoped_release release;
        return concat(graphs);
      },
      "graphs"_a);
  m.def(
      "concat",
      [](const std::vector<GV>& graphs) {
        py::gil_scoped_release release;
        return parallelMap(static_cast<G (*)(const GV&)>(&concat), graphs);
      },
      "graphs"_a);
  m.def("closure", unary(closure), "g"_a);
  m.def("closure", unaryList(closure), "graphs"_a);
  m.def(
      "union",
      [](const GV& graphs) {
        py::gil_scoped_release release;
        return union_(graphs);
      },
      "graphs"_a);
  m.def(
      "union",
      [](const std::vector<GV>& graphs) {
        py::gil_scoped_release release;
        return parallelMap(union_, graphs);
      },
      "graphs"_a);
  m.def(
      "remove",
      [](const G& g, int label) {
        py::gil_scoped_release release;
        return remove(g, label);
      },
      "g"_a, "label"_a = epsilon);
  m.def(
      "remove",
      [](const G& g, int ilabel, int olabel) {
        py::gil_scoped_release release;
        return remove(g, ilabel, olabel);
      },
      "g"_a, "ilabel"_a, "olabel"_a);
  m.def(
      "remove",
      [](const GV& graphs, const std::vector<int>& labels) {
        py::gil_scoped_release release;
        return parallelMap(static_cast<G (*)(const G&, int)>(&remove), graphs, labels);
      },
      "graphs"_a, "labels"_a = std::vector<int>{epsilon});

  // autograd (bindings/python/gtn/_autograd.cpp)
  m.def(
      "backward",
      [](Graph g, bool retain) {
        py::gil_scoped_release release;
        backward(g, retain);
      },
      "g"_a, "retain_graph"_a = false);
  m.def(
      "backward",
      [](Graph g, const Graph& grad, bool retain) {
        py::gil_scoped_release release;
        backward(g, grad, retain);
      },
      "g"_a, "grad"_a, "retain_graph"_a = false);
  m.def(
      "backward",
      [](std::vector<Graph> graphs, const std::vector<int>& retain) {
        py::gil_scoped_release release;
        bool uniform = !retain.empty();
        for (int r : retain) uniform = uniform && (r != 0) == (retain[0] != 0);
        if (uniform && (retain.size() == 1 || retain.size() == graphs.size()))
          backward(graphs, retain[0] != 0); // batched tapes are walked in this thread (gtn/batched.cpp)
        else
          parallelMap([](Graph g, int keep) { backward(g, keep != 0); }, graphs, retain);
      },
      "graphs"_a, "retain_graphs"_a = std::vector<int>({0}));
  m.def(
      "backward",
      [](std::vector<Graph> graphs, const std::vector<Graph>& grads, const std::vector<int>& retain) {
        py::gil_scoped_release release;
        parallelMap([](Graph g, const Graph& grad, int keep) { backward(g, grad, keep != 0); }, graphs, grads,
                    retain);
      },
      "graphs"_a, "grads"_a, "retain_graphs"_a = std::vector<int>({0}));

  // addition: kernels launched so far by the calling thread's context (tests / bench bookkeeping)
  // test / tuning hooks (not part of the reference's surface)
  m.def("compose_device_policy", []() { return detail::composeDevicePolicy(); });
  m.def("set_compose_device_policy", [](int p) { detail::setComposeDevicePolicy(p); }, "policy"_a);
  m.def("arc_lists", [](const Graph& g) {
    detail::ViewStorage vs;
    detail::makeView(g, vs);
    auto arr = [](const std::vector<int32_t>& v) { return py::array_t<int32_t>((py::ssize_t)v.size(), v.data()); };
    py::dict d;
    d["in_ptr"] = arr(vs.inPtr);
    d["in_arcs"] = arr(vs.inArcs);
    d["out_ptr"] = arr(vs.outPtr);
    d["out_arcs"] = arr(vs.outArcs);
    d["start"] = arr(vs.start);
    d["accept"] = arr(vs.accept);
    d["flags"] = py::array_t<uint8_t>((py::ssize_t)vs.flags.size(), vs.flags.data());
    d["src"] = arr(vs.src);
    d["dst"] = arr(vs.dst);
    d["ilabel"] = arr(vs.il);
    d["olabel"] = arr(vs.ol);
    d["weights"] = py::array_t<float>((py::ssize_t)vs.w.size(), vs.w.data());
    return d;
  }, "g"_a);
  m.def("device_launch_count", []() {
    auto c = detail::threadContext();
    return (long long)gtnb_ctx_launch_count(c->ctx);
  });

  // creations (bindings/python/gtn/_creations.cpp)
  m.def("scalar_graph", &scalarGraph, "val"_a, "calc_grad"_a = true);
  m.def("linear_graph", &linearGraph, "M"_a, "N"_a, "calc_grad"_a = true);

  // parallel (bindings/python/gtn/_parallel.cpp)
  m.def(
      "parallel_for",
      [](const std::function<void(int)>& fn, const std::vector<int>& ints) {
        py::gil_scoped_release release;
        parallelMap(fn, ints);
      },
      "function"_a, "int_list"_a);

  // utils (bindings/python/gtn/_utils.cpp) and rand (_rand.cpp)
  m.def("equal", &equal, "g1"_a, "g2"_a);
  m.def("isomorphic", &isomorphic, "g1"_a, "g2"_a);
  m.def(
      "write_dot",
      [](const Graph& g, const std::string& fileName, const SymbolMap& isymbols, const SymbolMap& osymbols) {
        draw(g, fileName, isymbols, osymbols);
      },
      "g"_a, "file_name"_a, "isymbols"_a = SymbolMap(), "osymbols"_a = SymbolMap());
  m.def("load", py::overload_cast<const std::string&>(&load), "file_name"_a);
  m.def("save", py::overload_cast<const std::string&, const Graph&>(&save), "file_name"_a, "graph"_a);
  m.def("savetxt", py::overload_cast<const std::string&, const Graph&>(&saveTxt), "file_name"_a, "graph"_a);
  m.def("loadtxt", py::overload_cast<const std::string&>(&loadTxt), "file_name"_a);
  m.def(
      "sample",
      [](const Graph& g, size_t maxLength) {
        py::gil_scoped_release release;
        return sample(g, maxLength);
      },
      "g"_a, "max_length"_a = 1000);
  m.def(
      "rand_equivalent",
      [](const Graph& g1, const Graph& g2, size_t numSamples, double tol, size_t maxLength) {
        py::gil_scoped_release release;
        return randEquivalent(g1, g2, numSamples, tol, maxLength);
      },
      "g1"_a, "g2"_a, "num_samples"_a = 1000, "tol"_a = 1e-4, "max_length"_a = 1000);
  // in-memory forms of the two wire formats (not in the reference: handy for tests and for
  // shipping graphs between processes without temporary files)
  m.def("dumps", [](const Graph& g) {
    std::ostringstream os;
    saveTxt(os, g);
    return os.str();
  });
  m.def("dumpb", [](const Graph& g) {
    std::ostringstream os;
    save(os, g);
    return py::bytes(os.str());
  });
  m.def("loadb", [](const std::string& blob) {
    std::istringstream in(blob);
    return load(in);
  });
  m.def("srand", [](unsigned seed) { std::srand(seed); }, "seed"_a);
  m.def("loads", [](const std::string& s) {
    std::istringstream in(s);
    return loadTxt(in);
  });
}
