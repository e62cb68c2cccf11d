#!/usr/bin/env python
"""Offline build of the UNMODIFIED reference (/root/reference, HugeCTR v25.03) for `bench.py --impl reference`.

The reference is a CMake project whose configure step downloads pybind11 (`HugeCTR/src/CMakeLists.txt:21-35`)
and links libaio / libnuma / tbb, none of which exist in this image, so `pip install /root/reference` and a
stock `cmake` both fail (DESIGN.md section 4).  This script does what that CMake tree does, with nothing
fetched: it globs the same source lists (`HugeCTR/core23/CMakeLists.txt`, `HugeCTR/embedding/CMakeLists.txt`,
`gpu_cache/src/CMakeLists.txt`, `HugeCTR/src/CMakeLists.txt` with `-DDISABLE_CUDF=ON -DSM=90`), compiles them
straight from the read-only tree with the same definitions and language flags, and links the same four
libraries plus the `hugectr` pybind11 module into `baseline/_ref/`.  No reference source file is edited.
Substitutions, all on the build side:
  * pybind11 headers come from the local Python environment instead of FetchContent;
  * `baseline/shim/{libaio,numa,numaif}.h` stand in for the two missing system packages (libaio = the five
    raw AIO syscalls; numa = single-node no-ops); tbb is only on the link line, no symbol of it is used;
  * `config.hpp` (configure_file output) is generated into the build directory;
  * `-Werror` is dropped (newer gcc / nvcc than the reference pins).

Usage: python baseline/build_reference.py [--jobs N] [--build-dir DIR] ; idempotent (ninja).
"""
import argparse
import glob
import os
import subprocess
import sys
import sysconfig

REF = "/root/reference"
HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_ref")


def rel_glob(base, pats, recursive=False):
    out = []
    for p in pats:
        out += glob.glob(os.path.join(base, p), recursive=recursive)
    return sorted(set(os.path.normpath(f) for f in out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--jobs", type=int, default=os.cpu_count())
    ap.add_argument("--build-dir", default="/tmp/hctr_ref_build")
    ap.add_argument("--only", default="", help="comma list of libs to build (core23,embedding,gpu_cache,shared,module)")
    args = ap.parse_args()
    bd = args.build_dir
    os.makedirs(bd + "/gen", exist_ok=True)
    os.makedirs(OUT, exist_ok=True)
    with open(bd + "/gen/config.hpp", "w") as f:
        f.write('#pragma once\n#include <string>\nnamespace HugeCTR {\n'
                f'const static std::string PROJECT_HOME_ = "{REF}/test/";\n}}\n')
    # empty link stubs so DT_NEEDED entries resolve on the GPU box (driver libs are absent here)
    stub = bd + "/stub"
    os.makedirs(stub, exist_ok=True)
    open(stub + "/e.c", "w").write("")
    subprocess.check_call(["gcc", "-shared", "-fPIC", "-Wl,-soname,libnvidia-ml.so.1", stub + "/e.c", "-o",
                           stub + "/libnvidia-ml.so"])

    import pybind11
    H = REF + "/HugeCTR"
    inc = [bd + "/gen", HERE + "/shim", REF, REF + "/test", H + "/include", H,
           REF + "/third_party/cuml/cpp", REF + "/third_party/cuml/cpp/include",
           REF + "/third_party/cuml/cpp/src_prims", REF + "/third_party", REF + "/third_party/argparse/include",
           REF + "/third_party/cpptqdm", REF + "/third_party/json/single_include",
           REF + "/third_party/parallel-hashmap", REF + "/gpu_cache/include",
           REF + "/third_party/dynamic_embedding_table",
           REF + "/third_party/dynamic_embedding_table/cuCollections/include",
           REF + "/third_party/HierarchicalKV/include", "/usr/local/cuda/include",
           "/usr/include/x86_64-linux-gnu", pybind11.get_include(), sysconfig.get_paths()["include"]]
    incf = " ".join("-I" + i for i in inc)
    defs = "-DDISABLE_CUDF -DLIBCUDACXX_ENABLE_EXPERIMENTAL_MEMORY_RESOURCE -DNDEBUG"
    cxxflags = f"-std=c++17 -O3 -fPIC -fopenmp -Wno-sign-compare -Wno-deprecated-declarations {defs} {incf}"
    cuflags = (f"-std=c++17 -O3 -gencode arch=compute_90,code=sm_90 --expt-extended-lambda "
               f"--expt-relaxed-constexpr -Xcompiler -fPIC,-fopenmp -Xcudafe --diag_suppress=177 "
               f"-w {defs} {incf}")

    core23 = [H + "/core23/" + f for f in """allocator_factory.cpp allocator_params.cpp buffer.cpp buffer_client.cpp
        buffer_channel.cpp buffer_channel_helpers.cpp buffer_factory.cpp buffer_params.cpp device.cpp device_guard.cpp
        device_type.cpp data_type.cpp offsetted_buffer.cpp low_level_primitives.cpp low_level_primitives.cu
        mpi_init_service.cpp details/simple_cuda_allocator.cpp details/managed_cuda_allocator.cpp
        details/low_level_cuda_allocator.cpp details/pool_cuda_allocator.cpp details/pinned_host_allocator.cpp
        details/new_delete_allocator.cpp details/unitary_buffer.cpp details/confederal_buffer.cpp
        details/tensor_impl.cpp details/tensor_helpers.cpp details/host_launch_helpers.cpp tensor.cpp
        tensor_operations.cpp kernel_params.cpp shape.cpp logger.cpp""".split()]
    core23 = [f for f in core23 if os.path.exists(f)]
    emb = rel_glob(H + "/embedding", ["*.cpp", "*.cu", "operators/*.cpp", "operators/*.cu", "data_distributor/*.cpp",
                                      "data_distributor/*.cu", "gpu_barrier/*.cpp", "gpu_barrier/*.cu"])
    gcache = [REF + "/gpu_cache/src/" + f for f in
              ("nv_gpu_cache.cu", "static_table.cu", "static_hash_table.cu", "uvm_table.cu")]
    shared = rel_glob(H + "/src", ["**/*.cpp", "**/*.cu"], recursive=True)
    shared += rel_glob(H + "/embedding_storage", ["**/*.cpp", "**/*.cu"], recursive=True)
    shared += rel_glob(REF + "/third_party/dynamic_embedding_table", ["**/*.cpp", "**/*.cu"], recursive=True)
    drop = {"pybind/module_main.cpp", "inference_benchmark/metrics.cpp", "data_readers/file_source_parquet.cpp",
            "data_readers/metadata.cpp", "data_readers/parquet_data_reader_worker.cpp",
            "data_readers/row_group_reading_thread.cpp", "data_readers/dataframe_container.cu",
            "data_readers/parquet_data_converter.cu"}
    shared = sorted(set(f for f in shared if os.path.relpath(f, H + "/src") not in drop))
    module = [H + "/src/pybind/module_main.cpp"]

    L = ["rule cxx", f"  command = g++ {cxxflags} -MMD -MF $out.d -c $in -o $out", "  depfile = $out.d",
         "  description = CXX $in",
         "rule cu", f"  command = nvcc {cuflags} -MD -MF $out.d -c $in -o $out", "  depfile = $out.d",
         "  description = NVCC $in",
         "rule link", "  command = g++ -shared -fopenmp -o $out $in $libs -Wl,-rpath,'$$ORIGIN'",
         "  description = LINK $out", ""]

    def objs(name, srcs):
        o = []
        for s in srcs:
            ob = f"{bd}/obj/{name}/" + os.path.relpath(s, REF).replace("/", "__") + ".o"
            L.append(f"build {ob}: {'cu' if s.endswith('.cu') else 'cxx'} {s}")
            o.append(ob)
        return o

    cuda_l = "-L/usr/local/cuda/lib64 -L/usr/local/cuda/lib64/stubs"
    libs = {}
    libs["core23"] = (OUT + "/libhugectr_core23.so", objs("core23", core23), f"{cuda_l} -lcuda -lcudart -lcurand")
    libs["embedding"] = (OUT + "/libembedding.so", objs("embedding", emb),
                         f"{cuda_l} -L{OUT} -lcudart -lnccl -lhugectr_core23")
    libs["gpu_cache"] = (OUT + "/libgpu_cache.so", objs("gpu_cache", gcache), f"{cuda_l} -lcudart")
    libs["shared"] = (OUT + "/libhuge_ctr_shared.so", objs("shared", shared),
                      f"{cuda_l} -L{OUT} -L{stub} -lhugectr_core23 -lembedding -lgpu_cache -lcuda -lcudart "
                      f"-lcublasLt -lcublas -lcurand -lnvidia-ml -lcudnn -lnccl -lpthread -lstdc++fs")
    libs["module"] = (OUT + "/hugectr.so", objs("module", module), f"-L{OUT} -lhuge_ctr_shared")
    dep = {"embedding": ["core23"], "shared": ["core23", "embedding", "gpu_cache"], "module": ["shared"]}
    for k, (out, ob, l) in libs.items():
        d = " ".join(libs[x][0] for x in dep.get(k, []))
        L.append(f"build {out}: link {' '.join(ob)}" + (f" | {d}" if d else ""))
        L.append(f"  libs = {l}")
    open(bd + "/build.ninja", "w").write("\n".join(L) + "\n")
    targets = [libs[k][0] for k in (args.only.split(",") if args.only else libs)]
    print(f"{len(core23)} core23, {len(emb)} embedding, {len(gcache)} gpu_cache, {len(shared)} shared sources",
          flush=True)
    rc = subprocess.call(["ninja", "-C", bd, "-j", str(args.jobs), "-k", "0"] + targets)
    sys.exit(rc)


if __name__ == "__main__":
    main()
