"""In-tree build: `python setup.py build_ext --inplace` compiles the sm_90a kernel library and the
host runtime into hugectr_b200/lib (same as `python __graft_entry__.py`)."""
from setuptools import Command, find_packages, setup


class BuildNative(Command):
    description = "compile libhctr_cuda.so (nvcc, sm_90a) and libhctr_host.so (g++)"
    user_options = [("inplace", "i", "kept for setuptools compatibility"), ("force", "f", "rebuild")]

    def initialize_options(self):
        self.inplace, self.force = 1, 0

    def finalize_options(self):
        pass

    def run(self):
        from hugectr_b200 import _native
        _native.build(force=bool(self.force), verbose=True)


setup(name="hugectr_b200", version="25.3.1", packages=find_packages(include=["hugectr_b200*", "hugectr", "hugectr2onnx"]),
      package_data={"hugectr_b200": ["csrc/*", "csrc/host/*", "lib/*.so"]},
      cmdclass={"build_ext": BuildNative}, python_requires=">=3.10")
