# Builds the C-ABI shared library (sm_90a only).
NVCC ?= /usr/local/cuda/bin/nvcc
PKG := 2dimageto3dmodel_b200
SRCS := $(wildcard $(PKG)/csrc/*.cu)
HDRS := $(wildcard $(PKG)/csrc/*.cuh) include/b3d.h
OBJS := $(patsubst $(PKG)/csrc/%.cu,build/%.o,$(SRCS))
NVFLAGS := -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC,-fvisibility=hidden \
           --expt-relaxed-constexpr -Iinclude
LIB := $(PKG)/b3d/libb3d.so

all: $(LIB)

build/%.o: $(PKG)/csrc/%.cu $(HDRS)
	@mkdir -p build
	$(NVCC) $(NVFLAGS) -Xptxas -v -c $< -o $@ 2> build/$*.ptxas.log || (cat build/$*.ptxas.log; exit 1)

$(LIB): $(OBJS)
	$(NVCC) -shared -o $@ $(OBJS)

clean:
	rm -rf build $(LIB)
.PHONY: all clean
