# Builds the product library (sm_90a only) and the CPU oracle (test infrastructure).
NVCC ?= /usr/local/cuda/bin/nvcc
ARCH  = -gencode arch=compute_90a,code=sm_90a
NVFLAGS = $(ARCH) -O3 -std=c++17 -lineinfo -Xcompiler -fPIC,-Wall,-Wno-unused-function -Xptxas -v --expt-relaxed-constexpr
SRC = $(wildcard tinysql_b200/csrc/*.cu)
OBJ = $(patsubst tinysql_b200/csrc/%.cu,build/%.o,$(SRC))
LIB = tinysql_b200/lib/libtinysql_b200.so

all: $(LIB) oracle

HDR = $(wildcard tinysql_b200/csrc/*.cuh) include/tinysql_b200.h
build/%.o: tinysql_b200/csrc/%.cu $(HDR)
	@mkdir -p build
	$(NVCC) $(NVFLAGS) -c $< -o $@ 2> build/$*.ptxas.log || (cat build/$*.ptxas.log; exit 1)

$(LIB): $(OBJ)
	@mkdir -p tinysql_b200/lib
	$(NVCC) $(ARCH) -shared -o $@ $(OBJ) -lpthread

oracle:
	$(MAKE) -C oracle

clean:
	rm -rf build $(LIB) oracle/liboracle.so

.PHONY: all oracle clean
