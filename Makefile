# Build of libape_b200.so (sm_90a only) and the oracle's C restatement.
# `python -c "import __graft_entry__ as g; g.build()"` runs the same commands.
NVCC      ?= nvcc
NVCCFLAGS ?= -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 \
             -Xcompiler -fPIC -Iinclude
CSRC      := $(wildcard ape_b200/csrc/*.cu)
OBJS      := $(patsubst ape_b200/csrc/%.cu,build/%.o,$(CSRC))
LIB       := ape_b200/libape_b200.so

all: $(LIB) oracle

build/%.o: ape_b200/csrc/%.cu $(wildcard ape_b200/csrc/*.cuh) include/ape_b200.h
	@mkdir -p build
	$(NVCC) $(NVCCFLAGS) -Xptxas -v -c $< -o $@ 2> build/$*.ptxas.log || (cat build/$*.ptxas.log; false)

$(LIB): $(OBJS)
	$(NVCC) -gencode arch=compute_90a,code=sm_90a -shared -o $@ $(OBJS)

oracle:
	$(MAKE) -C oracle

clean:
	rm -rf build $(LIB)
	$(MAKE) -C oracle clean

.PHONY: all oracle clean
