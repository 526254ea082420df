# TEST-ONLY sm_90a builds of ge_ops.cuh (see ge.cu), with the product's compiler flags: the default field arithmetic and the
# two alternatives afc_fe.cuh keeps behind switches, as for devsim.cu.  Not part of the product.  build() runs
# `make -C tests/devsim -f ge.mk`.
NVCC ?= nvcc
SRC := ../../agentfield_b200/csrc
NVFLAGS := -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -Xcompiler -fPIC -shared $(EXTRA)
DEPS := ge.cu ge_ops.cuh devsim_ops.cuh $(SRC)/afc_common.cuh $(SRC)/afc_sha.cuh $(SRC)/afc_fe.cuh $(SRC)/afc_sc.cuh \
        $(SRC)/afc_ge.cuh $(SRC)/afc_consts.inc
LIBS := libafc_ge.so libafc_ge_foldshift.so libafc_ge_kara.so

all: $(LIBS)

libafc_ge.so: $(DEPS)
	$(NVCC) $(NVFLAGS) -o $@ ge.cu
libafc_ge_foldshift.so: $(DEPS)
	$(NVCC) $(NVFLAGS) -DAFC_FOLD_SHIFT=1 -o $@ ge.cu
libafc_ge_kara.so: $(DEPS)
	$(NVCC) $(NVFLAGS) -DAFC_FE_KARATSUBA=1 -o $@ ge.cu

clean:
	rm -f $(LIBS)
.PHONY: all clean
