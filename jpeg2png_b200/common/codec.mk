# The build of one codec library (entropy, png, jpegenc, jpegopt, progressive): one .cu into one sm_90a shared object,
# kept out of libjpeg2png_b200.so, whose kernels are the solver's.  The including Makefile sets LIB,
# SRC, DEPS (its headers) and, where the library needs them, EXTRA_NVFLAGS.

NVCC    ?= /usr/local/cuda/bin/nvcc
HOSTCXX ?= $(firstword $(wildcard /usr/bin/g++) g++)

ARCH    = -gencode arch=compute_90a,code=sm_90a
NVFLAGS = $(ARCH) -O3 -lineinfo -std=c++17 -ccbin $(HOSTCXX) -Xcompiler -fPIC,-Wall -Xptxas -v $(EXTRA_NVFLAGS)
LOG     = $(SRC:.cu=.ptxas.log)

all: $(LIB)

$(LIB): $(SRC) $(DEPS) ../common/codec_host.h ../common/codec.mk
	$(NVCC) $(NVFLAGS) -shared -o $@ $(SRC) 2> $(LOG) || (cat $(LOG); exit 1)

clean:
	rm -f *.so *.ptxas.log

.PHONY: all clean
