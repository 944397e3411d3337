# Builds the product library kvazaar_b200/libkvzcuda.so (H100, sm_90a only) and, via oracle/Makefile, the test oracles.
NVCC      ?= nvcc
ARCH      := -gencode arch=compute_90a,code=sm_90a
# -fmad=false: cost arithmetic must not be contracted into FMAs (SURVEY.md H3); everything else is integer.
NVFLAGS   := $(ARCH) -O3 -lineinfo -std=c++17 -fmad=false -Xcompiler -fPIC,-Wall -Iinclude
SRCDIR    := kvazaar_b200/csrc
OBJDIR    := build/obj
SRCS      := $(wildcard $(SRCDIR)/*.cu)
OBJS      := $(patsubst $(SRCDIR)/%.cu,$(OBJDIR)/%.o,$(SRCS))
LIB       := kvazaar_b200/libkvzcuda.so

.PHONY: all lib oracle ref clean
all: lib oracle ref
lib: $(LIB)

# make PROF=1: the CTU driver with its phase profile (diagnostic; kvz_cuda_ctu_close prints it)
CTUFLAGS  := $(if $(PROF),-DKVZ_CTU_PROF,)

$(OBJDIR)/ctu_driver.o: $(SRCDIR)/ctu_driver.cu $(wildcard $(SRCDIR)/*.cuh) $(wildcard $(SRCDIR)/ctu/*.h) include/kvz_cuda.h include/kvz_cuda_ctu.h
	@mkdir -p $(OBJDIR)
	$(NVCC) $(NVFLAGS) $(CTUFLAGS) -c $< -o $@

$(OBJDIR)/me_search.o: $(SRCDIR)/me_search.cu $(wildcard $(SRCDIR)/*.cuh) $(wildcard $(SRCDIR)/me/*.h) include/kvz_cuda.h
	@mkdir -p $(OBJDIR)
	$(NVCC) $(NVFLAGS) -c $< -o $@

$(OBJDIR)/%.o: $(SRCDIR)/%.cu $(wildcard $(SRCDIR)/*.cuh) include/kvz_cuda.h
	@mkdir -p $(OBJDIR)
	$(NVCC) $(NVFLAGS) -c $< -o $@

$(LIB): $(OBJS)
	$(NVCC) $(ARCH) -shared -o $@ $(OBJS) -lcudart -ldl -lpthread

oracle:
	$(MAKE) -s -C oracle oracle
ref:
	$(MAKE) -s -C oracle ref

clean:
	rm -rf build $(LIB)
