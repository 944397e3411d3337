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

.PHONY: all lib probe oracle ref clean
all: lib probe oracle ref
lib: $(LIB)

# make PROF=1: the CTU driver with its phase profile (diagnostic; kvz_cuda_ctu_close prints it)
CTUFLAGS  := $(if $(PROF),-DKVZ_CTU_PROF,)

$(OBJDIR)/ctu_driver.o: $(SRCDIR)/ctu_driver.cu $(wildcard $(SRCDIR)/*.cuh) $(wildcard $(SRCDIR)/*.h) $(wildcard $(SRCDIR)/ctu/*.h) include/kvz_cuda.h include/kvz_cuda_ctu.h
	@mkdir -p $(OBJDIR)
	$(NVCC) $(NVFLAGS) $(CTUFLAGS) -c $< -o $@

$(OBJDIR)/me_search.o: $(SRCDIR)/me_search.cu $(wildcard $(SRCDIR)/*.cuh) $(wildcard $(SRCDIR)/me/*.h) include/kvz_cuda.h
	@mkdir -p $(OBJDIR)
	$(NVCC) $(NVFLAGS) -c $< -o $@

$(OBJDIR)/%.o: $(SRCDIR)/%.cu $(wildcard $(SRCDIR)/*.cuh) $(wildcard $(SRCDIR)/*.h) include/kvz_cuda.h
	@mkdir -p $(OBJDIR)
	$(NVCC) $(NVFLAGS) -c $< -o $@

$(LIB): $(OBJS)
	$(NVCC) $(ARCH) -shared -o $@ $(OBJS) -lcudart -ldl -lpthread

# test infrastructure: the CTU search driver's transform-unit jobs behind a C entry point (tests/test_ctu_tu_jobs.py),
# built with the product's flags (sm_90a) and for the host with the one-thread CTA (g++), which the device's results are
# compared with; never linked into the product library
PROBE     := tests/cuda/libkvzctu_probe.so
PROBE_HOST := tests/hostsim/libkvzctu_probe_host.so
# ... and the back half of its CTU job (deblocking, SAO search and application, model tracking) on injected decisions
# (tests/test_ctu_frame_stage.py), the same two builds
FPROBE    := tests/cuda/libkvzctu_frame_probe.so
FPROBE_HOST := tests/hostsim/libkvzctu_frame_probe_host.so
probe: $(PROBE) $(PROBE_HOST) $(FPROBE) $(FPROBE_HOST)
$(PROBE): tests/cuda/ctu_tu_probe.cu $(wildcard $(SRCDIR)/*.h) $(wildcard $(SRCDIR)/ctu/*.h)
	$(NVCC) $(ARCH) -O3 -std=c++17 -fmad=false -Xcompiler -fPIC,-Wall -shared -o $@ $< -lcudart
$(PROBE_HOST): tests/cuda/ctu_tu_probe.cu $(wildcard $(SRCDIR)/*.h) $(wildcard $(SRCDIR)/ctu/*.h)
	g++ -O2 -g -std=c++17 -fPIC -shared -ffp-contract=off -Wall -Wno-unused-function -Wno-unknown-pragmas -x c++ -o $@ $<
$(FPROBE): tests/cuda/ctu_frame_probe.cu $(wildcard $(SRCDIR)/*.h) $(wildcard $(SRCDIR)/ctu/*.h)
	$(NVCC) $(ARCH) -O3 -std=c++17 -fmad=false -Xcompiler -fPIC,-Wall -shared -o $@ $< -lcudart
$(FPROBE_HOST): tests/cuda/ctu_frame_probe.cu $(wildcard $(SRCDIR)/*.h) $(wildcard $(SRCDIR)/ctu/*.h)
	g++ -O2 -g -std=c++17 -fPIC -shared -ffp-contract=off -Wall -Wno-unused-function -Wno-unknown-pragmas -x c++ -o $@ $<

oracle:
	$(MAKE) -s -C oracle oracle
ref:
	$(MAKE) -s -C oracle ref

clean:
	rm -rf build $(LIB) $(PROBE) $(PROBE_HOST) $(FPROBE) $(FPROBE_HOST)
