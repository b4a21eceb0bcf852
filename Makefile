# bnet build: host engine (g++) + sm_90a kernels (nvcc) -> libnccl-net.so
#
#   make            build the plugin / runtime library into bagua_net_b200/lib/
#   make test       C++ unit + loopback tests (no GPU needed)
#   make bench      native benchmarks (all_reduce_perf clone, p2p_bw)
#   make sass       SASS / PTX / resource listings of every kernel -> docs/sass/
#   make tar        release tarball like the reference's `make tar`
#   make install    copy the plugin variants to $(PREFIX)/lib
#   make tsan asan emu-asan   sanitizer builds + tests (ci/run_sanitizers.sh)
#
# Counterpart of the reference build (reference: cc/Makefile:1-26): same product
# name — NCCL dlopen()s libnccl-net.so from LD_LIBRARY_PATH — but no cargo step.

CUDA_HOME ?= /usr/local/cuda
NVCC      := $(CUDA_HOME)/bin/nvcc
CXX       ?= g++
ARCH      := -gencode arch=compute_90a,code=sm_90a
OUT       := bagua_net_b200/lib
BUILD     := build

CXXFLAGS  := -O2 -g -fPIC -std=c++17 -Wall -Wno-invalid-offsetof -fvisibility=hidden -pthread \
             -Iinclude -Icsrc -I$(CUDA_HOME)/include
NVCCFLAGS := -O3 -std=c++17 $(ARCH) -lineinfo -Xcompiler -fPIC,-fvisibility=hidden,-Wno-invalid-offsetof \
             -Iinclude -Icsrc --expt-relaxed-constexpr
LDFLAGS   := -shared -cudart static -Xcompiler -pthread -ldl -lrt

HOST_SRCS := csrc/core/common.cc csrc/core/netif.cc csrc/core/telemetry.cc csrc/core/engine.cc \
             csrc/transport/tcp_threads.cc csrc/transport/tcp_async.cc csrc/transport/nvl.cc \
             csrc/cuda/cuda_iface.cc csrc/coll/transport_ring.cc csrc/coll/transport_mesh.cc csrc/plugin/tuner.cc csrc/capi.cc
CU_SRCS   := $(wildcard csrc/cuda/*.cu)

HOST_OBJS := $(patsubst csrc/%.cc,$(BUILD)/%.o,$(HOST_SRCS))
CU_OBJS   := $(patsubst csrc/%.cu,$(BUILD)/%.cu.o,$(CU_SRCS))
PLUGIN_OBJ  := $(BUILD)/plugin/plugin.o $(BUILD)/plugin/collnet.o
PLUGINX_OBJ := $(BUILD)/plugin/plugin_x.o $(BUILD)/plugin/collnet_x.o

PLUGIN_SO  := $(OUT)/libnccl-net.so
PLUGINX_SO := $(OUT)/libnccl-net-bnetx.so
ALIAS_SO   := $(OUT)/libnccl-net-bnet.so

default: $(PLUGIN_SO) $(PLUGINX_SO) $(ALIAS_SO)

$(BUILD)/%.o: csrc/%.cc
	@mkdir -p $(dir $@)
	$(CXX) $(CXXFLAGS) -MMD -MP -c $< -o $@

$(BUILD)/%.cu.o: csrc/%.cu
	@mkdir -p $(dir $@)
	$(NVCC) $(NVCCFLAGS) -MMD -MP -c $< -o $@

$(BUILD)/plugin/%_x.o: csrc/plugin/%.cc
	@mkdir -p $(dir $@)
	$(CXX) $(CXXFLAGS) -DBNET_EXPORT_V9_V10 -MMD -MP -c $< -o $@

# (link to a temporary name, then rename: a process that dlopen()s the library while another one is
#  rebuilding it never sees a half-written file)
$(PLUGIN_SO): $(HOST_OBJS) $(CU_OBJS) $(PLUGIN_OBJ)
	@mkdir -p $(OUT)
	$(NVCC) $(ARCH) $(LDFLAGS) -o $@.tmp $^ && mv -f $@.tmp $@

# same engine, additionally exports the v9/v10 tables (select with NCCL_NET_PLUGIN=bnetx)
$(PLUGINX_SO): $(HOST_OBJS) $(CU_OBJS) $(PLUGINX_OBJ)
	@mkdir -p $(OUT)
	$(NVCC) $(ARCH) $(LDFLAGS) -o $@.tmp $^ && mv -f $@.tmp $@

# NCCL_NET_PLUGIN=bnet  ->  libnccl-net-bnet.so ;  NCCL_TUNER_PLUGIN=bnet  ->  libnccl-tuner-bnet.so (same library)
$(ALIAS_SO): $(PLUGIN_SO)
	cp -f $< $@.tmp && mv -f $@.tmp $@
	ln -sf libnccl-net-bnet.so $(OUT)/libnccl-tuner-bnet.so

TEST_BINS := $(BUILD)/tests/unit_tests $(BUILD)/tests/loopback_test
$(BUILD)/tests/%: csrc/tests/%.cc $(PLUGIN_SO)
	@mkdir -p $(dir $@)
	$(CXX) $(CXXFLAGS) -fvisibility=default $< -o $@ -ldl -pthread

# the per-thread bodies of the device kernels (fused layers, transport executor), compiled by g++ and walked
# over an emulated grid / cluster
EMU_FLAGS := -O2 -g -std=c++17 -Wall -Wno-unknown-pragmas -fno-strict-aliasing -Icsrc -I$(CUDA_HOME)/include
$(BUILD)/tests/nn_emu_test: csrc/tests/nn_emu_test.cc csrc/cuda/nn_body.cuh
	@mkdir -p $(dir $@)
	$(CXX) $(EMU_FLAGS) $< -o $@
$(BUILD)/tests/exec_emu_test: csrc/tests/exec_emu_test.cc csrc/cuda/exec_body.cuh
	@mkdir -p $(dir $@)
	$(CXX) $(EMU_FLAGS) $< -o $@
# the wgmma linear kernel's index logic on an emulated TMA / MMA / accumulator
$(BUILD)/tests/tc_emu_test: csrc/tests/tc_emu_test.cc csrc/cuda/tc_body.cuh include/bnet/bnet_tc.h
	@mkdir -p $(dir $@)
	$(CXX) $(EMU_FLAGS) -Iinclude $< -o $@
# the fused SGD and AdamW kernels' per-element updates against long-double SGD and AdamW
$(BUILD)/tests/optim_emu_test: csrc/tests/optim_emu_test.cc csrc/cuda/optim_body.cuh
	@mkdir -p $(dir $@)
	$(CXX) $(EMU_FLAGS) $< -o $@

# the parameter-group lookup of the fused optimizer kernels against a brute-force map
$(BUILD)/tests/group_lookup_test: csrc/tests/group_lookup_test.cc csrc/cuda/optim_body.cuh
	@mkdir -p $(dir $@)
	$(CXX) $(EMU_FLAGS) $< -o $@

# the same emulation tests under Address/UB sanitizers: an out-of-bounds or misaligned access of a kernel body
# is caught here, on the CPU, instead of poisoning a CUDA context
emu-asan: csrc/tests/nn_emu_test.cc csrc/tests/exec_emu_test.cc csrc/tests/tc_emu_test.cc csrc/tests/optim_emu_test.cc csrc/cuda/nn_body.cuh csrc/cuda/exec_body.cuh csrc/cuda/tc_body.cuh csrc/cuda/optim_body.cuh
	@mkdir -p $(BUILD)/asan/tests
	$(SAN_CXX) $(EMU_FLAGS) -O1 -w $(SAN_FLAGS_asan) csrc/tests/nn_emu_test.cc -o $(BUILD)/asan/tests/nn_emu_test
	$(SAN_CXX) $(EMU_FLAGS) -O1 -w $(SAN_FLAGS_asan) csrc/tests/exec_emu_test.cc -o $(BUILD)/asan/tests/exec_emu_test
	$(SAN_CXX) $(EMU_FLAGS) -Iinclude -O1 -w $(SAN_FLAGS_asan) csrc/tests/tc_emu_test.cc -o $(BUILD)/asan/tests/tc_emu_test
	$(SAN_CXX) $(EMU_FLAGS) -O1 -w $(SAN_FLAGS_asan) csrc/tests/optim_emu_test.cc -o $(BUILD)/asan/tests/optim_emu_test
	$(BUILD)/asan/tests/nn_emu_test
	$(BUILD)/asan/tests/exec_emu_test
	$(BUILD)/asan/tests/tc_emu_test
	$(BUILD)/asan/tests/optim_emu_test

test: $(TEST_BINS) $(BUILD)/tests/nn_emu_test $(BUILD)/tests/exec_emu_test $(BUILD)/tests/tc_emu_test $(BUILD)/tests/optim_emu_test \
      $(BUILD)/tests/group_lookup_test
	$(BUILD)/tests/unit_tests $(PLUGIN_SO)
	$(BUILD)/tests/loopback_test $(PLUGIN_SO)
	$(BUILD)/tests/nn_emu_test
	$(BUILD)/tests/exec_emu_test
	$(BUILD)/tests/tc_emu_test
	$(BUILD)/tests/optim_emu_test
	$(BUILD)/tests/group_lookup_test

BENCH_BINS := $(BUILD)/bench/all_reduce_perf
NCCL_HOME ?= $(shell python -c "import nvidia.nccl, os; print(os.path.dirname(nvidia.nccl.__file__))" 2>/dev/null)
$(BUILD)/bench/%: bench/%.cu $(PLUGIN_SO)
	@mkdir -p $(dir $@)
	$(NVCC) -O3 -std=c++17 $(ARCH) -lineinfo -Iinclude -Icsrc -I$(NCCL_HOME)/include $< -o $@ \
	    -L$(NCCL_HOME)/lib -l:libnccl.so.2 -Xlinker -rpath=$(NCCL_HOME)/lib -ldl -lpthread -lrt

# host-only transport benchmark (no GPU, no NCCL): loopback TCP / shared-memory ring through the v8 table
$(BUILD)/bench/net_perf: bench/net_perf.cc $(PLUGIN_SO)
	@mkdir -p $(dir $@)
	$(CXX) $(CXXFLAGS) -fvisibility=default $< -o $@ -ldl -pthread

bench: $(BENCH_BINS) $(BUILD)/bench/net_perf

sass: $(PLUGIN_SO)
	@mkdir -p docs/sass
	for f in $(CU_SRCS); do b=$$(basename $$f .cu); \
	  $(NVCC) $(NVCCFLAGS) -Xptxas -v -cubin $$f -o $(BUILD)/$$b.cubin 2> docs/sass/$$b.ptxas.txt; \
	  $(CUDA_HOME)/bin/cuobjdump -sass $(BUILD)/$$b.cubin > docs/sass/$$b.sass; done

tar: default
	tar czf bagua-net-b200_x86_64.tar.gz -C $(OUT) libnccl-net.so libnccl-net-bnet.so libnccl-net-bnetx.so

# `make install PREFIX=/opt/bnet` puts the three plugin variants where LD_LIBRARY_PATH can find them
PREFIX ?= /usr/local
install: default
	install -d $(PREFIX)/lib
	install -m 0755 $(PLUGIN_SO) $(ALIAS_SO) $(PLUGINX_SO) $(PREFIX)/lib/
uninstall:
	rm -f $(PREFIX)/lib/libnccl-net.so $(PREFIX)/lib/libnccl-net-bnet.so $(PREFIX)/lib/libnccl-net-bnetx.so

clean:
	rm -rf $(BUILD) $(OUT)/*.so

# (the two plugin objects too: a header change that moves a vtable slot must rebuild the ABI shims with it)
-include $(HOST_OBJS:.o=.d) $(CU_OBJS:.o=.d) $(PLUGIN_OBJ:.o=.d) $(PLUGINX_OBJ:.o=.d)
.PHONY: default test bench sass tar clean emu-asan install uninstall

# ---- sanitizer builds of the host engine (SURVEY §5.2): `make tsan` / `make asan` rebuild every host
# object with the sanitizer into build/<san>/, link it with the (uninstrumented) kernel objects and run the
# C++ unit + loopback tests against that library.
SAN_CXX ?= /usr/bin/g++
SAN_FLAGS_tsan := -fsanitize=thread -Wno-tsan
SAN_FLAGS_asan := -fsanitize=address -fsanitize=undefined -fno-omit-frame-pointer
define SAN_RULES
$(BUILD)/$(1)/%.o: csrc/%.cc
	@mkdir -p $$(dir $$@)
	$(SAN_CXX) $(CXXFLAGS) -O1 -DBNET_EXPORT_V9_V10 $$(SAN_FLAGS_$(1)) -MMD -MP -c $$< -o $$@
$(BUILD)/$(1)/libnccl-net.so: $(patsubst csrc/%.cc,$(BUILD)/$(1)/%.o,$(HOST_SRCS) csrc/plugin/plugin.cc csrc/plugin/collnet.cc) $(CU_OBJS)
	$(NVCC) -ccbin $(SAN_CXX) $(ARCH) $(LDFLAGS) $$(addprefix -Xcompiler ,$$(SAN_FLAGS_$(1))) -o $$@ $$^
$(BUILD)/$(1)/tests/%: csrc/tests/%.cc $(BUILD)/$(1)/libnccl-net.so
	@mkdir -p $$(dir $$@)
	$(SAN_CXX) $(CXXFLAGS) -O1 $$(SAN_FLAGS_$(1)) -fvisibility=default $$< -o $$@ -ldl -pthread
-include $(patsubst csrc/%.cc,$(BUILD)/$(1)/%.d,$(HOST_SRCS) csrc/plugin/plugin.cc csrc/plugin/collnet.cc)
$(1): $(BUILD)/$(1)/tests/unit_tests $(BUILD)/$(1)/tests/loopback_test
	$(BUILD)/$(1)/tests/unit_tests $(BUILD)/$(1)/libnccl-net.so
	$(BUILD)/$(1)/tests/loopback_test $(BUILD)/$(1)/libnccl-net.so
.PHONY: $(1)
endef
$(eval $(call SAN_RULES,tsan))
$(eval $(call SAN_RULES,asan))
