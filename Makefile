# Build of the H100 BWA-MEM path.
#   make            -> bwa_b200/libbwa_b200.so (host glue in C + sm_90a CUDA kernels) and bwa_b200/bwa-b200 (CLI)
#   make oracle     -> oracle/_build/liboracle.so, oracle/_ref/* (needs /root/reference or a prebuilt _ref)
#   make testbin    -> tests/_build/bwa-b200-oracle : host glue linked against the CPU oracle stages (TEST ONLY)
#   make tsan       -> tests/_build/bwa-b200-tsan : the same host glue + oracle stages under ThreadSanitizer (TEST ONLY)
#   make cusim      -> tests/_build/libbwa_b200_cusim.so : the CUDA kernels compiled for the CPU SIMT emulator (TEST ONLY)
#   make asan       -> tests/_build/bwa-b200-cusim-asan : emulated kernels + host glue under AddressSanitizer (TEST ONLY)
NVCC  ?= /usr/local/cuda/bin/nvcc
CC    ?= gcc
CXX   ?= g++
HOST  := bwa_b200/csrc/host
CUDA  := bwa_b200/csrc/cuda
CFLAGS := -O2 -g -Wall -Wno-unused-function -fPIC -Iinclude -I$(HOST) -pthread
NVFLAGS := $(NVEXTRA) -O3 -lineinfo -std=c++17 -gencode arch=compute_90a,code=sm_90a -Xcompiler -fPIC,-Wall,-Wno-unused-function -Iinclude -I$(CUDA)
HOST_SRC := $(filter-out $(HOST)/bb_cli.c,$(wildcard $(HOST)/*.c))
HOST_OBJ := $(patsubst $(HOST)/%.c,build/host/%.o,$(HOST_SRC))
CUDA_SRC := $(wildcard $(CUDA)/*.cu)
CUDA_OBJ := $(patsubst $(CUDA)/%.cu,build/cuda/%.o,$(CUDA_SRC))
CUDA_HDR := $(wildcard $(CUDA)/*.cuh) $(wildcard $(CUDA)/*.h) $(wildcard include/*.h)

all: bwa_b200/libbwa_b200.so bwa_b200/bwa-b200

build/host/%.o: $(HOST)/%.c $(wildcard $(HOST)/*.h) $(wildcard include/*.h)
	@mkdir -p build/host
	$(CC) $(CFLAGS) -c $< -o $@

build/cuda/%.o: $(CUDA)/%.cu $(CUDA_HDR)
	@mkdir -p build/cuda
	$(NVCC) $(NVFLAGS) -c $< -o $@
# stage 4 decides integers (MAPQ, pair scores) from double expressions that must round as the host's do: no a*b+c contraction
build/cuda/bwag_tail.o: $(CUDA)/bwag_tail.cu $(CUDA_HDR)
	@mkdir -p build/cuda
	$(NVCC) $(NVFLAGS) -fmad=false -c $< -o $@

bwa_b200/libbwa_b200.so: $(HOST_OBJ) build/host/bb_cli.o $(CUDA_OBJ)
	$(NVCC) -shared -o $@ $^ -lz -lm -lpthread -cudart shared

build/host/bb_main.o: $(HOST)/bb_cli.c
	@mkdir -p build/host
	$(CC) $(CFLAGS) -DBB_MAIN -c $< -o $@

bwa_b200/bwa-b200: build/host/bb_main.o bwa_b200/libbwa_b200.so
	$(CC) -o $@ build/host/bb_main.o $(filter-out build/host/bb_cli.o,$(HOST_OBJ)) $(CUDA_OBJ) -L/usr/local/cuda/lib64 -lcudart -lstdc++ -lz -lm -lpthread -Wl,-rpath,/usr/local/cuda/lib64

oracle:
	$(MAKE) -C oracle all

# ---- test-only artefacts ----
testbin: tests/_build/bwa-b200-oracle
tests/_build/bwa-b200-oracle: $(HOST_OBJ) build/host/bb_main.o oracle/oracle_fm.c oracle/oracle_sw.c oracle/oracle_stages.c tests/oracle_index.c tests/oracle_index_steps.c tests/oracle_maxk.c tests/oracle_fastmap.c tests/oracle_aln.c tests/oracle_samse.c tests/oracle_sampe.c tests/oracle_pemerge.c
	@mkdir -p tests/_build
	$(CC) $(CFLAGS) -O3 -Ioracle -o $@ build/host/bb_main.o $(HOST_OBJ) oracle/oracle_fm.c oracle/oracle_sw.c oracle/oracle_stages.c tests/oracle_index.c tests/oracle_index_steps.c tests/oracle_maxk.c tests/oracle_fastmap.c tests/oracle_aln.c tests/oracle_samse.c tests/oracle_sampe.c tests/oracle_pemerge.c -lz -lm -lpthread

# host pipeline under ThreadSanitizer over the CPU oracle stages (TEST ONLY): make tsan
TSAN_CC ?= $(shell test -x /usr/bin/gcc && echo /usr/bin/gcc || echo $(CC))   # a compiler whose installation ships libtsan
tsan: tests/_build/bwa-b200-tsan
tests/_build/bwa-b200-tsan: $(HOST_SRC) $(HOST)/bb_cli.c $(wildcard $(HOST)/*.h) $(wildcard include/*.h) oracle/oracle_fm.c oracle/oracle_sw.c oracle/oracle_stages.c tests/oracle_index.c tests/oracle_index_steps.c tests/oracle_maxk.c tests/oracle_fastmap.c tests/oracle_aln.c tests/oracle_samse.c tests/oracle_sampe.c tests/oracle_pemerge.c
	@mkdir -p tests/_build
	$(TSAN_CC) -fsanitize=thread -O1 -g -Wall -Wno-unused-function -Iinclude -I$(HOST) -Ioracle -pthread -DBB_MAIN -o $@ $(HOST_SRC) $(HOST)/bb_cli.c oracle/oracle_fm.c oracle/oracle_sw.c oracle/oracle_stages.c tests/oracle_index.c tests/oracle_index_steps.c tests/oracle_maxk.c tests/oracle_fastmap.c tests/oracle_aln.c tests/oracle_samse.c tests/oracle_sampe.c tests/oracle_pemerge.c -lz -lm -lpthread

clean:
	rm -rf build bwa_b200/libbwa_b200.so bwa_b200/bwa-b200 tests/_build
.PHONY: all oracle testbin tsan clean

# CUDA kernels compiled for the CPU SIMT emulator (tests/cusim): TEST ONLY, checks kernel logic without a GPU
CUSIM_FLAGS := -O2 -g -std=c++17 -fPIC -x c++ -include tests/cusim/cusim.h -DBWAG_CUSIM -Iinclude -I$(CUDA) -Itests/cusim -Wall -Wno-unused-function -Wno-unknown-pragmas -Wno-unused-variable
cusim: tests/_build/libbwa_b200_cusim.so tests/_build/bwa-b200-cusim
tests/_build/cusim_%.o: $(CUDA)/%.cu $(CUDA_HDR) tests/cusim/cusim.h
	@mkdir -p tests/_build
	$(CXX) $(CUSIM_FLAGS) -c $< -o $@
tests/_build/cusim_rt.o: tests/cusim/cusim.cpp tests/cusim/cusim.h
	@mkdir -p tests/_build
	$(CXX) -O2 -g -std=c++17 -fPIC -Itests/cusim -c $< -o $@
CUSIM_OBJ := $(patsubst $(CUDA)/%.cu,tests/_build/cusim_%.o,$(CUDA_SRC)) tests/_build/cusim_rt.o
tests/_build/libbwa_b200_cusim.so: $(CUSIM_OBJ) $(HOST_OBJ) build/host/bb_cli.o
	$(CXX) -shared -Wl,-Bsymbolic -o $@ $^ -lz -lm -lpthread
tests/_build/bwa-b200-cusim: $(CUSIM_OBJ) $(HOST_OBJ) build/host/bb_main.o
	$(CXX) -o $@ build/host/bb_main.o $(HOST_OBJ) $(CUSIM_OBJ) -lz -lm -lpthread

# the emulated kernels + host glue under AddressSanitizer (TEST ONLY): make asan -> tests/_build/bwa-b200-cusim-asan.
# Device buffers are heap blocks in the emulator, so an out-of-bounds access of a kernel is reported like any other.
ASAN_CXX ?= $(shell test -x /usr/bin/g++ && echo /usr/bin/g++ || echo $(CXX))
ASAN_CC  ?= $(shell test -x /usr/bin/gcc && echo /usr/bin/gcc || echo $(CC))
asan: tests/_build/bwa-b200-cusim-asan
tests/_build/bwa-b200-cusim-asan: $(CUDA_SRC) $(CUDA_HDR) $(HOST_SRC) $(HOST)/bb_cli.c $(wildcard $(HOST)/*.h) $(wildcard include/*.h) tests/cusim/cusim.cpp tests/cusim/cusim.h
	@mkdir -p tests/_build/asan
	for f in $(CUDA_SRC); do $(ASAN_CXX) -O1 -g -std=c++17 -fPIC -fsanitize=address -fno-omit-frame-pointer -x c++ -include tests/cusim/cusim.h -DBWAG_CUSIM -Iinclude -I$(CUDA) -Itests/cusim -Wno-unknown-pragmas -c $$f -o tests/_build/asan/k_`basename $$f .cu`.o || exit 1; done
	$(ASAN_CXX) -O1 -g -std=c++17 -fPIC -fsanitize=address -Itests/cusim -c tests/cusim/cusim.cpp -o tests/_build/asan/rt.o
	for f in $(HOST_SRC); do $(ASAN_CC) -O1 -g -fsanitize=address -fno-omit-frame-pointer -Iinclude -I$(HOST) -pthread -c $$f -o tests/_build/asan/h_`basename $$f .c`.o || exit 1; done
	$(ASAN_CC) -O1 -g -fsanitize=address -fno-omit-frame-pointer -Iinclude -I$(HOST) -pthread -DBB_MAIN -c $(HOST)/bb_cli.c -o tests/_build/asan/h_main.o
	$(ASAN_CXX) -fsanitize=address -o $@ tests/_build/asan/*.o -lz -lm -lpthread
.PHONY: asan

# Variant with 2^16-symbol Occ superblocks (TEST ONLY): the u32-relative counts, the per-superblock absolute counts and every
# carry across a superblock boundary are exercised by a 1 Mbp reference the way a 3 Gbp reference exercises them in production
# (whose only superblock boundaries are at 2^31 and 2^32).  sb16: emulator build; sb16-cuda: the same for the GPU (prebuilt here, runs on the box).
SB16 := -DBWAG_SB_SHIFT=16 -DBWAG_MAX_SB=64
sb16: tests/_build/bwa-b200-cusim-sb16
tests/_build/bwa-b200-cusim-sb16: $(CUDA_SRC) $(CUDA_HDR) $(HOST_OBJ) build/host/bb_main.o tests/_build/cusim_rt.o
	@mkdir -p tests/_build/sb16
	for f in $(CUDA_SRC); do $(CXX) $(CUSIM_FLAGS) $(SB16) -c $$f -o tests/_build/sb16/c_`basename $$f .cu`.o || exit 1; done
	$(CXX) -o $@ build/host/bb_main.o $(HOST_OBJ) tests/_build/sb16/c_*.o tests/_build/cusim_rt.o -lz -lm -lpthread
sb16-cuda: tests/_build/bwa-b200-sb16
tests/_build/bwa-b200-sb16: $(CUDA_SRC) $(CUDA_HDR) $(HOST_OBJ) build/host/bb_main.o
	@mkdir -p tests/_build/sb16
	for f in $(CUDA_SRC); do $(NVCC) $(NVFLAGS) $(SB16) `test $$f = $(CUDA)/bwag_tail.cu && echo -fmad=false` -c $$f -o tests/_build/sb16/g_`basename $$f .cu`.o || exit 1; done
	$(CC) -o $@ build/host/bb_main.o $(HOST_OBJ) tests/_build/sb16/g_*.o -L/usr/local/cuda/lib64 -lcudart -lstdc++ -lz -lm -lpthread -Wl,-rpath,/usr/local/cuda/lib64
.PHONY: sb16 sb16-cuda
