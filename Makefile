# Build everything in-tree (artefacts are git-ignored):
#   smudgeplot_b200/lib/libhetmers_b200.so   CUDA kernels (sm_90a, H100) + C ABI (include/hetmers_b200.h)
#   smudgeplot_b200/bin/hetmers              the drop-in executable (plain C host)
#   smudgeplot_b200/bin/condition_kmer_table trim + symmetrise a table of any size into new table files
#   oracle/...                               the CPU checker (test infrastructure, see oracle/Makefile)
NVCC   ?= nvcc
CC     ?= gcc
ARCH   := -gencode arch=compute_90a,code=sm_90a
NVFLAGS := $(EXTRA) -O3 -std=c++17 $(ARCH) -lineinfo -Xcompiler -fPIC,-Wall,-Wextra -Iinclude -Ismudgeplot_b200/csrc
CFLAGS := -O2 -Wall -Wextra -fPIC -Iinclude -Ismudgeplot_b200/csrc

LIBDIR := smudgeplot_b200/lib
BINDIR := smudgeplot_b200/bin
OBJDIR := build
LIB    := $(LIBDIR)/libhetmers_b200.so
BIN    := $(BINDIR)/hetmers $(BINDIR)/extract_kmer_pairs $(BINDIR)/condition_kmer_table

CU_SRC := smudgeplot_b200/csrc/hm_kernels.cu smudgeplot_b200/csrc/hm_scan.cu smudgeplot_b200/csrc/hm_peer.cu \
          smudgeplot_b200/csrc/hm_condition.cu smudgeplot_b200/csrc/hm_symm.cu \
          smudgeplot_b200/csrc/hm_shard_condition.cu smudgeplot_b200/csrc/hm_pairs.cu
CU_OBJ := $(patsubst smudgeplot_b200/csrc/%.cu,$(OBJDIR)/%.o,$(CU_SRC))
C_OBJ  := $(OBJDIR)/fastk_table.o
HDRS   := include/hetmers_b200.h smudgeplot_b200/csrc/hm_internal.h smudgeplot_b200/csrc/hm_device.cuh

.PHONY: all lib bin oracle clean
all: lib bin oracle
lib: $(LIB)
bin: $(BIN)

$(OBJDIR)/%.o: smudgeplot_b200/csrc/%.cu $(HDRS)
	@mkdir -p $(OBJDIR)
	$(NVCC) $(NVFLAGS) -Xptxas -v -c $< -o $@ 2> $(OBJDIR)/$*.ptxas.log || (cat $(OBJDIR)/$*.ptxas.log; false)

$(OBJDIR)/fastk_table.o: smudgeplot_b200/host/fastk_table.c $(HDRS)
	@mkdir -p $(OBJDIR)
	$(CC) $(CFLAGS) -c $< -o $@

$(LIB): $(CU_OBJ) $(C_OBJ)
	@mkdir -p $(LIBDIR)
	$(NVCC) -shared $(ARCH) -o $@ $^ -cudart static -lpthread

$(BINDIR)/hetmers: smudgeplot_b200/host/hetmers_main.c $(LIB) $(HDRS)
	@mkdir -p $(BINDIR)
	$(CC) $(CFLAGS) -o $@ $< -L$(LIBDIR) -lhetmers_b200 -Wl,-rpath,'$$ORIGIN/../lib'

# the same host source with the pair-listing output stage (the reference ships PloidyList.c,
# a near copy of PloidyPlot.c, for this)
$(BINDIR)/extract_kmer_pairs: smudgeplot_b200/host/hetmers_main.c $(LIB) $(HDRS)
	@mkdir -p $(BINDIR)
	$(CC) $(CFLAGS) -DEXTRACT_PAIRS -o $@ $< -L$(LIBDIR) -lhetmers_b200 -Wl,-rpath,'$$ORIGIN/../lib'

# conditioning of tables of any size into new table files (hm_scan_condition_files)
$(BINDIR)/condition_kmer_table: smudgeplot_b200/host/condition_main.c $(LIB) $(HDRS)
	@mkdir -p $(BINDIR)
	$(CC) $(CFLAGS) -o $@ $< -L$(LIBDIR) -lhetmers_b200 -Wl,-rpath,'$$ORIGIN/../lib'

oracle:
	$(MAKE) -C oracle

clean:
	rm -rf $(OBJDIR) $(LIBDIR) $(BINDIR)
	$(MAKE) -C oracle clean
