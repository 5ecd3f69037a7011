# The fused sink fed from a registered page-locked pool (chunks forwarded to sr_fragment_push_chunks), checked against
# the CPU oracle.  Links the product library and -- as test infrastructure -- oracle/libsr_oracle.so.
#   make -C tests/cpp -f frag_chunk_list_test.mk [OUT=<path of the binary>]
CXX ?= g++
CXXFLAGS ?= -O2 -std=c++17 -Wall -Wno-unused-parameter -Wno-reorder
HOST := ../../starrocks_b200/host
HDRS := $(HOST)/column/chunk.h $(HOST)/exec/pipeline/operator.h $(HOST)/gpu/gpu_operators.h ../../include/sr_gpu_ops.h ../../oracle/sr_oracle.h
OUT ?= frag_chunk_list_test
LIBDIR := $(abspath ../../starrocks_b200)
ORCDIR := $(abspath ../../oracle)

$(OUT): frag_chunk_list_test.cpp $(HDRS) $(LIBDIR)/libsr_gpu.so $(ORCDIR)/libsr_oracle.so
	$(CXX) $(CXXFLAGS) -o $@ frag_chunk_list_test.cpp -L$(LIBDIR) -lsr_gpu -L$(ORCDIR) -lsr_oracle \
	    -Wl,-rpath,$(LIBDIR) -Wl,-rpath,$(ORCDIR) -ldl -lpthread

clean:
	rm -f $(OUT)
