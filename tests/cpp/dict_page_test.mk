# CPU-only test of a segment's dictionary page and the code -> global id table the device decode takes (no library is
# linked).  make -C tests/cpp -f dict_page_test.mk [OUT=<path of the binary>]
CXX ?= g++
CXXFLAGS ?= -O2 -std=c++17 -Wall -Wno-unused-parameter -Wno-reorder
HOST := ../../starrocks_b200/host
OUT ?= dict_page_test

$(OUT): dict_page_test.cpp $(HOST)/column/chunk.h $(HOST)/column/binary_column.h $(HOST)/exec/global_dict.h $(HOST)/exec/pipeline/operator.h
	$(CXX) $(CXXFLAGS) -o $@ dict_page_test.cpp

clean:
	rm -f $(OUT)
