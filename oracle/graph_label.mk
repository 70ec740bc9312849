# TEST INFRASTRUCTURE.  Builds oracle/_ref/libeuler_ref_labels.so: ref_shim/graph_label_shim.cc over the reference graph and
# engine of oracle/_ref/libeuler_ref.so (make -C oracle first).  Only where $(REF) exists, as oracle/Makefile's `ref` target.
REF ?= /root/reference
OUT := _ref
CXX := g++
CXXFLAGS := -std=c++11 -O2 -fPIC -ffp-contract=off -include cstdint -include stdexcept -D_GLIBCXX_USE_CXX11_ABI=0 \
            -I$(REF) -I$(REF)/third_party -w

all: $(if $(wildcard $(REF)/euler/core/api/api.cc),$(OUT)/libeuler_ref_labels.so,)

$(OUT)/libeuler_ref_labels.so: ref_shim/graph_label_shim.cc $(OUT)/libeuler_ref.so
	$(CXX) $(CXXFLAGS) -shared -o $@ ref_shim/graph_label_shim.cc -L$(OUT) -l:libeuler_ref.so -Wl,-rpath,'$$ORIGIN'

.PHONY: all
