# Test infrastructure only:  make -C oracle -f qoi.mk   (after oracle/Makefile)
# oracle/_ref/libtimg_qoi_ref.so - oracle/ref_qoi.cc, an extern "C" door onto the UNMODIFIED reference QOIImageSource,
# linked against the reference translation units in oracle/_ref/libtimg_ref.so.  tests/golden/make_qoi_golden.py and
# the QOI tests read it.  Only built when $(REF) exists; elsewhere the tests use what was built (or skip).
REF ?= /root/reference
B   := _ref
CXX ?= g++
# The reference's own flags (src/CMakeLists.txt:1,36): -O3, no -march, no fast-math.
REF_CXXFLAGS := -std=gnu++17 -O3 -W -Wall -Wextra -Wno-unused-parameter -fPIC \
   -DWITH_TIMG_STB_RESIZE -DWITH_TIMG_STB -DWITH_TIMG_QOI \
   -I$(B) -I$(REF)/third_party -I$(REF)/third_party/qoi -I$(REF)/src

ifneq ($(wildcard $(REF)/src/qoi-image-source.cc),)
all: $(B)/libtimg_qoi_ref.so
$(B)/ref_qoi.o: ref_qoi.cc $(B)/libtimg_ref.so
	$(CXX) $(REF_CXXFLAGS) -c $< -o $@
$(B)/libtimg_qoi_ref.so: $(B)/ref_qoi.o $(B)/libtimg_ref.so
	$(CXX) -shared -o $@ $< -L$(B) -ltimg_ref -Wl,-rpath,'$$ORIGIN' -lpthread
else
all:
	@echo "reference sources absent: using prebuilt $(B)/libtimg_qoi_ref.so if present"
endif

clean:
	rm -f $(B)/ref_qoi.o $(B)/libtimg_qoi_ref.so
.PHONY: all clean
