# Test infrastructure only:  make -C oracle -f graphics_deflate.mk
# The reference's framing around this library's compressed (B200TIMG_DEFLATE) PNG streams:
#  oracle/_ref/libtimg_graphics_replay.so - the UNMODIFIED reference translation units of the PNG writer and the kitty
#      (plain and tmux form) / iTerm2 canvases (plus the ones they use), compiled where they lie under $(REF) with
#      deflate_replay/libdeflate.h (replays a given zlib stream) in place of libdeflate, and
#      oracle/ref_graphics_replay.cc, their extern "C" door.  tests/test_graphics_deflate_*.py read it.
#  oracle/_ref/graphics_deflate_adapter_check - the same reference canvases against B200KittyCanvas / B200ITerm2Canvas
#      (timg_b200/csrc/adapters.h) with deflate = true, the reference fed the adapters' own zlib streams (runs on the GPU).
# Only built when $(REF) exists; elsewhere the tests use what was built (or skip).
REF ?= /root/reference
B   := _ref/graphics_deflate
CXX ?= g++
# The reference's own flags (src/CMakeLists.txt:1,36): -O3, no -march, no fast-math.
REF_CXXFLAGS := -std=gnu++17 -O3 -W -Wall -Wextra -Wno-unused-parameter -fPIC \
   -DWITH_TIMG_STB_RESIZE -DWITH_TIMG_STB -DWITH_TIMG_QOI \
   -I$(B) -I$(REF)/third_party -I$(REF)/third_party/qoi -I$(REF)/src
BASE_TUS := framebuffer terminal-canvas buffered-write-sequencer utils
GFX_TUS  := timg-png kitty-canvas iterm2-canvas
BASE_OBJS := $(addprefix $(B)/,$(addsuffix .o,$(BASE_TUS)))
GFX_OBJS  := $(addprefix $(B)/,$(addsuffix .o,$(GFX_TUS)))

ifneq ($(wildcard $(REF)/src/kitty-canvas.cc),)
all: _ref/libtimg_graphics_replay.so _ref/graphics_deflate_adapter_check
$(B)/timg-version.h:
	mkdir -p $(B) && echo '#define TIMG_VERSION "oracle"' > $@
$(GFX_OBJS): $(B)/%.o: $(REF)/src/%.cc $(B)/timg-version.h deflate_replay/libdeflate.h
	$(CXX) $(REF_CXXFLAGS) -Ideflate_replay -c $< -o $@
$(BASE_OBJS): $(B)/%.o: $(REF)/src/%.cc $(B)/timg-version.h
	$(CXX) $(REF_CXXFLAGS) -c $< -o $@
$(B)/ref_graphics_replay.o: ref_graphics_replay.cc $(B)/timg-version.h
	$(CXX) $(REF_CXXFLAGS) -c $< -o $@
# -Bsymbolic-functions: the reference's objects call ref_graphics_replay.cc's system(), not libc's
_ref/libtimg_graphics_replay.so: $(BASE_OBJS) $(GFX_OBJS) $(B)/ref_graphics_replay.o
	$(CXX) -shared -Wl,-Bsymbolic-functions -o $@ $^ -lz -lpthread
_ref/graphics_deflate_adapter_check: graphics_deflate_adapter_check.cc ../timg_b200/csrc/adapters.h $(BASE_OBJS) $(GFX_OBJS) ../timg_b200/libb200timg.so
	$(CXX) $(REF_CXXFLAGS) -Wno-missing-field-initializers -I../include -I../timg_b200/csrc graphics_deflate_adapter_check.cc \
	    $(BASE_OBJS) $(GFX_OBJS) -L../timg_b200 -lb200timg -Wl,-rpath,'$$ORIGIN/../../timg_b200' -lz -lpthread -o $@
else
all:
	@echo "reference sources absent: using prebuilt _ref/libtimg_graphics_replay.so / graphics_deflate_adapter_check if present"
endif

clean:
	rm -rf $(B) _ref/libtimg_graphics_replay.so _ref/graphics_deflate_adapter_check
.PHONY: all clean
