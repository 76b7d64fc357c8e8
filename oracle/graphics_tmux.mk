# Test infrastructure only:  make -C oracle -f graphics_tmux.mk
# kitty's tmux form on the reference side, next to what oracle/graphics.mk builds for the plain canvases:
#  (1) oracle/_ref/libtimg_graphics_tmux_ref.so - the UNMODIFIED reference translation units of the PNG writer and
#      the kitty canvas (plus the ones they use), compiled where they lie under $(REF) with
#      deflate_stored/libdeflate.h (stored deflate blocks) in place of libdeflate, and oracle/ref_graphics_tmux.cc,
#      their extern "C" door, which also defines system() and time() for them.
#      tests/golden/make_graphics_tmux_golden.py reads it.
#  (2) oracle/_ref/kitty_tmux_adapter_check - the reference canvas against B200KittyCanvas (timg_b200/csrc/adapters.h)
#      in tmux mode through the same TerminalCanvas interface, time() pinned and system() recorded inside the binary
#      (runs on the GPU).
# Only built when $(REF) exists; elsewhere the tests use what was built (or skip).
REF ?= /root/reference
B   := _ref/graphics_tmux
CXX ?= g++
# The reference's own flags (src/CMakeLists.txt:1,36): -O3, no -march, no fast-math.
REF_CXXFLAGS := -std=gnu++17 -O3 -W -Wall -Wextra -Wno-unused-parameter -fPIC \
   -DWITH_TIMG_STB_RESIZE -DWITH_TIMG_STB -DWITH_TIMG_QOI \
   -I$(B) -I$(REF)/third_party -I$(REF)/third_party/qoi -I$(REF)/src
BASE_TUS := framebuffer terminal-canvas buffered-write-sequencer utils
GFX_TUS  := timg-png kitty-canvas
BASE_OBJS := $(addprefix $(B)/,$(addsuffix .o,$(BASE_TUS)))
GFX_OBJS  := $(addprefix $(B)/,$(addsuffix .o,$(GFX_TUS)))

ifneq ($(wildcard $(REF)/src/kitty-canvas.cc),)
all: _ref/libtimg_graphics_tmux_ref.so _ref/kitty_tmux_adapter_check
$(B)/timg-version.h:
	mkdir -p $(B) && echo '#define TIMG_VERSION "oracle"' > $@
$(GFX_OBJS): $(B)/%.o: $(REF)/src/%.cc $(B)/timg-version.h deflate_stored/libdeflate.h
	$(CXX) $(REF_CXXFLAGS) -Ideflate_stored -c $< -o $@
$(BASE_OBJS): $(B)/%.o: $(REF)/src/%.cc $(B)/timg-version.h
	$(CXX) $(REF_CXXFLAGS) -c $< -o $@
$(B)/ref_graphics_tmux.o: ref_graphics_tmux.cc $(B)/timg-version.h
	$(CXX) $(REF_CXXFLAGS) -c $< -o $@
# -Bsymbolic-functions: the reference's objects call ref_graphics_tmux.cc's system() and time(), not libc's
_ref/libtimg_graphics_tmux_ref.so: $(BASE_OBJS) $(GFX_OBJS) $(B)/ref_graphics_tmux.o
	$(CXX) -shared -Wl,-Bsymbolic-functions -o $@ $^ -lz -lpthread
_ref/kitty_tmux_adapter_check: kitty_tmux_adapter_check.cc ../timg_b200/csrc/adapters.h $(BASE_OBJS) $(GFX_OBJS) ../timg_b200/libb200timg.so
	$(CXX) $(REF_CXXFLAGS) -Wno-missing-field-initializers -I../include -I../timg_b200/csrc kitty_tmux_adapter_check.cc \
	    $(BASE_OBJS) $(GFX_OBJS) -L../timg_b200 -lb200timg -Wl,-rpath,'$$ORIGIN/../../timg_b200' -lz -lpthread -o $@
else
all:
	@echo "reference sources absent: using prebuilt _ref/libtimg_graphics_tmux_ref.so / kitty_tmux_adapter_check if present"
endif

clean:
	rm -rf $(B) _ref/libtimg_graphics_tmux_ref.so _ref/kitty_tmux_adapter_check
.PHONY: all clean
