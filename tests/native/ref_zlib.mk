# tests/native/ref_zlib.mk — test infrastructure: builds tests/native/ref_compact_zlib.cc (the reference driver with the zlib
# CompressionOptions of the input files) with oracle/Makefile's flags, next to the driver it wraps:
#   make -C oracle -f ../tests/native/ref_zlib.mk zlib
include Makefile
SELF := ../tests/native/ref_zlib.mk
ZLIB_SRC := ../tests/native/ref_compact_zlib.cc

.PHONY: zlib
zlib:
	@if [ -d $(REF)/db ]; then $(MAKE) -f $(SELF) $(OUT)/ref_compact_zlib && \
	  if [ -f $(B200_LIB_DIR)/libb200c.so ]; then $(MAKE) -f $(SELF) $(OUT)/ref_compact_zlib_b200; fi; \
	else echo "no $(REF): using prebuilt $(OUT)/ if present"; fi

$(OUT)/ref_compact_zlib: $(ZLIB_SRC) ref_compact.cc $(OUT)/libtoplingdb_ref.so
	$(CXX) $(REF_CXXFLAGS) -I$(CURDIR)/.. -o $@ $(ZLIB_SRC) -L$(OUT) -ltoplingdb_ref -Wl,-rpath,'$$ORIGIN' -pthread -ldl

$(OUT)/ref_compact_zlib_b200: $(ZLIB_SRC) ref_compact.cc $(PLUGIN_SRCS) $(PLUGIN_HDRS) $(OUT)/libtoplingdb_ref.so $(B200_LIB_DIR)/libb200c.so
	$(CXX) $(REF_CXXFLAGS) -DWITH_B200_PLUGIN -I$(CURDIR)/.. -I$(CURDIR)/../include -o $@ $(ZLIB_SRC) \
	  $(PLUGIN_SRCS) -L$(OUT) -ltoplingdb_ref -L$(B200_LIB_DIR) -lb200c \
	  -Wl,-rpath,'$$ORIGIN' -Wl,-rpath,'$$ORIGIN/../../toplingdb_b200' -pthread -ldl
