# Top-level build of the TEST infrastructure (sim + oracle).  The product (CUDA) is built by
# ltesniffer_b200/build.py / __graft_entry__.build().
CC ?= gcc
CXX ?= g++
CFLAGS = -O3 -g -fPIC -std=gnu11 -Wall -Wno-unused-function -ffp-contract=off -fno-fast-math
CXXFLAGS = -O2 -g -fPIC -std=c++17 -Wall -ffp-contract=off -fno-fast-math

all: sim/libltesim.so oracle/liblteoracle.so oracle/liblteosync.so oracle/liblteomib.so oracle_track/liblteotrack.so oracle/liblteochan.so oracle/liblteochanpoly.so oracle_ul/liblteopuschrx.so

sim/libltesim.so: sim/lte_common.c sim/lte_sim.c sim/lte_common.h sim/lte_sim.h include/lte_tables.h
	$(CC) $(CFLAGS) -shared -o $@ sim/lte_common.c sim/lte_sim.c -lm

oracle/liblteoracle.so: oracle/lte_oracle.c oracle/lte_oracle.h sim/lte_common.c sim/lte_common.h include/lte_tables.h
	$(CC) $(CFLAGS) -shared -o $@ oracle/lte_oracle.c sim/lte_common.c -lm -lpthread

# cell search oracle: lteo_det_sum and the shared PSS / SSS sequences come from liblteoracle.so
oracle/liblteosync.so: oracle/lte_sync_oracle.c oracle/lte_sync_oracle.h oracle/lte_oracle.h oracle/liblteoracle.so
	$(CC) $(CFLAGS) -shared -o $@ oracle/lte_sync_oracle.c -Loracle -llteoracle -Wl,-rpath,'$$ORIGIN' -lm

# PBCH combining oracle: lteo_dci_decode and the shared primitives come from liblteoracle.so
oracle/liblteomib.so: oracle/lte_mib_oracle.c oracle/lte_mib_oracle.h oracle/lte_oracle.h oracle/liblteoracle.so
	$(CC) $(CFLAGS) -shared -o $@ oracle/lte_mib_oracle.c -Loracle -llteoracle -Wl,-rpath,'$$ORIGIN' -lm

# tracker oracle: its find state (LTEO_TRACK_REACQUIRE) is lteo_cell_search of liblteosync.so
oracle_track/liblteotrack.so: oracle_track/lte_track_oracle.c oracle_track/lte_track_oracle.h oracle/lte_sync_oracle.h oracle/liblteosync.so
	$(CC) $(CFLAGS) -shared -o $@ oracle_track/lte_track_oracle.c -Loracle -llteosync -Wl,-rpath,'$$ORIGIN/../oracle' -lm

# PUSCH with one or two receive antennas: lteo_det_sum, lteo_idft, lteo_dlsch_decode and the shared primitives come from liblteoracle.so
oracle_ul/liblteopuschrx.so: oracle_ul/lte_pusch_rx_oracle.c oracle_ul/lte_pusch_rx_oracle.h oracle/lte_oracle.h oracle/liblteoracle.so
	$(CC) $(CFLAGS) -shared -o $@ oracle_ul/lte_pusch_rx_oracle.c -Loracle -llteoracle -Wl,-rpath,'$$ORIGIN/../oracle' -lm

# channeliser oracle: stands alone
oracle/liblteochan.so: oracle/lte_chan_oracle.c oracle/lte_chan_oracle.h
	$(CC) $(CFLAGS) -shared -o $@ oracle/lte_chan_oracle.c -lm

# rational carriers and integer samples: integer carriers are lteo_chan_design's, from liblteochan.so
oracle/liblteochanpoly.so: oracle/lte_chan_poly_oracle.c oracle/lte_chan_poly_oracle.h oracle/lte_chan_oracle.h oracle/liblteochan.so
	$(CC) $(CFLAGS) -shared -o $@ oracle/lte_chan_poly_oracle.c -Loracle -llteochan -Wl,-rpath,'$$ORIGIN' -lm

# C++ example of the C-ABI (needs ltesniffer_b200/libltephy_b200.so, built by ltesniffer_b200/build.py)
examples/offline_decode: examples/offline_decode.cpp examples/cell_chain.h include/ltephy_b200.h include/ltephy_search.h include/ltephy_sinks.h
	$(CXX) -O2 -std=c++17 -Wall -Iinclude -o $@ examples/offline_decode.cpp -Lltesniffer_b200 -lltephy_b200 -Wl,-rpath,'$$ORIGIN/../ltesniffer_b200'

examples/offline_ul: examples/offline_ul.cpp examples/cell_chain.h include/ltephy_b200.h include/ltephy_search.h include/ltephy_sinks.h
	$(CXX) -O2 -std=c++17 -Wall -Iinclude -o $@ examples/offline_ul.cpp -Lltesniffer_b200 -lltephy_b200 -Wl,-rpath,'$$ORIGIN/../ltesniffer_b200'

examples/cell_search: examples/cell_search.cpp examples/cell_chain.h include/ltephy_b200.h include/ltephy_search.h include/ltephy_sinks.h
	$(CXX) -O2 -std=c++17 -Wall -Iinclude -o $@ examples/cell_search.cpp -Lltesniffer_b200 -lltephy_b200 -Wl,-rpath,'$$ORIGIN/../ltesniffer_b200'

examples/decode_recording: examples/decode_recording.cpp examples/cell_chain.h include/ltephy_b200.h include/ltephy_search.h include/ltephy_sinks.h
	$(CXX) -O2 -std=c++17 -Wall -Iinclude -o $@ examples/decode_recording.cpp -Lltesniffer_b200 -lltephy_b200 -Wl,-rpath,'$$ORIGIN/../ltesniffer_b200'

examples/decode_wideband: examples/decode_wideband.cpp examples/cell_chain.h include/ltephy_b200.h include/ltephy_search.h include/ltephy_sinks.h
	$(CXX) -O2 -std=c++17 -Wall -Iinclude -o $@ examples/decode_wideband.cpp -Lltesniffer_b200 -lltephy_b200 -Wl,-rpath,'$$ORIGIN/../ltesniffer_b200'

examples/decode_recording_ul: examples/decode_recording_ul.cpp examples/cell_chain.h include/ltephy_b200.h include/ltephy_search.h include/ltephy_sinks.h
	$(CXX) -O2 -std=c++17 -Wall -Iinclude -o $@ examples/decode_recording_ul.cpp -Lltesniffer_b200 -lltephy_b200 -Wl,-rpath,'$$ORIGIN/../ltesniffer_b200'

examples/compat_check: examples/compat_check.cpp compat/srsran/srsran.h compat/ltephy_compat_ext.h include/ltephy_b200.h
	$(CXX) -O2 -std=c++17 -Wall -Iinclude -Icompat -o $@ examples/compat_check.cpp -Lltesniffer_b200 -lltephy_srsran_compat -lltephy_b200 -Wl,-rpath,'$$ORIGIN/../ltesniffer_b200'

examples/compat_ul_check: examples/compat_ul_check.cpp compat/srsran/srsran.h include/ltephy_b200.h
	$(CXX) -O2 -std=c++17 -Wall -Iinclude -Icompat -o $@ examples/compat_ul_check.cpp -Lltesniffer_b200 -lltephy_srsran_compat -lltephy_b200 -Wl,-rpath,'$$ORIGIN/../ltesniffer_b200'

clean:
	rm -f sim/*.so oracle/*.so oracle_track/*.so oracle_ul/*.so examples/offline_decode examples/offline_ul examples/compat_check examples/compat_ul_check examples/cell_search examples/decode_recording examples/decode_recording_ul examples/decode_wideband
