// NOTE: this file has never been compiled — the build image has no Go toolchain.  It is reviewed source, written
// against include/swec.h; the same C ABI is exercised from C (tests/c/cgo_shaped_harness.c) and Python on the GPU.
//go:build swec && cgo

// weed/storage/erasure_coding/ec_swec.go
package erasure_coding

/*
#cgo CFLAGS:  -I${SRCDIR}/../../../third_party/swec/include
#cgo LDFLAGS: -L${SRCDIR}/../../../third_party/swec/lib -lswec -lstdc++ -ldl -lpthread
#include <stdlib.h>
#include "swec.h"
*/
import "C"

import (
	"fmt"
	"io"
	"os"
	"runtime"
	"strings"
	"sync/atomic"
	"unsafe"

	"github.com/klauspost/reedsolomon"
)

// One volume server process drives every GPU of the box: each encoder / file-level call takes the next
// GPU round-robin (volume v → GPU v mod N — independent volumes need no collective), the same way the
// shell already runs up to 10 volumes concurrently (weed/shell/common.go:11).  The round-robin walks the
// library's socket-interleaved order (0,4,1,5,… on a two-socket box): n concurrent volumes then use both
// sockets' memory controllers — one socket cannot feed four GPUs at full PCIe rate.  Set -ec.gpu=N to pin one.
var (
	swecPinned  = -1 // -ec.gpu flag; -1 = round-robin over all devices
	swecNext    uint32
	swecDevices = func() []C.int {
		var order [64]C.int
		var n C.int
		if C.swec_device_spread_order(&order[0], 64, &n) != C.SWEC_OK || n < 1 {
			return []C.int{0} // calls will fail with SWEC_ERR_NO_DEVICE and surface as Go errors
		}
		return append([]C.int(nil), order[:int(n)]...)
	}()
)

func swecPickDevice() C.int {
	if swecPinned >= 0 {
		return C.int(swecPinned)
	}
	return swecDevices[int(atomic.AddUint32(&swecNext, 1))%len(swecDevices)]
}

type swecEncoder struct {
	h          *C.swec_encoder
	data, par  int
}

// swecCall runs one C entry point and, on failure, fetches its detail string.  swec_last_error() is
// thread-local and the Go scheduler may move a goroutine to another OS thread BETWEEN two cgo calls, so the
// failing call and the read of its detail are bracketed by LockOSThread.
func swecCall(f func() C.int) error {
	runtime.LockOSThread()
	defer runtime.UnlockOSThread()
	return swecErr(f())
}

// swecErr must run on the OS thread that made the failing call (see swecCall).
func swecErr(rc C.int) error {
	if rc == C.SWEC_OK {
		return nil
	}
	msg := C.GoString(C.swec_last_error())
	switch rc {
	case C.SWEC_ERR_TOO_FEW_SHARDS:
		return reedsolomon.ErrTooFewShards
	case C.SWEC_ERR_SHARD_SIZE:
		return reedsolomon.ErrShardSize
	}
	return fmt.Errorf("swec: %s: %s", C.GoString(C.swec_strerror(rc)), msg)
}

// newSwecEncoder replaces reedsolomon.New(ds, ps) (ec_context.go:35, store_ec.go:485).
func newSwecEncoder(dataShards, parityShards int) (reedsolomon.Encoder, error) {
	var h *C.swec_encoder
	if err := swecCall(func() C.int {
		return C.swec_encoder_new(C.int(dataShards), C.int(parityShards), swecPickDevice(), &h)
	}); err != nil {
		return nil, err
	}
	e := &swecEncoder{h: h, data: dataShards, par: parityShards}
	runtime.SetFinalizer(e, func(e *swecEncoder) { C.swec_encoder_free(e.h) })
	return e, nil
}

// pin builds the C pointer table. The slices' backing arrays are Go memory: cgo forbids storing Go
// pointers in C memory across calls, but passing a C array of Go pointers for the duration of one
// call is allowed with runtime.Pinner (Go ≥ 1.21).
func (e *swecEncoder) pin(shards [][]byte, p *runtime.Pinner) (**C.uint8_t, func()) {
	n := e.data + e.par
	tbl := (*[1 << 10]*C.uint8_t)(C.malloc(C.size_t(n) * C.size_t(unsafe.Sizeof(uintptr(0)))))
	for i := 0; i < n; i++ {
		if len(shards[i]) > 0 {
			p.Pin(&shards[i][0])
			tbl[i] = (*C.uint8_t)(unsafe.Pointer(&shards[i][0]))
		} else {
			tbl[i] = nil
		}
	}
	return (**C.uint8_t)(unsafe.Pointer(tbl)), func() { C.free(unsafe.Pointer(tbl)) }
}

func shardLen(shards [][]byte) (int, error) {
	n := 0
	for _, s := range shards {
		if len(s) == 0 {
			continue
		}
		if n == 0 {
			n = len(s)
		} else if len(s) != n {
			return 0, reedsolomon.ErrShardSize
		}
	}
	if n == 0 {
		return 0, reedsolomon.ErrShardNoData
	}
	return n, nil
}

// Encode: parity slices overwritten in place, data untouched (ec_encoder.go:265).
func (e *swecEncoder) Encode(shards [][]byte) error {
	if len(shards) != e.data+e.par {
		return reedsolomon.ErrTooFewShards
	}
	n, err := shardLen(shards)
	if err != nil {
		return err
	}
	for _, s := range shards {
		if len(s) != n {
			return reedsolomon.ErrShardSize
		}
	}
	var p runtime.Pinner
	defer p.Unpin()
	tbl, free := e.pin(shards, &p)
	defer free()
	return swecCall(func() C.int { return C.swec_encode(e.h, tbl, C.size_t(n)) })
}

func (e *swecEncoder) reconstruct(shards [][]byte, dataOnly bool) error {
	if len(shards) != e.data+e.par {
		return reedsolomon.ErrTooFewShards
	}
	n, err := shardLen(shards)
	if err != nil {
		return err
	}
	present := make([]C.uint8_t, len(shards))
	have := 0
	for i, s := range shards {
		if len(s) > 0 {
			present[i] = 1
			have++
		}
	}
	if have == len(shards) {
		return nil
	}
	if have < e.data {
		return reedsolomon.ErrTooFewShards
	}
	for i := range shards { // klauspost allocates nil/empty shards (re-using capacity when it can)
		if present[i] == 0 && (i < e.data || !dataOnly) {
			if cap(shards[i]) >= n {
				shards[i] = shards[i][:n]
			} else {
				shards[i] = make([]byte, n)
			}
		}
	}
	var p runtime.Pinner
	defer p.Unpin()
	tbl, free := e.pin(shards, &p)
	defer free()
	d := C.int(0)
	if dataOnly {
		d = 1
	}
	return swecCall(func() C.int { return C.swec_reconstruct(e.h, tbl, &present[0], C.size_t(n), d) })
}

func (e *swecEncoder) Reconstruct(shards [][]byte) error     { return e.reconstruct(shards, false) } // ec_encoder.go:360
func (e *swecEncoder) ReconstructData(shards [][]byte) error { return e.reconstruct(shards, true) }  // store_ec.go:551

func (e *swecEncoder) Verify(shards [][]byte) (bool, error) {
	n, err := shardLen(shards)
	if err != nil {
		return false, err
	}
	var p runtime.Pinner
	defer p.Unpin()
	tbl, free := e.pin(shards, &p)
	defer free()
	var ok C.int
	if err := swecCall(func() C.int { return C.swec_verify(e.h, tbl, C.size_t(n), &ok) }); err != nil {
		return false, err
	}
	return ok != 0, nil
}

// The remaining reedsolomon.Encoder methods are not used by SeaweedFS on this path
// (grep: only Encode, Reconstruct, ReconstructData are called); they return ErrNotSupported.
func (e *swecEncoder) EncodeIdx([]byte, int, [][]byte) error          { return reedsolomon.ErrNotSupported }
func (e *swecEncoder) ReconstructSome([][]byte, []bool) error         { return reedsolomon.ErrNotSupported }
func (e *swecEncoder) Update([][]byte, [][]byte) error                { return reedsolomon.ErrNotSupported }
func (e *swecEncoder) Split([]byte) ([][]byte, error)                 { return nil, reedsolomon.ErrNotSupported }
func (e *swecEncoder) Join(w io.Writer, s [][]byte, n int) error      { return reedsolomon.ErrNotSupported }

// ---- file-level entry points (preferred: one cgo crossing per volume instead of 12,288) ----------

// generateEcFilesSwec replaces the body of generateEcFiles (ec_encoder.go:110-128).
func generateEcFilesSwec(baseFileName string, bufferSize int, largeBlockSize, smallBlockSize int64, ctx *ECContext) error {
	cs := C.CString(baseFileName)
	defer C.free(unsafe.Pointer(cs))
	if err := swecCall(func() C.int {
		return C.swec_generate_ec_files(cs, C.int64_t(bufferSize), C.int64_t(largeBlockSize), C.int64_t(smallBlockSize),
			C.int(ctx.DataShards), C.int(ctx.ParityShards), swecPickDevice())
	}); err != nil {
		return fmt.Errorf("encodeDatFile: %w", err)
	}
	return nil
}

// generateMissingEcFilesSwec replaces generateMissingEcFiles (ec_encoder.go:146-200).
func generateMissingEcFilesSwec(baseFileName string, ctx *ECContext, additionalDirs []string) ([]uint32, error) {
	cs := C.CString(baseFileName)
	defer C.free(unsafe.Pointer(cs))
	dirs := make([]*C.char, len(additionalDirs)+1)
	for i, d := range additionalDirs {
		dirs[i] = C.CString(d)
		defer C.free(unsafe.Pointer(dirs[i]))
	}
	var rebuilt [C.SWEC_MAX_SHARDS]C.uint32_t
	var n C.int
	if err := swecCall(func() C.int {
		return C.swec_rebuild_ec_files(cs, (**C.char)(unsafe.Pointer(&dirs[0])), C.int(len(additionalDirs)),
			C.int(ctx.DataShards), C.int(ctx.ParityShards), swecPickDevice(), &rebuilt[0], &n)
	}); err != nil {
		return nil, fmt.Errorf("rebuildEcFiles: %w", err)
	}
	ids := make([]uint32, int(n))
	for i := range ids {
		ids[i] = uint32(rebuilt[i])
	}
	return ids, nil
}

// ---- volume-level entry points: the file work of the three EC gRPC handlers, one cgo crossing each --------

// ecShardsGenerateSwec replaces the file work of VolumeEcShardsGenerate (weed/server/volume_grpc_erasure_coding.go:43-146):
// EC ratio from an existing .vif, .ecx before the shards, .dat size snapshot, shards on the GPU, .vif, cleanup on error.
// The handler keeps the volume lookup, the collection check and the maintenance-mode check.
func ecShardsGenerateSwec(dataBaseFileName, indexBaseFileName string, needleVersion uint32, expireAtSec uint64) error {
	cd, ci := C.CString(dataBaseFileName), C.CString(indexBaseFileName)
	defer C.free(unsafe.Pointer(cd))
	defer C.free(unsafe.Pointer(ci))
	return swecCall(func() C.int {
		return C.swec_ec_shards_generate(cd, ci, C.uint32_t(needleVersion), C.uint64_t(expireAtSec), swecPickDevice())
	})
}

// ecShardsRebuildSwec replaces RebuildEcFiles + RebuildEcxFile in VolumeEcShardsRebuild (:149-225).
func ecShardsRebuildSwec(dataBaseFileName, indexBaseFileName string, additionalDirs []string) ([]uint32, error) {
	cd, ci := C.CString(dataBaseFileName), C.CString(indexBaseFileName)
	defer C.free(unsafe.Pointer(cd))
	defer C.free(unsafe.Pointer(ci))
	dirs := make([]*C.char, len(additionalDirs)+1)
	for i, d := range additionalDirs {
		dirs[i] = C.CString(d)
		defer C.free(unsafe.Pointer(dirs[i]))
	}
	var rebuilt [C.SWEC_MAX_SHARDS]C.uint32_t
	var n C.int
	if err := swecCall(func() C.int {
		return C.swec_ec_shards_rebuild(cd, ci, (**C.char)(unsafe.Pointer(&dirs[0])), C.int(len(additionalDirs)),
			swecPickDevice(), &rebuilt[0], &n)
	}); err != nil {
		return nil, err
	}
	ids := make([]uint32, int(n))
	for i := range ids {
		ids[i] = uint32(rebuilt[i])
	}
	return ids, nil
}

// ecShardsToVolumeSwec replaces the file work of VolumeEcShardsToVolume (:578-668); errNoLiveEntries maps to the
// handler's FailedPrecondition with EcNoLiveEntriesSubstring.  Compaction stays in Go.
var errNoLiveEntries = fmt.Errorf("ec volume %s", EcNoLiveEntriesSubstring)

func ecShardsToVolumeSwec(dataBaseFileName, indexBaseFileName string, additionalDirs []string) (datFileSize int64, err error) {
	cd, ci := C.CString(dataBaseFileName), C.CString(indexBaseFileName)
	defer C.free(unsafe.Pointer(cd))
	defer C.free(unsafe.Pointer(ci))
	dirs := make([]*C.char, len(additionalDirs)+1)
	for i, d := range additionalDirs {
		dirs[i] = C.CString(d)
		defer C.free(unsafe.Pointer(dirs[i]))
	}
	var size C.int64_t
	runtime.LockOSThread()
	defer runtime.UnlockOSThread()
	rc := C.swec_ec_shards_to_volume(cd, ci, (**C.char)(unsafe.Pointer(&dirs[0])), C.int(len(additionalDirs)), &size)
	if rc == C.SWEC_ERR_NO_LIVE_NEEDLES {
		return 0, errNoLiveEntries
	}
	return int64(size), swecErr(rc)
}

// ecShardsToVolumeCheckedSwec is ecShardsToVolumeSwec from any k of the k+m shards, with the damage the present parity
// locates in the data shards corrected on the GPU before the .dat is written.  ec.decode deletes every shard once the
// handler succeeds, so this is the last point at which such damage can be fixed.  Columns that cannot be corrected fail
// the call (no .dat, no .idx) with the damaged page ranges in the error, and the shell keeps the EC shards.  Radius 1
// by default; radius 0 decodes only a set whose checked columns are all clean.  The check needs parity shards next to
// the data shards: collectEcShards copies only data shards today, and without parity the call decodes unchecked
// (checked = false), exactly as ecShardsToVolumeSwec.
func ecShardsToVolumeCheckedSwec(dataBaseFileName, indexBaseFileName string, additionalDirs []string, radius int) (datFileSize int64, checked bool, err error) {
	cd, ci := C.CString(dataBaseFileName), C.CString(indexBaseFileName)
	defer C.free(unsafe.Pointer(cd))
	defer C.free(unsafe.Pointer(ci))
	dirs := make([]*C.char, len(additionalDirs)+1)
	for i, d := range additionalDirs {
		dirs[i] = C.CString(d)
		defer C.free(unsafe.Pointer(dirs[i]))
	}
	var size C.int64_t
	var report C.swec_damage_report
	var ranges [64]C.swec_damage_range
	var nRanges, ok C.int
	runtime.LockOSThread()
	defer runtime.UnlockOSThread()
	rc := C.swec_ec_shards_to_volume_checked(cd, ci, (**C.char)(unsafe.Pointer(&dirs[0])), C.int(len(additionalDirs)),
		swecPickDevice(), C.int(radius), &size, &report, &ranges[0], C.int(len(ranges)), &nRanges, &ok)
	switch rc {
	case C.SWEC_OK:
		return int64(size), ok != 0, nil
	case C.SWEC_ERR_NO_LIVE_NEEDLES:
		return 0, false, errNoLiveEntries
	case C.SWEC_ERR_UNCORRECTABLE:
		var where []string
		for i := 0; i < int(nRanges) && i < len(ranges); i++ {
			r := ranges[i]
			who := fmt.Sprintf("ec shard %d", int(r.shard_id))
			if r.shard_id < 0 {
				who = "uncorrectable"
			}
			where = append(where, fmt.Sprintf("%s [%d, %d)", who, int64(r.offset), int64(r.offset)+int64(r.length)))
		}
		if int(nRanges) > len(ranges) {
			where = append(where, fmt.Sprintf("and %d more ranges", int(nRanges)-len(ranges)))
		}
		return 0, false, fmt.Errorf("%w; %d byte columns cannot be corrected, damaged pages: %s", swecErr(rc),
			uint64(report.uncorrectable_columns), strings.Join(where, ", "))
	}
	return 0, false, swecErr(rc)
}

// ---- the read path of a mounted EC volume whose shards are local files ----------------------------------------

// swecEcVolume is the twin of the long-lived EcVolume (ec_volume.go:36-160) for Store.ReadEcShardNeedle
// (weed/storage/store_ec.go:252-355): one handle per mounted volume, closed on unmount.
type swecEcVolume struct{ h *C.swec_ec_volume }

func openSwecEcVolume(dataBaseFileName, indexBaseFileName string, additionalDirs []string) (*swecEcVolume, error) {
	cd, ci := C.CString(dataBaseFileName), C.CString(indexBaseFileName)
	defer C.free(unsafe.Pointer(cd))
	defer C.free(unsafe.Pointer(ci))
	dirs := make([]*C.char, len(additionalDirs)+1)
	for i, d := range additionalDirs {
		dirs[i] = C.CString(d)
		defer C.free(unsafe.Pointer(dirs[i]))
	}
	var h *C.swec_ec_volume
	if err := swecCall(func() C.int {
		return C.swec_ec_volume_open(cd, ci, (**C.char)(unsafe.Pointer(&dirs[0])), C.int(len(additionalDirs)), swecPickDevice(), &h)
	}); err != nil {
		return nil, err
	}
	return &swecEcVolume{h: h}, nil
}

func (v *swecEcVolume) Close() { C.swec_ec_volume_close(v.h); v.h = nil }

// ReadNeedles returns the raw record bytes of every id (nil where the needle is unknown or deleted), reading present
// shards directly and rebuilding the intervals that lived on lost shards in ONE batched GPU call.  bufs are C memory
// (C.malloc), because the call writes through pointers stored in a C array.
func (v *swecEcVolume) ReadNeedles(ids []uint64, capacity int) ([][]byte, []error, error) {
	n := len(ids)
	if n == 0 {
		return nil, nil, nil
	}
	reads := (*[1 << 20]C.swec_needle_read)(C.calloc(C.size_t(n), C.size_t(unsafe.Sizeof(C.swec_needle_read{}))))[:n:n]
	defer C.free(unsafe.Pointer(&reads[0]))
	arena := C.malloc(C.size_t(n * capacity))
	defer C.free(arena)
	for i, id := range ids {
		reads[i].needle_id = C.uint64_t(id)
		reads[i].buf = (*C.uint8_t)(unsafe.Add(arena, i*capacity))
		reads[i].capacity = C.size_t(capacity)
	}
	if err := swecCall(func() C.int { return C.swec_ec_volume_read_needles(v.h, &reads[0], C.int(n)) }); err != nil {
		return nil, nil, err
	}
	out, errs := make([][]byte, n), make([]error, n)
	for i := range reads {
		switch reads[i].status {
		case C.SWEC_OK:
			out[i] = C.GoBytes(unsafe.Pointer(reads[i].buf), C.int(reads[i].n_bytes))
		case C.SWEC_ERR_NOT_FOUND:
			errs[i] = NotFoundError
		case C.SWEC_ERR_DELETED:
			errs[i] = fmt.Errorf("already deleted") // storage.ErrorDeleted at the call site
		default:
			errs[i] = fmt.Errorf("swec: needle %x: %s", ids[i], C.GoString(C.swec_strerror(C.int(reads[i].status))))
		}
	}
	return out, errs, nil
}

// DeleteNeedleFromEcx: journal append (ec_volume_delete.go:28-93).
func (v *swecEcVolume) DeleteNeedleFromEcx(id uint64) error {
	return swecCall(func() C.int { return C.swec_ec_volume_delete_needle(v.h, C.uint64_t(id)) })
}

// ScrubLocal is the whole EcVolume.ScrubLocal (ec_volume_scrub.go:27-118): the index check, the chunk walk over the
// local shards, and Needle.ReadBytes (size, layout, CRC32-C) of every record whose chunks are all local, checked on the
// GPU.  Findings come back in the reference's order and wording.
func (v *swecEcVolume) ScrubLocal(volumeId uint32) (int64, []uint32, []error, error) {
	var entries C.int64_t
	var broken [C.SWEC_MAX_SHARDS]C.uint32_t
	var nBroken, nErrors C.int
	text := make([]byte, 4<<20)
	if err := swecCall(func() C.int {
		return C.swec_ec_volume_scrub_needles(v.h, C.uint32_t(volumeId), &entries, &broken[0], &nBroken,
			(*C.char)(unsafe.Pointer(&text[0])), C.size_t(len(text)), &nErrors)
	}); err != nil {
		return 0, nil, nil, err
	}
	shards := make([]uint32, int(nBroken))
	for i := range shards {
		shards[i] = uint32(broken[i])
	}
	var errs []error
	if nErrors > 0 {
		for _, line := range strings.Split(C.GoString((*C.char)(unsafe.Pointer(&text[0]))), "\n") {
			errs = append(errs, fmt.Errorf("%s", line))
		}
	}
	return int64(entries), shards, errs, nil
}

// swecNeedleDamage is one needle that located damage hits: DamagedBytes a repair restores, UncorrectableBytes it
// cannot (restore that needle from a replica or a backup).  ShardMask has bit i set for each data shard i holding a
// counted byte.
type swecNeedleDamage struct {
	NeedleId           uint64
	Offset             int64
	Size               int32
	ShardMask          uint32
	DamagedBytes       uint64
	UncorrectableBytes uint64
}

// LocateNeedleDamage runs in the scrub of a volume whose shards are all local, next to swecLocateEcDamage: it names the
// live needles the located damage hits (ascending id, at most maxNeedles of them; total is how many there are), and
// the damaged / uncorrectable bytes no live needle owns.  It only reads the shard files.  After swecRepairEcDamage, the
// needles with UncorrectableBytes > 0 are the ones to restore from another copy.
func (v *swecEcVolume) LocateNeedleDamage(radius int, maxNeedles int) (needles []swecNeedleDamage, total int, unowned [2]uint64, err error) {
	var report C.swec_damage_report
	var nRanges, nNeedles, ok C.int
	var cUnowned [2]C.uint64_t
	buf := make([]C.swec_needle_damage, maxNeedles+1)
	if err := swecCall(func() C.int {
		return C.swec_ec_volume_locate_needle_damage(v.h, C.int(radius), &report, nil, 0, &nRanges, &buf[0],
			C.int(maxNeedles), &nNeedles, &cUnowned[0], &ok)
	}); err != nil {
		return nil, 0, unowned, fmt.Errorf("locate needle damage: %w", err)
	}
	total = int(nNeedles)
	for i := 0; i < total && i < maxNeedles; i++ {
		d := buf[i]
		needles = append(needles, swecNeedleDamage{uint64(d.needle_id), int64(d.offset), int32(d.size), uint32(d.shard_mask),
			uint64(d.damaged_bytes), uint64(d.uncorrectable_bytes)})
	}
	unowned = [2]uint64{uint64(cUnowned[0]), uint64(cUnowned[1])}
	return needles, total, unowned, nil
}

// PageSketch answers the shard holder's side of a distributed parity scrub (a VolumeEcShardSketch RPC) for shards this
// volume has mounted: the page sketches of the shards in shardIds, 8 bytes per 4 KiB page under the coordinator's
// seed, all read in one pass through the volume's own descriptors and under its lock, so that a sketch never mixes
// pages from before and after a RepairNeedleDamage.  The caller must check that the coordinator asked for
// SWEC_PAGE_SKETCH_VERSION.  A shard that is not mounted here is an error (SWEC_ERR_TOO_FEW_SHARDS).
func (v *swecEcVolume) PageSketch(seed uint64, shardIds []int) (sketches map[int][]uint64, shardSize int64, err error) {
	var k, m C.int
	var shardDatSize C.int64_t
	if err := swecCall(func() C.int { return C.swec_ec_volume_info(v.h, &k, &m, nil, &shardDatSize, nil) }); err != nil {
		return nil, 0, fmt.Errorf("page sketch: %w", err)
	}
	for _, id := range shardIds {
		if id < 0 || id >= int(k+m) {
			return nil, 0, fmt.Errorf("page sketch: no ec shard %d in a %d+%d volume", id, k, m)
		}
	}
	ptrs := (*[C.SWEC_MAX_SHARDS]*C.uint64_t)(C.calloc(C.SWEC_MAX_SHARDS, C.size_t(unsafe.Sizeof(uintptr(0)))))
	defer C.free(unsafe.Pointer(ptrs))
	// a shard holds shard_dat_size bytes plus at most one small block of padding; a longer one is asked again
	for capPages := (int64(shardDatSize) + 1<<20 + 4096) / 4096; ; {
		var p runtime.Pinner
		bufs := make(map[int][]uint64, len(shardIds))
		for _, id := range shardIds {
			bufs[id] = make([]uint64, capPages+1) // +1: never a zero-length slice to take the address of
			p.Pin(&bufs[id][0])
			ptrs[id] = (*C.uint64_t)(unsafe.Pointer(&bufs[id][0]))
		}
		var length, nPages C.int64_t
		err := swecCall(func() C.int {
			return C.swec_ec_volume_page_sketch(v.h, C.uint64_t(seed), &ptrs[0], C.int64_t(capPages), &length, &nPages)
		})
		p.Unpin()
		if err != nil {
			return nil, 0, fmt.Errorf("page sketch: %w", err)
		}
		if int64(nPages) <= capPages {
			for id, b := range bufs {
				bufs[id] = b[:nPages]
			}
			return bufs, int64(length), nil
		}
		capPages = int64(nPages)
	}
}

// SketchNeedleDamage names the live needles that the pages swecLocateSketchDamage (or its checked twin) flagged hit, from
// this volume's .ecx alone: any holder's ScrubEcVolume handler can report per needle before a single page is fetched.
// needles are in ascending id, at most maxNeedles of them (total is how many there are); unowned are the damaged /
// uncorrectable bytes no live needle owns.  The counts are page-granular upper bounds: every needle with a byte on a
// flagged page is named.  shardSize is the holders' shard size; a mounted shard of another size is an error.
func (v *swecEcVolume) SketchNeedleDamage(pages []swecSketchPage, shardSize int64, maxNeedles int) (needles []swecNeedleDamage, total int, unowned [2]uint64, err error) {
	in := make([]C.swec_sketch_page, len(pages)+1)
	for i, q := range pages {
		in[i].page, in[i].blamed_mask = C.int64_t(q.Page), C.uint32_t(q.Blamed)
		if q.Uncorrectable {
			in[i].uncorrectable = 1
		}
	}
	var nNeedles C.int
	var cUnowned [2]C.uint64_t
	buf := make([]C.swec_needle_damage, maxNeedles+1)
	if err := swecCall(func() C.int {
		return C.swec_ec_volume_sketch_needle_damage(v.h, C.int64_t(shardSize), &in[0], C.int64_t(len(pages)), &buf[0],
			C.int(maxNeedles), &nNeedles, &cUnowned[0])
	}); err != nil {
		return nil, 0, unowned, fmt.Errorf("sketch needle damage: %w", err)
	}
	total = int(nNeedles)
	for i := 0; i < total && i < maxNeedles; i++ {
		d := buf[i]
		needles = append(needles, swecNeedleDamage{uint64(d.needle_id), int64(d.offset), int32(d.size), uint32(d.shard_mask),
			uint64(d.damaged_bytes), uint64(d.uncorrectable_bytes)})
	}
	unowned = [2]uint64{uint64(cUnowned[0]), uint64(cUnowned[1])}
	return needles, total, unowned, nil
}

// swecNeedleRepair is a needle RepairNeedleDamage touched, and how it reads back from the repaired files: Status 0 means
// Needle.ReadBytes accepts it (size, layout and CRC32-C); any other status (1 size mismatch, 2 out of range, 3 bad CRC,
// 4 past the end of its shard) means the needle has to come from a replica or a backup.
type swecNeedleRepair struct {
	swecNeedleDamage
	Status  int32
	CrcGot  uint32
	CrcWant uint32
}

// RepairNeedleDamage is LocateNeedleDamage and swecRepairEcDamage in one pass over the shard files the volume reads,
// under the volume's lock, then a CRC check of every needle the repair touched.  ok is false when an uncorrectable
// column remains or a touched needle does not read back: that is how a column miscorrected beyond the guarantee of the
// code (more than m-t wrong shards) shows.  needles, total and unowned are what LocateNeedleDamage reported before.
func (v *swecEcVolume) RepairNeedleDamage(radius int, maxNeedles int) (needles []swecNeedleRepair, total int, unowned [2]uint64, ok bool, err error) {
	var report C.swec_damage_report
	var nRanges, nNeedles, cOk C.int
	var cUnowned [2]C.uint64_t
	buf := make([]C.swec_needle_damage, maxNeedles+1)
	checks := make([]C.swec_needle_check, maxNeedles+1)
	if err := swecCall(func() C.int {
		return C.swec_ec_volume_repair_needle_damage(v.h, C.int(radius), &report, nil, 0, &nRanges, &buf[0], &checks[0],
			C.int(maxNeedles), &nNeedles, &cUnowned[0], &cOk)
	}); err != nil {
		return nil, 0, unowned, false, fmt.Errorf("repair needle damage: %w", err)
	}
	total = int(nNeedles)
	for i := 0; i < total && i < maxNeedles; i++ {
		d, c := buf[i], checks[i]
		needles = append(needles, swecNeedleRepair{swecNeedleDamage{uint64(d.needle_id), int64(d.offset), int32(d.size),
			uint32(d.shard_mask), uint64(d.damaged_bytes), uint64(d.uncorrectable_bytes)}, int32(c.status),
			uint32(c.crc_got), uint32(c.crc_want)})
	}
	unowned = [2]uint64{uint64(cUnowned[0]), uint64(cUnowned[1])}
	return needles, total, unowned, cOk == 1, nil
}

// swecLocateEcDamage is the parity side of a scrub of a volume whose shards are all local, run before ec.rebuild: it
// names the shard FILES that are wrong, where verify_ec_shards (seaweed-volume/src/storage/erasure_coding/
// ec_encoder.rs:240-258) can only name the parity shards that disagree.  broken is ready to become EcShardInfos (delete
// those files, then rebuild); details say where, one line per blamed shard and one for columns damaged in more shards
// than one (radius 1) that no single shard explains.
func swecLocateEcDamage(baseFileName string, ctx *ECContext, additionalDirs []string) (broken []uint32, details []string, err error) {
	cs := C.CString(baseFileName)
	defer C.free(unsafe.Pointer(cs))
	dirs := make([]*C.char, len(additionalDirs)+1)
	for i, d := range additionalDirs {
		dirs[i] = C.CString(d)
		defer C.free(unsafe.Pointer(dirs[i]))
	}
	var report C.swec_damage_report
	var nRanges, ok C.int
	if err := swecCall(func() C.int {
		return C.swec_locate_ec_damage(cs, (**C.char)(unsafe.Pointer(&dirs[0])), C.int(len(additionalDirs)),
			C.int(ctx.DataShards), C.int(ctx.ParityShards), swecPickDevice(), 1, &report, nil, 0, &nRanges, &ok)
	}); err != nil {
		return nil, nil, fmt.Errorf("locate ec damage: %w", err)
	}
	for i := 0; i < ctx.DataShards+ctx.ParityShards; i++ {
		if n := uint64(report.shard_bytes[i]); n > 0 {
			broken = append(broken, uint32(i))
			details = append(details, fmt.Sprintf("ec shard %d: %d bytes do not match the other shards, offsets %d..%d",
				i, n, int64(report.shard_first[i]), int64(report.shard_last[i])))
		}
	}
	if report.uncorrectable_columns > 0 {
		details = append(details, fmt.Sprintf("%d byte columns are damaged in more shards than can be located, offsets %d..%d",
			uint64(report.uncorrectable_columns), int64(report.first_uncorrectable), int64(report.last_uncorrectable)))
	}
	return broken, details, nil
}

// swecPageSketchFile answers the shard holder's side of a distributed parity scrub (a VolumeEcShardSketch RPC): the
// page sketches of one local shard file, 8 bytes per 4 KiB page, under the coordinator's seed.  The caller must check
// that the coordinator asked for SWEC_PAGE_SKETCH_VERSION.  The file is only read.
func swecPageSketchFile(shardFileName string, seed uint64) (sketches []uint64, shardSize int64, err error) {
	cs := C.CString(shardFileName)
	defer C.free(unsafe.Pointer(cs))
	st, err := os.Stat(shardFileName)
	if err != nil {
		return nil, 0, err
	}
	for capPages := (st.Size() + 4095) / 4096; ; {
		buf := make([]uint64, capPages+1) // +1: never a zero-length slice to take the address of
		var length, nPages C.int64_t
		if err := swecCall(func() C.int {
			return C.swec_page_sketch_file(cs, swecPickDevice(), C.uint64_t(seed), (*C.uint64_t)(unsafe.Pointer(&buf[0])),
				C.int64_t(capPages), &length, &nPages)
		}); err != nil {
			return nil, 0, fmt.Errorf("page sketch %s: %w", shardFileName, err)
		}
		if int64(nPages) <= capPages {
			return buf[:nPages], int64(length), nil
		}
		capPages = int64(nPages) // the file grew since the stat
	}
}

// swecSketchPage is one page the coordinator must fetch: blamed on the shards of Blamed (bit i = shard i), or
// Uncorrectable (fetch it from all k+m shards and run swec_correct_damage_device on them).
type swecSketchPage struct {
	Page          int64
	Blamed        uint32
	Uncorrectable bool
}

// swecLocateSketchDamage is the coordinator's side (the ScrubEcVolume FULL handler or ec.scrub): the pages of a balanced
// volume that are damaged, from every shard holder's sketches and shard size, all taken with one fresh seed.  Unequal
// sizes are the ErrShardSize of a rebuild; a shard whose holder did not answer must be rebuilt first.  Radius 1 blames a
// page on one shard; a page damaged in two shards comes back Uncorrectable even when no column of it is (INTEGRATION.md).
func swecLocateSketchDamage(enc *swecEncoder, sketches [][]uint64, shardSizes []int64) (pages []swecSketchPage, err error) {
	for _, s := range shardSizes[1:] {
		if s != shardSizes[0] {
			return nil, fmt.Errorf("ec shard size expected %d actual %d", shardSizes[0], s)
		}
	}
	nPages := (shardSizes[0] + 4095) / 4096
	var p runtime.Pinner
	defer p.Unpin()
	ptrs := (*[C.SWEC_MAX_SHARDS]*C.uint64_t)(C.calloc(C.SWEC_MAX_SHARDS, C.size_t(unsafe.Sizeof(uintptr(0)))))
	defer C.free(unsafe.Pointer(ptrs))
	for i, s := range sketches {
		if int64(len(s)) != nPages {
			return nil, fmt.Errorf("ec shard %d: %d sketches for %d pages", i, len(s), nPages)
		}
		if nPages > 0 {
			p.Pin(&s[0])
			ptrs[i] = (*C.uint64_t)(unsafe.Pointer(&s[0]))
		}
	}
	out := make([]C.swec_sketch_page, nPages+1)
	var nFlagged C.int64_t
	var ok C.int
	if err := swecCall(func() C.int {
		return C.swec_locate_sketch_damage(enc.h, &ptrs[0], C.int64_t(shardSizes[0]), 1, &out[0], C.int64_t(nPages),
			&nFlagged, nil, &ok)
	}); err != nil {
		return nil, fmt.Errorf("locate sketch damage: %w", err)
	}
	for _, q := range out[:nFlagged] {
		pages = append(pages, swecSketchPage{int64(q.page), uint32(q.blamed_mask), q.uncorrectable != 0})
	}
	return pages, nil
}

// swecLocateSketchDamageChecked is swecLocateSketchDamage for a volume with lost shards (a nil sketch; its shardSizes
// entry is ignored), before ec.rebuild.  The first k present shards are checked against the other c present ones at
// radius min(1, c/2); with c = 0 nothing is checked and no page comes back.  Repair the blamed pages at their holders
// first (a page blamed on B has k present shards outside B), then rebuild.  rebuilt[id] is the sketch lost shard id must
// have afterwards: sketch the rebuilt file with the same seed and compare it outside the Uncorrectable pages, where the
// prediction is what the plain rebuild writes from the shards as found (INTEGRATION.md).
func swecLocateSketchDamageChecked(enc *swecEncoder, sketches [][]uint64, shardSizes []int64) (pages []swecSketchPage, rebuilt map[int][]uint64, err error) {
	size := int64(-1)
	for i, s := range sketches {
		if s == nil {
			continue
		}
		if size < 0 {
			size = shardSizes[i]
		} else if shardSizes[i] != size {
			return nil, nil, fmt.Errorf("ec shard size expected %d actual %d", size, shardSizes[i])
		}
	}
	if size < 0 {
		size = 0 // no shard present: the call reports too few shards
	}
	nPages := (size + 4095) / 4096
	var p runtime.Pinner
	defer p.Unpin()
	ptrs := (*[C.SWEC_MAX_SHARDS]*C.uint64_t)(C.calloc(C.SWEC_MAX_SHARDS, C.size_t(unsafe.Sizeof(uintptr(0)))))
	defer C.free(unsafe.Pointer(ptrs))
	outs := (*[C.SWEC_MAX_SHARDS]*C.uint64_t)(C.calloc(C.SWEC_MAX_SHARDS, C.size_t(unsafe.Sizeof(uintptr(0)))))
	defer C.free(unsafe.Pointer(outs))
	rebuilt = map[int][]uint64{}
	for i, s := range sketches {
		if s == nil {
			r := make([]uint64, nPages+1) // +1: never a zero-length slice to take the address of
			p.Pin(&r[0])
			outs[i] = (*C.uint64_t)(unsafe.Pointer(&r[0]))
			rebuilt[i] = r[:nPages]
			continue
		}
		if int64(len(s)) != nPages {
			return nil, nil, fmt.Errorf("ec shard %d: %d sketches for %d pages", i, len(s), nPages)
		}
		if nPages == 0 {
			s = make([]uint64, 1) // present, with no pages: NULL would mark it lost
		}
		p.Pin(&s[0])
		ptrs[i] = (*C.uint64_t)(unsafe.Pointer(&s[0]))
	}
	out := make([]C.swec_sketch_page, nPages+1)
	var nFlagged C.int64_t
	var ok C.int
	if err := swecCall(func() C.int {
		return C.swec_locate_sketch_damage_checked(enc.h, &ptrs[0], C.int64_t(size), 1, &out[0], C.int64_t(nPages),
			&nFlagged, nil, &outs[0], &ok)
	}); err != nil {
		return nil, nil, fmt.Errorf("locate sketch damage (checked): %w", err)
	}
	for _, q := range out[:nFlagged] {
		pages = append(pages, swecSketchPage{int64(q.page), uint32(q.blamed_mask), q.uncorrectable != 0})
	}
	return pages, rebuilt, nil
}

// swecRepairEcDamage is swecLocateEcDamage, which also corrects the located bytes in the shard files: only the damaged
// pages of the damaged shards are rewritten, so scattered bit rot in more than ParityShards shards is still repaired,
// where deleting and rebuilding that many shards is impossible.  repaired are the shards written; details say where.
// Fall back to delete-and-rebuild in two cases: details report uncorrectable columns (more wrong shards in a column
// than radius 1 corrects; those columns are left as they were), or a shard file is missing (the call fails with
// SWEC_ERR_TOO_FEW_SHARDS: rebuild first, then repair).  Radius 1 never miscorrects a column with up to ParityShards-1
// wrong shards.  Nobody else may write the shard files during the call.
func swecRepairEcDamage(baseFileName string, ctx *ECContext, additionalDirs []string) (repaired []uint32, details []string, err error) {
	cs := C.CString(baseFileName)
	defer C.free(unsafe.Pointer(cs))
	dirs := make([]*C.char, len(additionalDirs)+1)
	for i, d := range additionalDirs {
		dirs[i] = C.CString(d)
		defer C.free(unsafe.Pointer(dirs[i]))
	}
	var report C.swec_damage_report
	var nRanges, ok C.int
	if err := swecCall(func() C.int {
		return C.swec_repair_ec_damage(cs, (**C.char)(unsafe.Pointer(&dirs[0])), C.int(len(additionalDirs)),
			C.int(ctx.DataShards), C.int(ctx.ParityShards), swecPickDevice(), 1, &report, nil, 0, &nRanges, &ok)
	}); err != nil {
		return nil, nil, fmt.Errorf("repair ec damage: %w", err)
	}
	for i := 0; i < ctx.DataShards+ctx.ParityShards; i++ {
		if n := uint64(report.shard_bytes[i]); n > 0 {
			repaired = append(repaired, uint32(i))
			details = append(details, fmt.Sprintf("ec shard %d: %d bytes corrected, offsets %d..%d",
				i, n, int64(report.shard_first[i]), int64(report.shard_last[i])))
		}
	}
	if report.uncorrectable_columns > 0 {
		details = append(details, fmt.Sprintf("%d byte columns are damaged in more shards than can be corrected, offsets %d..%d",
			uint64(report.uncorrectable_columns), int64(report.first_uncorrectable), int64(report.last_uncorrectable)))
	}
	return repaired, details, nil
}

// swecRebuildEcFilesChecked is RebuildEcFiles reading every present shard (rebuildEcFiles, ec_encoder.go:342-357),
// which corrects the damage it locates in the shards it rebuilds from instead of copying it into every rebuilt shard:
// a lost disk plus bit rot on the others is the common case.  Use radius 1 by default.  Use radius 0 when two or more
// shards are lost and no guess is wanted: with few check shards left, radius 1 can blame the wrong shard, and radius 0
// only reports the damaged columns, rebuilding them as plain rebuild does.  Present shard files are never written; run
// swecRepairEcDamage on the completed set afterwards to fix them.  details say where damage was found or left.
func swecRebuildEcFilesChecked(baseFileName string, ctx *ECContext, additionalDirs []string, radius int) (generated []uint32, details []string, err error) {
	cs := C.CString(baseFileName)
	defer C.free(unsafe.Pointer(cs))
	dirs := make([]*C.char, len(additionalDirs)+1)
	for i, d := range additionalDirs {
		dirs[i] = C.CString(d)
		defer C.free(unsafe.Pointer(dirs[i]))
	}
	var ids [C.SWEC_MAX_SHARDS]C.uint32_t
	var report C.swec_damage_report
	var nIds, nRanges, ok C.int
	if err := swecCall(func() C.int {
		return C.swec_rebuild_ec_files_checked(cs, (**C.char)(unsafe.Pointer(&dirs[0])), C.int(len(additionalDirs)),
			C.int(ctx.DataShards), C.int(ctx.ParityShards), swecPickDevice(), C.int(radius), &ids[0], &nIds, &report,
			nil, 0, &nRanges, &ok)
	}); err != nil {
		return nil, nil, fmt.Errorf("rebuild ec files checked: %w", err)
	}
	for i := 0; i < int(nIds); i++ {
		generated = append(generated, uint32(ids[i]))
	}
	for i := 0; i < ctx.DataShards+ctx.ParityShards; i++ {
		if n := uint64(report.shard_bytes[i]); n > 0 {
			details = append(details, fmt.Sprintf("ec shard %d: %d bytes wrong, kept out of the rebuilt shards, offsets %d..%d",
				i, n, int64(report.shard_first[i]), int64(report.shard_last[i])))
		}
	}
	if report.uncorrectable_columns > 0 {
		details = append(details, fmt.Sprintf("%d byte columns are damaged in more shards than can be corrected, rebuilt from the shards as found, offsets %d..%d",
			uint64(report.uncorrectable_columns), int64(report.first_uncorrectable), int64(report.last_uncorrectable)))
	}
	return generated, details, nil
}

// swecHealEcFiles is swecRebuildEcFilesChecked that also corrects the damage it locates in the present shard files, in
// the same full read plus a re-read of the flagged pages: the lost shards are rebuilt and the damaged present ones
// repaired in place, where the checked rebuild followed by swecRepairEcDamage reads every shard twice.  Columns with
// more wrong shards than the radius corrects are left as they were (details say where); the two-call flow could rewrite
// such a column into a wrong codeword.  Only the blamed shards' flagged pages are rewritten, so nobody else may write
// the shard files during the call.  generated are the rebuilt ids; details say what was corrected or left.
func swecHealEcFiles(baseFileName string, ctx *ECContext, additionalDirs []string, radius int) (generated []uint32, details []string, err error) {
	cs := C.CString(baseFileName)
	defer C.free(unsafe.Pointer(cs))
	dirs := make([]*C.char, len(additionalDirs)+1)
	for i, d := range additionalDirs {
		dirs[i] = C.CString(d)
		defer C.free(unsafe.Pointer(dirs[i]))
	}
	var ids [C.SWEC_MAX_SHARDS]C.uint32_t
	var report C.swec_damage_report
	var nIds, nRanges, ok C.int
	if err := swecCall(func() C.int {
		return C.swec_heal_ec_files(cs, (**C.char)(unsafe.Pointer(&dirs[0])), C.int(len(additionalDirs)),
			C.int(ctx.DataShards), C.int(ctx.ParityShards), swecPickDevice(), C.int(radius), &ids[0], &nIds, &report,
			nil, 0, &nRanges, &ok)
	}); err != nil {
		return nil, nil, fmt.Errorf("heal ec files: %w", err)
	}
	generated, details = swecHealResult(ids[:nIds], &report)
	return generated, details, nil
}

// ecShardsHealSwec is ecShardsRebuildSwec through swecHealEcFiles: RebuildEcFiles healing the present shards, then
// RebuildEcxFile, in VolumeEcShardsRebuild (:149-225).  The ratio comes from .vif, else 10+4.
func ecShardsHealSwec(dataBaseFileName, indexBaseFileName string, additionalDirs []string, radius int) (generated []uint32, details []string, err error) {
	cd, ci := C.CString(dataBaseFileName), C.CString(indexBaseFileName)
	defer C.free(unsafe.Pointer(cd))
	defer C.free(unsafe.Pointer(ci))
	dirs := make([]*C.char, len(additionalDirs)+1)
	for i, d := range additionalDirs {
		dirs[i] = C.CString(d)
		defer C.free(unsafe.Pointer(dirs[i]))
	}
	var ids [C.SWEC_MAX_SHARDS]C.uint32_t
	var report C.swec_damage_report
	var nIds, nRanges, ok C.int
	if err := swecCall(func() C.int {
		return C.swec_ec_shards_heal(cd, ci, (**C.char)(unsafe.Pointer(&dirs[0])), C.int(len(additionalDirs)),
			swecPickDevice(), C.int(radius), &ids[0], &nIds, &report, nil, 0, &nRanges, &ok)
	}); err != nil {
		return nil, nil, fmt.Errorf("heal ec shards: %w", err)
	}
	generated, details = swecHealResult(ids[:nIds], &report)
	return generated, details, nil
}

func swecHealResult(ids []C.uint32_t, report *C.swec_damage_report) (generated []uint32, details []string) {
	for _, id := range ids {
		generated = append(generated, uint32(id))
	}
	for i := 0; i < C.SWEC_MAX_SHARDS; i++ {
		if n := uint64(report.shard_bytes[i]); n > 0 {
			details = append(details, fmt.Sprintf("ec shard %d: %d bytes corrected, offsets %d..%d",
				i, n, int64(report.shard_first[i]), int64(report.shard_last[i])))
		}
	}
	if report.uncorrectable_columns > 0 {
		details = append(details, fmt.Sprintf("%d byte columns are damaged in more shards than can be corrected, left as they were and rebuilt from the shards as found, offsets %d..%d",
			uint64(report.uncorrectable_columns), int64(report.first_uncorrectable), int64(report.last_uncorrectable)))
	}
	return generated, details
}

// ---- pinned batch buffers ---------------------------------------------------------------------------------
// runtime.Pinner only stops the Go GC from moving a slice; to CUDA such memory is PAGEABLE, so every Encode /
// Reconstruct on it bounces through the library's pinned ring (a memcpy per shard each way).  The batch buffers of
// the two file loops are allocated once per volume and reused for every batch, so they are the place to hand the
// library memory it can DMA — or read from the kernel — directly:
//
//   encodeDatFile      ec_encoder.go:289-292   buffers[i] = make([]byte, bufferSize)   ×TotalShards
//   rebuildEcFiles     ec_encoder.go:330-335   buffers[i] = make([]byte, ErasureCodingSmallBlockSize) ×TotalShards
//   recoverOneRemoteEcShardInterval  store_ec.go:493-500   bufs[i] = make([]byte, len(buf))  (per degraded read)
//
// become   buffers, release := swecAllocShardBuffers(ctx.Total(), bufferSize); defer release()
//
// The n slices are cut from ONE pinned, GPU-mapped allocation on the GPU's NUMA node at a constant pitch: the library
// recognises that shape and moves all k inputs (and all m outputs) with one strided DMA each way, or — for calls up to
// 2 MiB per shard — runs the kernel directly on the host memory over PCIe (include/swec.h "host_zero_copy").
// The memory is C memory: no Pinner, no cgo pointer-passing rules, and the slices must not outlive release().
func swecAllocShardBuffers(n int, shardLen int) (bufs [][]byte, release func()) {
	pitch := (shardLen + 4095) &^ 4095
	dev := swecPickDevice()
	base := C.swec_alloc_pinned_for_device(dev, C.size_t(n*pitch))
	if base == nil { // no GPU / out of pinned memory: plain Go memory still works (pageable path)
		bufs = make([][]byte, n)
		for i := range bufs {
			bufs[i] = make([]byte, shardLen)
		}
		return bufs, func() {}
	}
	bufs = make([][]byte, n)
	for i := range bufs {
		bufs[i] = unsafe.Slice((*byte)(unsafe.Add(base, i*pitch)), shardLen)
	}
	return bufs, func() { C.swec_free_pinned(base) }
}
