// Package model -- cgo shims for the model-level boundary: the transformer's weights, KV cache and
// activations live in HBM; LlamaTransformer.Forward is ONE call through the C-ABI.
//
// Integration points in the reference (signatures unchanged):
//   NewLlamaTransformer  src/model/llamatransformer.go:64-113   -> lnb_model_create + upload of every getTensor result
//   NewInferenceContext  src/model/inferencecontext.go:17-46    -> lnb_session_create
//   (*LlamaTransformer).Forward  src/model/llamatransformer.go:145-180 -> lnb_forward
//   (*Model).Free        src/model/model.go:56                  -> lnb_model_destroy
// NOT compiled in this repository (no Go toolchain in the build image; see INTEGRATION.md).
package model

/*
#cgo CFLAGS: -I${SRCDIR}/../../include
#cgo LDFLAGS: -L${SRCDIR}/../../llama-nuts-and-bolts_b200 -llnb -lcudart -ldl
#include <stdlib.h>
#include "lnb.h"
*/
import "C"

import (
	"fmt"
	"unsafe"

	"github.com/adalkiran/llama-nuts-and-bolts/src/common"
	"github.com/adalkiran/llama-nuts-and-bolts/src/ml"
)

func lnbErr(rc C.int) error {
	if rc >= 0 {
		return nil
	}
	return fmt.Errorf("lnb: %s", C.GoString(C.lnb_last_error()))
}

type deviceModel struct{ h *C.lnb_model }
type deviceSession struct{ h *C.lnb_session }

// called at the end of NewLlamaTransformer, after every getTensor succeeded.  weightFormat: C.LNB_WEIGHTS_BF16, or
// C.LNB_WEIGHTS_MXFP8 / C.LNB_WEIGHTS_MXFP4 to quantize the linear weights at finalize (tpSize 1 only)
func newDeviceModel(args *ModelArgs, tensors map[string]*ml.Tensor, device, tpRank, tpSize int, ncclID []byte,
	weightFormat int) (*deviceModel, error) {
	ca := C.lnb_model_args{
		dim: C.int32_t(args.Dim), n_layers: C.int32_t(args.N_Layers), n_heads: C.int32_t(args.N_Heads),
		n_kv_heads: C.int32_t(args.N_KVHeads), head_dim: C.int32_t(args.HeadDim), ffn_dim: C.int32_t(args.FFNDim),
		vocab_size: C.int32_t(args.VocabSize), max_seq_len: C.int32_t(args.MaxSequenceLength),
		norm_eps: C.float(args.NormEpsilon), rope_theta: C.double(args.RopeTheta),
	}
	if args.UseScaledRope {
		ca.use_scaled_rope = 1
	}
	var id unsafe.Pointer
	if tpSize > 1 {
		id = C.CBytes(ncclID) // 128 bytes from lnb_nccl_unique_id of rank 0
		defer C.free(id)
	}
	dm := &deviceModel{}
	if err := lnbErr(C.lnb_model_create(&ca, C.int(device), C.int(tpRank), C.int(tpSize), id, &dm.h)); err != nil {
		return nil, err
	}
	if err := lnbErr(C.lnb_model_set_weight_format(dm.h, C.int(weightFormat))); err != nil {
		C.lnb_model_destroy(dm.h)
		return nil, err
	}
	for name, t := range tensors { // RawData aliases the checkpoint mmap (src/torch/types.go:51-56); the library copies it
		cname := C.CString(name)
		shape := make([]C.int64_t, len(t.Size))
		for i, d := range t.Size {
			shape[i] = C.int64_t(d)
		}
		rc := C.lnb_model_upload_tensor(dm.h, cname, (*C.uint16_t)(unsafe.Pointer(&t.RawData[0])), &shape[0], C.int(len(shape)))
		C.free(unsafe.Pointer(cname))
		if err := lnbErr(rc); err != nil {
			return nil, err
		}
	}
	// the tables may also be uploaded from the Go-computed PrecomputedFreqsCis / TABLE_SILU:
	// lnb_model_set_rope_table / lnb_model_set_silu_table; by default the library builds identical ones
	return dm, lnbErr(C.lnb_model_finalize(dm.h))
}

// the E4M3 codes [rows*cols] and E8M0 scales [rows*ceil(cols/32)] of a linear tensor of an MXFP8 model (tests, tools)
func (dm *deviceModel) mxfp8Read(name string, rows, cols int) ([]byte, []byte, error) {
	codes := make([]byte, rows*cols)
	scales := make([]byte, rows*((cols+31)/32))
	cname := C.CString(name)
	defer C.free(unsafe.Pointer(cname))
	rc := C.lnb_model_mxfp8_read(dm.h, cname, (*C.uint8_t)(unsafe.Pointer(&codes[0])), (*C.uint8_t)(unsafe.Pointer(&scales[0])))
	return codes, scales, lnbErr(rc)
}

// the E2M1 codes [rows*cols/2] (the even column in a byte's low nibble) and E8M0 scales [rows*ceil(cols/32)] of a linear
// tensor of an MXFP4 model (tests, tools)
func (dm *deviceModel) mxfp4Read(name string, rows, cols int) ([]byte, []byte, error) {
	codes := make([]byte, rows*(cols/2))
	scales := make([]byte, rows*((cols+31)/32))
	cname := C.CString(name)
	defer C.free(unsafe.Pointer(cname))
	rc := C.lnb_model_mxfp4_read(dm.h, cname, (*C.uint8_t)(unsafe.Pointer(&codes[0])), (*C.uint8_t)(unsafe.Pointer(&scales[0])))
	return codes, scales, lnbErr(rc)
}

// the format of the linear weights, the weight bytes held in HBM and the weight bytes one S = 1 step reads
func (dm *deviceModel) weightInfo() (format int, deviceBytes, stepBytes int64, err error) {
	var f C.int
	var d, s C.int64_t
	err = lnbErr(C.lnb_model_weight_info(dm.h, &f, &d, &s))
	return int(f), int64(d), int64(s), err
}

func newDeviceSession(dm *deviceModel, inferenceArgs common.InferenceArgs, maxRows int, accMode int) (*deviceSession, error) {
	ds := &deviceSession{}
	return ds, lnbErr(C.lnb_session_create(dm.h, C.int(inferenceArgs.SequenceLength), C.int(maxRows), C.int(accMode), &ds.h))
}

// newDeviceSessionKV: newDeviceSession with n_seq sequences and the KV cache in format kvFormat (C.LNB_KV_BF16 or
// C.LNB_KV_MXFP8, lnb_session_create_kv)
func newDeviceSessionKV(dm *deviceModel, inferenceArgs common.InferenceArgs, nSeq, maxRows, accMode, kvFormat int) (*deviceSession, error) {
	ds := &deviceSession{}
	return ds, lnbErr(C.lnb_session_create_kv(dm.h, C.int(inferenceArgs.SequenceLength), C.int(nSeq), C.int(maxRows), C.int(accMode),
		C.int(kvFormat), &ds.h))
}

// deviceLogits is what Forward returns when the logits stay in HBM (lnb_forward_device): ml.Tensor carries it instead of
// S x vocab floats; Slice keeps it and ml.Argmax on such a tensor calls argmaxRows (4 bytes per row over PCIe), anything
// that touches RawData calls read.  Valid until the session's next forward.
type deviceLogits struct {
	ds         *deviceSession
	generation C.int64_t
	rows       int
}

func (ds *deviceSession) forwardDevice(inputTokens *ml.Tensor, startPos int, allRows bool) (*deviceLogits, error) {
	s := inputTokens.Size[0]
	if s == 0 {
		return nil, fmt.Errorf("empty token array")
	}
	d := &deviceLogits{ds: ds, rows: 1}
	if allRows {
		d.rows = s
	}
	rc := C.lnb_forward_device(ds.h, (*C.int32_t)(unsafe.Pointer(&inputTokens.RawData[0])), C.int(s), C.int(startPos), C.int(d.rows),
		nil, &d.generation)
	return d, lnbErr(rc)
}

func (d *deviceLogits) argmaxRows(row0, rows int) ([]int32, error) {
	out := make([]int32, rows)
	rc := C.lnb_session_logits_argmax(d.ds.h, d.generation, C.int(row0), C.int(rows), (*C.int32_t)(unsafe.Pointer(&out[0])))
	return out, lnbErr(rc)
}

func (d *deviceLogits) read(row0, rows, vocab int) (*ml.Tensor, error) {
	t := ml.NewEmptyTensor([]int{rows, vocab}, ml.DT_F32)
	rc := C.lnb_session_logits_read(d.ds.h, d.generation, C.int(row0), C.int(rows), (*C.float)(unsafe.Pointer(&t.RawData[0])))
	return t, lnbErr(rc)
}

// chunked prefill (extension): S > 1 at startPos > 0 with the [S,T] causal mask
func (ds *deviceSession) allowChunkedPrefill(on bool) error {
	v := C.int(0)
	if on {
		v = 1
	}
	return lnbErr(C.lnb_session_set_chunked_prefill(ds.h, v))
}

// after an LNB_ETIMEOUT of the peer all-reduce: back to ncclAllReduce (every rank must do the same)
func (ds *deviceSession) disablePeerAllReduce() error { return lnbErr(C.lnb_session_p2p_disable(ds.h)) }

// body of (*LlamaTransformer).Forward: tokens [S] int32 -> logits [S, vocab] f32
func (ds *deviceSession) forward(inputTokens *ml.Tensor, startPos int, vocab int) (*ml.Tensor, error) {
	s := inputTokens.Size[0]
	if s == 0 {
		return nil, fmt.Errorf("empty token array")
	}
	logits := ml.NewEmptyTensor([]int{s, vocab}, ml.DT_F32)
	rc := C.lnb_forward(ds.h, (*C.int32_t)(unsafe.Pointer(&inputTokens.RawData[0])), C.int(s), C.int(startPos),
		(*C.float)(unsafe.Pointer(&logits.RawData[0])), 1, nil)
	return logits, lnbErr(rc)
}
